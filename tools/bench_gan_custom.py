"""Images/s of the reference's own train_D / train_G (/ train_Q) as an override, trained by the reference loop over the
differentiable G, autoencoder D and Q, against the fused train() of the same MLP BEGAN / InfoGAN, in one run.  One JSON
line per (model, batch).

    python tools/bench_gan_custom.py [--models began,info] [--batch-sizes 64,4096] [--batches 20] [--epochs 2]

The first epoch of each leg warms up (plans, buffers, the allocator); then --repeats timed runs of --epochs epochs each
alternate between the legs (host clock around epochs that end in a device synchronise), and the median, min and max are
reported.  Both legs read their batches from the same host DataLoader (process_batch, as the reference does)."""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "generative-models_b200")]

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402


def _began_override(be_gan):
    class Custom(be_gan.BEGANTrainer):                  # src/be_gan.py:212-258
        def train_D(self, images, K):
            DX_reconst = self.model.D(images)
            DX_loss = torch.mean(torch.sum(torch.abs(DX_reconst - images), dim=1))
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            G_output = self.model.G(noise)
            DG_reconst = self.model.D(G_output)
            DG_loss = torch.mean(torch.sum(torch.abs(DG_reconst - G_output), dim=1))
            return DX_loss - (K * DG_loss), DX_loss, DG_loss

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            G_output = self.model.G(noise)
            DG_reconst = self.model.D(G_output)
            return torch.mean(torch.sum(torch.abs(DG_reconst - G_output), dim=1))
    return Custom


def _info_override(info_gan):
    class Custom(info_gan.InfoGANTrainer):              # src/info_gan.py:223-304
        def train_D(self, images):
            DX_score = self.model.D(images)
            noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim)
            DG_score = self.model.D(self.model.G(noise))
            return torch.sum(-torch.mean(torch.log(DX_score + 1e-8) + torch.log(1 - DG_score + 1e-8)))

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim)
            DG_score = self.model.D(self.model.G(noise))
            return -torch.mean(torch.log(DG_score + 1e-8))

        def train_Q(self, images, LAMBDA=1):
            m = self.model
            noise = self.compute_noise(images.shape[0], m.z_dim, m.disc_dim, m.cont_dim)
            Q_discrete, Q_continuous = m.Q(m.G(noise))
            disc_loss = F.cross_entropy(Q_discrete, torch.max(noise[:, m.z_dim:m.z_dim + m.disc_dim], 1)[1])
            cont_loss = F.mse_loss(Q_continuous, noise[:, m.z_dim + m.disc_dim:])
            return LAMBDA * (disc_loss + cont_loss)
    return Custom


def _trainer(name, custom, B, batches):
    import be_gan
    import info_gan
    torch.manual_seed(0)
    imgs = (torch.rand(B * batches, 1, 28, 28) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(len(imgs))), batch_size=B)
    if name == "began":
        model, Trainer = be_gan.BEGAN(784, 400, 20), (_began_override(be_gan) if custom else be_gan.BEGANTrainer)
    else:
        model, Trainer = info_gan.InfoGAN(784, 400, 20, 10, 10), (_info_override(info_gan) if custom else info_gan.InfoGANTrainer)
    tr = Trainer(model, loader, loader, loader)
    _quiet(lambda: tr.train(num_epochs=1))              # warm-up epoch
    return tr, len(imgs)


def _quiet(fn):
    with contextlib.redirect_stdout(io.StringIO()):
        fn()


def _rate(fn, images):
    torch.cuda.synchronize()
    t = time.perf_counter()
    _quiet(fn)
    torch.cuda.synchronize()
    return images / (time.perf_counter() - t)


def _stats(v, digits=1):
    v = sorted(v)
    return dict(median=round(v[len(v) // 2], digits), min=round(v[0], digits), max=round(v[-1], digits))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="began,info")
    ap.add_argument("--batch-sizes", default="64,4096")
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5, help="timed runs per leg, the legs alternated")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for name in a.models.split(","):
        for B in [int(b) for b in a.batch_sizes.split(",")]:
            (fused, n), (custom, _) = _trainer(name, False, B, a.batches), _trainer(name, True, B, a.batches)
            rates = {"fused": [], "override": []}
            for _ in range(a.repeats):
                rates["fused"].append(_rate(lambda: fused.train(num_epochs=a.epochs), a.epochs * n))
                rates["override"].append(_rate(lambda: custom.train(num_epochs=a.epochs), a.epochs * n))
            ratio = [c / f for c, f in zip(rates["override"], rates["fused"])]
            print(json.dumps(dict(model=name, batch=B, gpu=gpu, repeats=a.repeats, fused_images_per_s=_stats(rates["fused"]),
                                  override_images_per_s=_stats(rates["override"]),
                                  override_over_fused=_stats(ratio, 3))))
            sys.stdout.flush()
            del fused, custom
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
