"""Images/s of a user-written compute_batch (the reference's own body as an override, trained by the reference loop over
the differentiable encoder / decoder) against the fused train() of the same model, in one run, for vae, ae, dc_vae and
dc_ae; and the device memory one encoder and one decoder slot hold.  One JSON line per model.

    python tools/bench_vae_custom.py [--models vae,ae,dc_vae,dc_ae] [--batches 20] [--epochs 2]

The first epoch of each leg warms up (plans, buffers, the allocator); then --repeats timed runs of --epochs epochs each
alternate between the legs (host clock around epochs that end in a device synchronise), and the median, min and max are
reported.  loader_only is the host loader alone (collate and copy to the device), the ceiling of both legs.  The loaders are in host memory for both legs: the fused MLP VAE's
resident-dataset path and the conv trainers' device_dataset are off, so the two legs read the same batches."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "generative-models_b200")]

import torch  # noqa: E402

SPEC = {  # module, model class, trainer class, model kwargs, image shape, batch
    "vae": ("vae", "VAE", "VAETrainer", dict(image_size=784, hidden_dim=400, z_dim=20), (1, 28, 28), 128),
    "ae": ("ae", "Autoencoder", "AutoencoderTrainer", dict(image_size=784, hidden_dim=32), (1, 28, 28), 128),
    "dc_vae": ("dc_vae", "DCVAE", "DCVAETrainer", dict(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100), (3, 64, 64), 128),
    "dc_ae": ("dc_ae", "DCAutoencoder", "DCAutoencoderTrainer", dict(image_size=64 * 64 * 3, hidden_dim=64, z_dim=32), (3, 64, 64), 128),
}


def _override(Trainer, two_losses, to_cuda):
    def compute_batch(self, batch):                     # the reference's body (src/vae.py:193-208, src/ae.py:147-160)
        images, _ = batch
        images = to_cuda(images.view(images.shape[0], -1))
        if two_losses:
            outputs, mu, log_var = self.model(images)
            return torch.sum((images - outputs) ** 2), self.kl_divergence(mu, log_var)
        return torch.sum((images - self.model(images)) ** 2)
    return type("Custom" + Trainer.__name__, (Trainer,), {"compute_batch": compute_batch})


def _trainer(name, custom, batches):
    import importlib
    mod, mcls, tcls, kw, shape, B = SPEC[name]
    M = importlib.import_module(mod)
    torch.manual_seed(0)
    imgs = (torch.rand(B * batches, *shape) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(len(imgs))), batch_size=B)
    val = [next(iter(loader))]
    Trainer = getattr(M, tcls)
    if custom:
        Trainer = _override(Trainer, name.endswith("vae"), M.to_cuda)
    tr = Trainer(getattr(M, mcls)(**kw), loader, val, val)
    tr.device_noise = False
    tr.device_dataset = False
    tr.train(num_epochs=1)                              # warm-up epoch
    return tr, len(imgs)


def _rate(fn, images):
    torch.cuda.synchronize()
    t = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return images / (time.perf_counter() - t)


def _loader_pass(loader):
    """the host loader alone: every batch collated and copied to the device, as both legs read it"""
    for images, _ in loader:
        images.view(images.shape[0], -1).cuda()


def _stats(v):
    v = sorted(v)
    return dict(median=round(v[len(v) // 2], 1), min=round(v[0], 1), max=round(v[-1], 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default="vae,ae,dc_vae,dc_ae")
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--repeats", type=int, default=5, help="timed runs per leg, the legs alternated")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    for name in a.models.split(","):
        (fused, n), (custom, _) = _trainer(name, False, a.batches), _trainer(name, True, a.batches)
        rates = {"fused": [], "override": [], "loader": []}
        for _ in range(a.repeats):
            rates["fused"].append(_rate(lambda: fused.train(num_epochs=a.epochs), a.epochs * n))
            rates["override"].append(_rate(lambda: custom.train(num_epochs=a.epochs), a.epochs * n))
            rates["loader"].append(_rate(lambda: [_loader_pass(fused.train_iter) for _ in range(a.epochs)], a.epochs * n))
        eng = custom._engine
        if hasattr(eng, "slot_bytes"):
            slots = dict(zip(("encoder_slot_bytes", "decoder_slot_bytes"), eng.slot_bytes()))
        else:
            slots = {"conv_slot_buffers_bytes": sum(v.numel() * v.element_size() for k, v in eng._bufs.items() if k.startswith(("cd", "cg")))}
        ratio = [c / f for c, f in zip(rates["override"], rates["fused"])]
        print(json.dumps(dict(model=name, batch=SPEC[name][5], gpu=gpu, repeats=a.repeats,
                              fused_images_per_s=_stats(rates["fused"]), override_images_per_s=_stats(rates["override"]),
                              loader_only_images_per_s=_stats(rates["loader"]),
                              override_over_fused=_stats([round(r, 3) for r in ratio]), **slots)))
        sys.stdout.flush()
        del fused, custom, eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
