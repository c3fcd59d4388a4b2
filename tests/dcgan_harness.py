"""Shared pieces of the DCGAN conv path's GPU tests: the norm-relative error, the parity report, the seeded setup of an
engine and a plain-PyTorch oracle (oracle/dcgan_torch.py) holding the same weights, and the bodies of the checks that
several variants run alike (the drop-ins' driver lines, the penalised critics' split batch and penalty descent)."""
import importlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import dcgan_torch as O


def nrel(a, b):
    a, b = a.detach().double().reshape(-1).cpu(), b.detach().double().reshape(-1).cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


class Report(dict):
    """The measured errors of one test file, written to $GM_PARITY_DIR/parity_<name>.json when GM_PARITY_DIR is set."""

    def __init__(self, name):
        super().__init__()
        self.name = name

    def add(self, key, rep):
        self[key] = rep
        out = os.environ.get("GM_PARITY_DIR")
        if not out:
            return
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_%s.json" % self.name), "w") as f:
            json.dump(self, f, indent=1, sort_keys=True)


def setup(variant="ns", out_act=None, hd=16, z=100, wstd=0.05, seed=11):
    """engine + oracle G / D with the same weights: N(0, wstd) conv weights from torch.Generator(seed) (better conditioned
    than DCGAN's 0.02: D's outputs spread over (0, 1) instead of sitting at 0.5).  A batch-norm D and G evaluate at the
    CUDA path's bf16 storage points (O.bf16_points); a critic takes its rounding per call.  Returns (eng, G, D, the
    generator) so that callers continue the same stream of draws."""
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant=variant, d_out_act=out_act)
    g = torch.Generator().manual_seed(seed)
    for net in (eng.G, eng.D):
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.D.view("l5.weight")[1:].zero_()
    eng.G.refresh(); eng.D.refresh()
    G = O.Generator(hd, z)
    D = O.Discriminator(hd) if eng.d_bn else O.Critic(hd, 3, eng.d_out_act)
    sd = eng.torch_weights()
    assert eng.d_bn or not any(k.startswith("D.bn") for k in sd)
    O.load_from_engine_weights(G, D, sd)
    G.train(); D.train()
    if eng.d_bn:
        G.q = D.q = staticmethod(O.bf16_points)
    return eng, G, D, g


def critic_setup(variant, out_act=None, n=8, live="xhat"):
    """setup() of a penalised critic ("wgp" or "dra") and n images, noise and the penalty's random inputs drawn after the
    weights: (eps,) for WGAN-GP, (delta, u) for DRAGAN.  For a relu critic the last layer's sign is chosen so that at
    least half of the x_hat rows (live="xhat") or of the generated rows (live="fake") are live (at a sign that kills them
    every row would compare zero with zero)."""
    eng, G, D, g = setup(variant, out_act)
    imgs = torch.rand(n, 3 * 64 * 64, generator=g)
    zz = torch.randn(n, 100, generator=g)
    if variant == "wgp":
        rnd = (torch.rand(n, generator=g),)
    else:
        rnd = (torch.rand(n, generator=g), torch.rand(n, 3 * 64 * 64, generator=g))
    if eng.d_out_act == "relu":
        with torch.no_grad():
            fake = G(zz)
            xh = O.interpolate(imgs, fake, rnd[0]) if live == "xhat" else fake
            if int((D.trace(xh)[0] > 0).sum()) < n // 2:
                eng.D.view("l5.weight").neg_(); eng.D.refresh()
                D.l5.weight.neg_()
    return eng, G, D, imgs, zz, rnd


# module, model, trainer, and the train() arguments of the reference's __main__ (src/ns_gan.py, src/w_gp_gan.py,
# src/ra_gan.py, src/fisher_gan.py, src/dra_gan.py)
_DROPINS = {"ns": ("dc_gan", "DCGAN", "DCGANTrainer", dict(G_lr=2e-4, D_lr=2e-4, D_steps=1)),
            "wgp": ("dc_w_gp_gan", "DCWGPGAN", "DCWGPGANTrainer", dict(G_lr=1e-4, D_lr=1e-4, D_steps=1)),
            "ra": ("dc_ra_gan", "DCRaNSGAN", "DCRaNSGANTrainer", dict(G_lr=2e-4, D_lr=2e-4, D_steps=1)),
            "fisher": ("dc_fisher_gan", "DCFisherGAN", "DCFisherGANTrainer", dict(G_lr=1e-4, D_lr=1e-4, D_steps=1, RHO=1e-6)),
            "dra": ("dc_dra_gan", "DCDRAGAN", "DCDRAGANTrainer", dict(G_lr=1e-4, D_lr=1e-4, D_steps=1))}


def run_reference_driver_lines(which):
    """The reference's driver lines on the conv drop-in `which` at hidden 16 and 64x64x3 synthetic images: train(), losses
    logged per step, generate_images, save_model / load_model round trip with torch-layout state_dict keys, and the loop
    body (loss.backward() delivers torch-layout gradients to the modules)."""
    import tempfile
    modname, model_name, trainer_name, train_args = _DROPINS[which]
    mod = importlib.import_module(modname)
    Model, Trainer = getattr(mod, model_name), getattr(mod, trainer_name)
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(64, 3, 64, 64, generator=g)
    if which == "ns":
        imgs = (imgs < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(64)), batch_size=16, shuffle=True)
    torch.manual_seed(3)
    model = Model(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    trainer = Trainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=2, **train_args)
    if which == "fisher":
        assert trainer.LAMBDA.shape == (1,) and float(trainer.LAMBDA) != 0.0 and float(trainer.RHO) == pytest.approx(1e-6)
    assert len(trainer.Dlosses) == 8 and len(trainer.Glosses) == 8
    assert all(np.isfinite(trainer.Dlosses)) and all(np.isfinite(trainer.Glosses))
    after = model.state_dict()
    if which == "ns":
        assert any(not torch.equal(before[k], after[k]) for k in before if k.endswith("weight"))   # parameters came back from the engine
    else:
        assert all(not torch.equal(before[k], after[k]) for k in before if k.startswith("D.l") and k.endswith("weight"))
        assert any(not torch.equal(before[k], after[k]) for k in before if k.startswith("G.") and k.endswith("weight"))
    out = trainer.generate_images(0, num_outputs=4)
    assert out.shape == (4, 3, 64, 64)
    if which == "ns":
        assert float(out.min()) >= 0 and float(out.max()) <= 1
    d = model.D(imgs[:8])
    if which == "wgp":
        assert d.shape == (8, 1) and float(d.min()) >= 0                                     # relu output
    else:
        assert d.shape == (8, 1) and float(d.min()) > 0 and float(d.max()) < 1               # sigmoid output
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        trainer.save_model(path)
        model2 = Model(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
        tr2 = Trainer(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        zz = torch.randn(4, 100)
        assert nrel(model2.G(zz), model.G(zz)) < 1e-6
        if which == "wgp":
            assert not any(k.startswith("D.bn") for k in model2.state_dict())
            assert nrel(model2.D(imgs[:4]), model.D(imgs[:4])) < 1e-6
    model.D.zero_grad()
    if which == "ns":
        loss = trainer.train_D(imgs[:16])
    elif which == "wgp":
        loss = trainer.train_D(imgs[:16].reshape(16, -1), LAMBDA=10)
    elif which == "fisher":
        loss, ipm = trainer.train_D(imgs[:16].reshape(16, -1))
        assert isinstance(ipm, float)
    elif which == "dra":
        loss = trainer.train_D(imgs[:16].reshape(16, -1), LAMBDA=10, K=1, C=1)
    else:
        loss = trainer.train_D(imgs[:16].reshape(16, -1))
    loss.backward()
    assert model.D.l4.weight.grad is not None and model.D.l4.weight.grad.shape == model.D.l4.weight.shape
    assert float(model.D.l4.weight.grad.abs().sum()) > 0
    gl = trainer.train_G(imgs[:16])
    gl.backward()
    assert np.isfinite(float(gl))


def split_batch_sums_to_the_full_batch(variant, report, key):
    """data-parallel contract on one GPU: the critic gradient of 2n images equals the SUM of the two n-image gradients
    computed with inv_global_batch = 1/(2n); the losses are local means.  DRAGAN's std(x) is summed over both halves
    through stats_reduce."""
    n = 4
    eng, G, D, imgs, z, rnd = critic_setup(variant, "none" if variant == "wgp" else None, n=2 * n)
    fake, _ = eng.g_forward(2 * n, z.cuda())
    fake = fake.clone()
    real = eng.stage_images(imgs.cuda())
    inv = 1.0 / (2 * n)
    rnd = [t.cuda() for t in rnd]
    if variant == "dra":
        loc = []
        for k in range(2):
            s = torch.zeros(2, device="cuda", dtype=torch.float64)
            eng.dra_std_sums(real[k * n * 4096:(k + 1) * n * 4096].clone(), n, s)
            loc.append(s)
        total = loc[0] + loc[1]
        eng.stats_reduce = lambda buf: buf.copy_(total)

    def critic_grad(x, f, m, r):
        if variant == "wgp":
            return eng.wgp_critic_grad(x, f, m, inv, 10.0, *r).item()
        return eng.dra_critic_grad(x, f, m, inv, 10.0, 1.0, 1.0, *r, stat_batch=2 * n).item()

    L = critic_grad(real, fake, 2 * n, rnd)
    full = eng.D.grads.clone()
    parts, losses = [], []
    for k in range(2):
        rows = slice(k * n * 4096, (k + 1) * n * 4096)
        losses.append(critic_grad(real[rows].clone(), fake[rows].clone(), n, [t[k * n:(k + 1) * n].clone() for t in rnd]))
        parts.append(eng.D.grads.clone())
    eng.stats_reduce = None
    rel = nrel(parts[0] + parts[1], full)
    report.add(key, {"grad_nrel": rel, "loss_abs": abs(L - 0.5 * (losses[0] + losses[1]))})
    assert rel <= 1e-5, rel
    assert abs(L - 0.5 * (losses[0] + losses[1])) <= 1e-5 * max(1.0, abs(L)), (L, losses)


def penalty_pulls_gradient_norms_to_one(variant, out_act, report, key):
    """30 D steps on one batch with the penalty's target K = 1: the mean |norm - 1| over the live x_hat rows falls"""
    import gm_b200
    n = 16
    eng, G, D, imgs, z, rnd = critic_setup(variant, out_act, n=n)
    x, zc = eng.stage_images(imgs.cuda()), z.cuda()
    rnd = dict(zip(("eps",) if variant == "wgp" else ("delta", "u"), (t.cuda() for t in rnd)))
    hp = gm_b200.AdamHP.make(1e-4)
    dev = []
    for _ in range(30):
        eng.d_grad(x, n, noise=zc, **rnd)
        nm = eng.gp_norms_
        if variant == "wgp":
            nm = nm[nm > 0]
        dev.append(float((nm - 1).abs().mean()))
        eng.apply(1, hp)
    report.add(key, {"first": dev[0], "last": dev[-1]})
    assert all(np.isfinite(dev)) and dev[-1] < dev[0], dev
