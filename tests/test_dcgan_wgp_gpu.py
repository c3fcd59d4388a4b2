"""WGAN-GP on the DCGAN conv path on the GPU: the new kernels against torch (interpolation, masked im2col, penalty), one
critic step against autograd's double backward and against the closed-form oracle at the CUDA path's bf16 storage points
(tests/dcgan_wgp_oracle.py), the generator step, the data-parallel split, and the dc_w_gp_gan drop-in on the reference's
driver lines.  With GM_PARITY_DIR set, the measured errors are written to $GM_PARITY_DIR/parity_dcgan_wgp.json."""
import json
import os

import numpy as np
import pytest
import torch

import dcgan_wgp_oracle as W

pytestmark = pytest.mark.gpu
_REPORT = {}


def _nrel(a, b):
    a, b = a.detach().double().reshape(-1).cpu(), b.detach().double().reshape(-1).cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _dump():
    out = os.environ.get("GM_PARITY_DIR")
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "parity_dcgan_wgp.json"), "w") as f:
        json.dump(_REPORT, f, indent=1, sort_keys=True)


def _ctx():
    import gm_b200
    from gm_b200 import _lib
    return gm_b200, _lib, _lib.ctx()


def test_interpolation_is_bit_exact_and_philox_is_keyed():
    gm_b200, L, h = _ctx()
    n, C = 5, 3
    g = torch.Generator(device="cuda").manual_seed(1)
    xr = torch.rand(n * 4096, C, device="cuda", generator=g).to(torch.bfloat16)
    xf = torch.rand(n * 4096, C, device="cuda", generator=g).to(torch.bfloat16)
    eps = torch.rand(n, device="cuda", generator=g)
    out = torch.empty_like(xr)
    eo = torch.zeros(n, device="cuda")
    L.check(h, L.lib().gm_gp_interp_rows(h, L._ptr(xr), C, L._ptr(xf), C, n, 4096, C, L._ptr(eps), L._ptr(eo), 0, 0, L._ptr(out), C,
                                         L._stream()))
    e = eps.repeat_interleave(4096).view(-1, 1)
    want = (e * xr.float() + (1 - e) * xf.float()).to(torch.bfloat16)
    assert torch.equal(out, want) and torch.equal(eo, eps)
    draws = []
    for seed, sid in ((7, 2), (7, 2), (7, 4), (8, 2)):
        L.check(h, L.lib().gm_gp_interp_rows(h, L._ptr(xr), C, L._ptr(xf), C, n, 4096, C, None, L._ptr(eo), seed, sid, L._ptr(out), C,
                                             L._stream()))
        draws.append(eo.clone())
        e = eo.repeat_interleave(4096).view(-1, 1)
        assert torch.equal(out, (e * xr.float() + (1 - e) * xf.float()).to(torch.bfloat16))
    assert torch.equal(draws[0], draws[1]) and not torch.equal(draws[0], draws[2]) and not torch.equal(draws[0], draws[3])
    assert float(draws[0].min()) > 0 and float(draws[0].max()) <= 1 and len(set(draws[0].tolist())) == n


@pytest.mark.parametrize("H,W,Cc", [(8, 8, 16), (12, 20, 24)])
def test_masked_im2col_and_row_mask_are_bit_exact(H, W, Cc):
    from gm_b200 import dcgan as DC
    B = 3
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(B * H * W, Cc, device="cuda", generator=g).to(torch.bfloat16)
    m = torch.randn(B * H * W, Cc, device="cuda", generator=g).to(torch.bfloat16)
    m[::7] = 0                                                        # LeakyReLU'(0) = slope, like torch's leaky_relu
    masked = (x.float() * torch.where(m.float() > 0, 1.0, DC.SLOPE)).to(torch.bfloat16)
    L = (H // 2) * (W // 2)
    col = torch.empty(B * L, 16 * Cc, device="cuda", dtype=torch.bfloat16)
    DC._im2col_lrelu_mask(x, B, H, W, Cc, m, col)
    ref = torch.nn.functional.unfold(masked.float().view(B, H, W, Cc).permute(0, 3, 1, 2), 4, padding=1, stride=2)
    assert torch.equal(col.float(), ref.view(B, Cc, 16, -1).permute(0, 3, 2, 1).reshape(B * L, 16 * Cc))
    out = torch.empty_like(x)
    DC._lrelu_mask(x, m, out)
    assert torch.equal(out, masked)
    DC._lrelu_mask(x, m, m)                                           # in place over the mask source
    assert torch.equal(m, masked)


def test_penalty_kernel_norm_coefficient_seed_and_loss():
    gm_b200, L, h = _ctx()
    n, C, lam, inv = 6, 3, 10.0, 1.0 / 16
    g = torch.Generator(device="cuda").manual_seed(3)
    gi = (torch.randn(n * 4096, C, device="cuda", generator=g) * torch.tensor([0.001, 0.005, 0.01, 0.02, 1.0, 1.0], device="cuda")
          .repeat_interleave(4096).view(-1, 1)).to(torch.bfloat16)
    gi[4 * 4096:5 * 4096] = 0                                          # ||g|| = 0: coefficient 0, loss term 1
    r = torch.full_like(gi, 7.0)
    norms = torch.zeros(n, device="cuda")
    loss = torch.full((2,), 0.25, device="cuda")
    L.check(h, L.lib().gm_gp_penalty(h, L._ptr(gi), C, n, 4096, C, lam, inv, 1.0 / n, L._ptr(r), C, L._ptr(norms), L._ptr(loss),
                                     L._stream()))
    gd = gi.double().view(n, -1)
    nref = gd.norm(dim=1)
    coef = torch.where(nref > 0, 2 * lam * inv * (nref - 1) / nref.clamp_min(1e-30), torch.zeros_like(nref))
    rref = coef.view(n, 1) * gd
    lref = 0.25 + lam * float(((nref - 1) ** 2).mean())
    rep = {"norm": _nrel(norms, nref), "r": _nrel(r.view(n, -1), rref), "loss": abs(float(loss[0]) - lref) / lref}
    _REPORT["penalty_kernel"] = rep
    _dump()
    assert float(norms[4]) == 0.0 and bool((r[4 * 4096:5 * 4096] == 0).all())
    assert rep["norm"] < 1e-6 and rep["loss"] < 1e-6 and rep["r"] < 4e-3, rep        # r: bf16 rounding of the stored seed
    assert float(loss[1]) == 0.25


def _wgp_setup(out_act, hd=16, z=100, n=8, wstd=0.05, seed=11, live="xhat"):
    """engine + oracle G / critic with the same weights; for relu the last layer's sign is chosen so that at least half of
    the x_hat rows (live="xhat") or of the generated rows (live="fake") are live (at a sign that kills them every row
    would compare zero with zero)"""
    import gm_b200
    from oracle import dcgan_torch as O
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant="wgp", d_out_act=out_act)
    g = torch.Generator().manual_seed(seed)
    for net in (eng.G, eng.D):
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.D.view("l5.weight")[1:].zero_()
    eng.G.refresh(); eng.D.refresh()
    G = O.Generator(hd, z)
    D = W.Critic(hd, 3, out_act)
    sd = eng.torch_weights()
    assert not any(k.startswith("D.bn") for k in sd)
    with torch.no_grad():
        for name, p in G.named_parameters():
            p.copy_(sd["G." + name])
    W.load_engine_weights(D, sd)
    G.train()
    imgs = torch.rand(n, 3 * 64 * 64, generator=g)
    zz = torch.randn(n, z, generator=g)
    eps = torch.rand(n, generator=g)
    if out_act == "relu":
        with torch.no_grad():
            fake = G(zz)
            xh = eps.view(n, 1) * imgs + (1 - eps.view(n, 1)) * fake if live == "xhat" else fake
            if int((D.trace(xh)[0] > 0).sum()) < n // 2:
                eng.D.view("l5.weight").neg_(); eng.D.refresh()
                D.l5.weight.neg_()
    return eng, G, D, imgs, zz, eps


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_wgp_d_step_matches_autograd_and_the_closed_form_oracle(out_act):
    from oracle import dcgan_torch as O
    n = 8
    eng, G, D, imgs, z, eps = _wgp_setup(out_act, n=n)
    lam = 10.0
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z.cuda(), gp_lambda=lam, eps=eps.cuda()).item()
    norms = eng.gp_norms_.cpu().double()
    gp = lam * float(((norms - 1) ** 2).mean())
    got = []
    for i in range(5):
        w = eng.D.view("l%d.weight" % (i + 1), eng.D.grads).detach().cpu()
        p = D.layers()[i].weight
        got.append(w[: p.shape[0]].view(p.shape[0], 4, 4, -1).permute(0, 3, 1, 2))
    assert torch.equal(eng.gp_eps_.cpu(), eps)
    # exact: fp32 autograd double backward (generator and critic in fp32)
    with torch.no_grad():
        fake = G(z)
    ex = W.autograd_d_step(D, imgs, fake, eps, lam)
    # closed form at the CUDA path's bf16 storage points
    Gq = O.Generator(D.l1.weight.shape[0], z.shape[1])
    Gq.load_state_dict(G.state_dict())
    Gq.q = staticmethod(O.bf16_points)
    Gq.train()
    with torch.no_grad():
        fake_q = Gq(z)
    cf = W.closed_form_d_step(D, imgs, fake_q, eps, lam, q=W.bf16_points)
    live = int((norms > 0).sum())
    rep = {"live_rows": live, "D_loss": abs(Ld - float(ex["loss"])) / abs(float(ex["loss"])),
           "GP": abs(gp - float(ex["gp"])) / abs(float(ex["gp"])),
           "W_part": abs((Ld - gp) - float(ex["w_part"])) / max(abs(float(ex["w_part"])), 1e-30),
           "norms_vs_exact": _nrel(norms, ex["norms"])}
    for i in range(5):
        rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] = _nrel(got[i], cf["grads"][i])
        rep["gradD_l%d_vs_exact" % (i + 1)] = _nrel(got[i], ex["grads"][i])
        # the gradient is a sum of three parts (real rows, fake rows, penalty) of which the first two nearly cancel: the
        # bf16 rounding of each part shows against the size of the parts, not of their sum
        scale = sum(float(cf["parts"][k][i].norm()) for k in ("real", "fake", "penalty"))
        rep["gradD_l%d_cancellation" % (i + 1)] = scale / float(cf["grads"][i].norm())
        rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] = float((got[i].double() - cf["grads"][i].double()).norm()) / scale
    _REPORT["d_step_" + out_act] = rep
    _dump()
    if out_act == "relu":
        assert live >= n // 2, rep
    assert rep["D_loss"] < 5e-3 and rep["GP"] < 5e-3, rep
    # the W part is a difference of two means of similar size; measured against the scale of its terms
    with torch.no_grad():
        w_scale = float(D(imgs).abs().mean() + D(fake).abs().mean())
    assert abs((Ld - gp) - float(ex["w_part"])) < 5e-3 * w_scale, (rep, w_scale)
    for i in range(5):
        assert rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] < 3e-2, rep
        assert rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] < 5e-2, rep


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_wgp_g_step_matches_the_oracle(out_act):
    from oracle import dcgan_torch as O
    n = 8
    eng, G, D, imgs, z, eps = _wgp_setup(out_act, n=n, live="fake")
    Lg = eng.g_grad(n, noise=z.cuda()).item()
    G.q = staticmethod(O.bf16_points)
    zq = z.clone()
    s, _ = D.trace(G(zq), W.bf16_points)
    loss = -D.out(s).mean()                                             # src/w_gp_gan.py:237
    gg = torch.autograd.grad(loss, list(G.parameters()))
    live = int((s > 0).sum())
    rep = {"live_rows": live, "G_loss": abs(Lg - loss.item()) / abs(loss.item())}
    assert live >= n // 2 or out_act == "none", rep
    for (name, p), gref in zip(G.named_parameters(), gg):
        got = eng.G.view(name, eng.G.grads).detach().cpu()
        if name.startswith("l"):
            got = got.view(4, 4, p.shape[1], p.shape[0]).permute(3, 2, 0, 1)
        rep["gradG_" + name] = _nrel(got, gref)
    _REPORT["g_step_" + out_act] = rep
    _dump()
    assert rep["G_loss"] < 5e-3, rep
    # as in test_dcgan_gpu: the upstream gradient is one number per sample (-1/n), BatchNorm's backward removes that common
    # mode and the bf16 rounding of what is left reads as several percent
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.12, (k, v, rep)


def test_wgp_split_batch_sums_to_the_full_batch():
    """data-parallel contract on one GPU: the critic gradient of 2n images equals the SUM of the two n-image gradients
    computed with inv_global_batch = 1/(2n); the losses are local means"""
    n = 4
    eng, G, D, imgs, z, eps = _wgp_setup("none", n=2 * n)
    fake, _ = eng.g_forward(2 * n, z.cuda())
    fake = fake.clone()
    real = eng.stage_images(imgs.cuda())
    inv = 1.0 / (2 * n)
    e = eps.cuda()
    L = eng.wgp_critic_grad(real, fake, 2 * n, inv, 10.0, e).item()
    full = eng.D.grads.clone()
    parts, losses = [], []
    for k in range(2):
        rows = slice(k * n * 4096, (k + 1) * n * 4096)
        losses.append(eng.wgp_critic_grad(real[rows].clone(), fake[rows].clone(), n, inv, 10.0, e[k * n:(k + 1) * n].clone()).item())
        parts.append(eng.D.grads.clone())
    rel = _nrel(parts[0] + parts[1], full)
    _REPORT["split_batch"] = {"grad_nrel": rel, "loss_abs": abs(L - 0.5 * (losses[0] + losses[1]))}
    _dump()
    assert rel <= 1e-5, rel
    assert abs(L - 0.5 * (losses[0] + losses[1])) <= 1e-5 * max(1.0, abs(L)), (L, losses)


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_the_penalty_pulls_gradient_norms_to_one(out_act):
    import gm_b200
    n = 16
    eng, G, D, imgs, z, eps = _wgp_setup(out_act, n=n)
    x, zc, ec = eng.stage_images(imgs.cuda()), z.cuda(), eps.cuda()
    hp = gm_b200.AdamHP.make(1e-4)
    dev = []
    for _ in range(30):
        eng.d_grad(x, n, noise=zc, eps=ec)
        nm = eng.gp_norms_
        dev.append(float((nm[nm > 0] - 1).abs().mean()))
        eng.apply(1, hp)
    _REPORT["penalty_descent_" + out_act] = {"first": dev[0], "last": dev[-1]}
    _dump()
    assert all(np.isfinite(dev)) and dev[-1] < dev[0], dev


def test_dc_w_gp_gan_runs_the_reference_driver_code():
    """src/w_gp_gan.py's __main__ lines on the conv model at hidden 16 and 64x64x3 synthetic images"""
    import tempfile
    import dc_w_gp_gan
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(64, 3, 64, 64, generator=g)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(64)), batch_size=16, shuffle=True)
    torch.manual_seed(3)
    model = dc_w_gp_gan.DCWGPGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    trainer = dc_w_gp_gan.DCWGPGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=2, G_lr=1e-4, D_lr=1e-4, D_steps=1)
    assert len(trainer.Dlosses) == 8 and len(trainer.Glosses) == 8
    assert all(np.isfinite(trainer.Dlosses)) and all(np.isfinite(trainer.Glosses))
    after = model.state_dict()
    assert all(not torch.equal(before[k], after[k]) for k in before if k.startswith("D.") and k.endswith("weight"))
    assert any(not torch.equal(before[k], after[k]) for k in before if k.startswith("G.") and k.endswith("weight"))
    out = trainer.generate_images(0, num_outputs=4)
    assert out.shape == (4, 3, 64, 64)
    d = model.D(imgs[:8])
    assert d.shape == (8, 1) and float(d.min()) >= 0                  # relu output
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "dcwgpgan.ckpt")
        trainer.save_model(path)
        model2 = dc_w_gp_gan.DCWGPGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
        tr2 = dc_w_gp_gan.DCWGPGANTrainer(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        assert not any(k.startswith("D.bn") for k in model2.state_dict())
        zz = torch.randn(4, 100)
        assert _nrel(model2.G(zz), model.G(zz)) < 1e-6
        assert _nrel(model2.D(imgs[:4]), model.D(imgs[:4])) < 1e-6
    # the reference's loop body: D_loss.backward() delivers torch-layout gradients
    model.D.zero_grad()
    loss = trainer.train_D(imgs[:16].reshape(16, -1), LAMBDA=10)
    loss.backward()
    assert model.D.l4.weight.grad is not None and float(model.D.l4.weight.grad.abs().sum()) > 0
    gl = trainer.train_G(imgs[:16])
    gl.backward()
    assert np.isfinite(float(gl))
