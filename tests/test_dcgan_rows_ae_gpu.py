"""MMGAN, WGAN, LSGAN, f-GAN and the autoencoder on the DCGAN conv path, on the GPU: one seeded D and G step of every row
variant against fp32 autograd of the torch oracle (tests/dcgan_rows_oracle.py), gm_loss_rows_c's constants, WGAN's clamp in
the D Adam kernel, the f-GAN method switch, the autoencoder's latent kernels (gm_ae_latent_rows, gm_ae_dlatent_rows) against
float64, ae_grad against the oracle (tests/dcgan_ae_oracle.py), and every new drop-in on the reference's driver lines.  With
GM_PARITY_DIR set, the measured errors are written to $GM_PARITY_DIR/parity_dcgan_rows_ae.json."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

import dcgan_ae_oracle as AO
import dcgan_harness as H
import dcgan_rows_oracle as RO
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_rows_ae")
BF = 2.0 ** -8


def _lib():
    from gm_b200 import _lib
    return _lib, _lib.ctx()


# ------------------------------------------------------------------ the row losses
_STEPS = [(v, (0.0, 1.0, 1.0)) for v in RO.ROW_VARIANTS] + [("ls", (-1.0, 1.0, 0.0))]


@pytest.mark.parametrize("variant,abc", _STEPS, ids=["%s-%g,%g,%g" % ((v,) + abc) for v, abc in _STEPS])
def test_row_variant_steps_match_the_torch_oracle(variant, abc):
    """d_grad + g_grad at hidden 16, batch 8 against fp32 autograd, with the bounds of
    test_dcgan_gpu.py::test_dcgan_train_step_matches_the_torch_oracle (the losses relative to max(|L|, 0.5): W's and
    f-GAN's losses are differences of means that can sit near 0, and 0.5 is the scale of the sigmoid scores they difference)"""
    a, b, c = abc
    eng, G, D, g = H.setup()
    eng.variant = variant
    eng.ls_a, eng.ls_b, eng.ls_c = abc
    n = 8
    imgs = torch.rand(n, 3 * 64 * 64, generator=g)
    z1, z2 = torch.randn(n, 100, generator=g), torch.randn(n, 100, generator=g)
    rep = {}
    Ld_ref = RO.d_loss(G, D, imgs, z1, variant, a, b)
    gd = torch.autograd.grad(Ld_ref, list(D.parameters()))
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z1.cuda()).item()
    rep["D_loss"] = abs(Ld - Ld_ref.item()) / max(abs(Ld_ref.item()), 0.5)
    got = eng.torch_grads()
    for (name, _), gref in zip(D.named_parameters(), gd):
        rep["gradD_" + name] = nrel(got["D." + name], gref)
    Lg_ref = RO.g_loss(G, D, z2, variant, c)
    gg = torch.autograd.grad(Lg_ref, list(G.parameters()))
    Lg = eng.g_grad(n, noise=z2.cuda()).item()
    rep["G_loss"] = abs(Lg - Lg_ref.item()) / max(abs(Lg_ref.item()), 0.5)
    got = eng.torch_grads()
    for (name, _), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(got["G." + name], gref)
    _REPORT.add("step_%s_%g_%g_%g" % ((variant,) + abc), rep)
    assert rep["D_loss"] < 5e-3 and rep["G_loss"] < 1e-2, rep
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.12, (k, v, rep)


@pytest.mark.parametrize("variant", ["ns", "ls", "w", "f_pearson"])
def test_loss_rows_c_null_is_gm_loss_rows_and_ls_targets_apply(variant):
    """gm_loss_rows_c(NULL) gives gm_loss_rows' bits; with the defaults spelled out too; with LS targets (a, b, c) the rows are
    0.5 (d - t)^2 / n and (d - t) d (1 - d) / n"""
    from gm_b200._lib import VARIANTS, LossConsts
    L, h = _lib()
    n = 300
    g = torch.Generator(device="cuda").manual_seed(4)
    logits = 2 * torch.randn(2 * n, device="cuda", generator=g)
    outs = []
    for lc in ("old", None, LossConsts(10.0, 1.0, 1.0, 0.0, 1.0, 1.0)):
        for g_step in (0, 1):
            ds = torch.full((2 * n,), 7.0, device="cuda")
            loss = torch.zeros(4, device="cuda")
            rows = logits[:n] if g_step else logits
            if lc == "old":
                rc = L.lib().gm_loss_rows(h, VARIANTS[variant], 0, L._ptr(rows), n, g_step, 1.0 / n, L._ptr(ds), None, L._ptr(loss), L._stream())
            else:
                rc = L.lib().gm_loss_rows_c(h, VARIANTS[variant], 0, L._ptr(rows), n, g_step, 1.0 / n, None if lc is None else C.byref(lc),
                                            L._ptr(ds), None, L._ptr(loss), L._stream())
            L.check(h, rc)
            outs.append((ds.clone(), loss[:2].clone()))
    for k in range(2, 6):
        assert torch.equal(outs[k][0], outs[k % 2][0]) and torch.equal(outs[k][1], outs[k % 2][1]), k
    if variant != "ls":
        return
    a, b, c = -1.0, 0.5, 0.25
    lc = LossConsts(10.0, 1.0, 1.0, a, b, c)
    d = torch.sigmoid(logits.double())
    for g_step, tgt in ((0, torch.cat([torch.full((n,), b), torch.full((n,), a)]).double().cuda()), (1, torch.full((n,), c).double().cuda())):
        m = n if g_step else 2 * n
        ds = torch.zeros(2 * n, device="cuda")
        loss = torch.zeros(4, device="cuda")
        L.check(h, L.lib().gm_loss_rows_c(h, VARIANTS["ls"], 0, L._ptr(logits), n, g_step, 1.0 / n, C.byref(lc), L._ptr(ds), None, L._ptr(loss),
                                          L._stream()))
        dd, tt = d[:m], tgt[:m]
        want_loss = float(0.5 * ((dd - tt) ** 2).sum() / n)
        want_ds = (dd - tt) * dd * (1 - dd) / n
        assert abs(float(loss[0]) - want_loss) <= 1e-5 * abs(want_loss)
        assert float((ds[:m].double() - want_ds).abs().max()) <= 1e-5 * float(want_ds.abs().max())


# ------------------------------------------------------------------ WGAN's clamp
def _loader(n=64, bs=16, seed=0):
    """k / 255 images (ToTensor's values): few enough distinct bf16 values for device_dataset's 8-bit pool"""
    g = torch.Generator().manual_seed(seed)
    imgs = torch.randint(0, 256, (n, 3, 64, 64), generator=g).float() / 255
    return imgs, torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(n)), batch_size=bs, shuffle=True)


def test_wgan_adam_clamp_is_torch_adam_then_clamp():
    """one D step: the engine's Adam with clamp = torch.optim.Adam.step() then clamp_ on the same gradients, every D parameter
    (BatchNorm's included) in [-clip, clip]"""
    import gm_b200
    eng, _, _, g = H.setup("w")
    clip, lr = 0.03, 5e-3
    imgs = torch.rand(8, 3 * 4096, generator=g)
    eng.d_grad(eng.stage_images(imgs.cuda()), 8, noise=torch.randn(8, 100, generator=g).cuda())
    p0, g0 = eng.D.params.clone(), eng.D.grads.clone()
    eng.apply(1, gm_b200.AdamHP.make(lr, clamp=clip))
    p = p0.clone().requires_grad_(True)
    opt = torch.optim.Adam([p], lr=lr)
    p.grad = g0.clone()
    opt.step()
    with torch.no_grad():
        p.clamp_(-clip, clip)
    err = float((eng.D.params - p.detach()).abs().max())
    _REPORT.add("wgan_clamp_step", {"abs_max": err, "clamped_share": float((p.detach().abs() == clip).float().mean())})
    assert err <= 1e-6, err
    assert float(eng.D.params.abs().max()) <= clip
    assert float((p.detach().abs() == clip).float().mean()) > 0.1                   # the clamp is active on many weights


def test_dc_w_gan_train_and_the_overridden_loop_clamp_every_d_parameter():
    import dc_w_gan as M
    _, loader = _loader()
    torch.manual_seed(1)
    model = M.DCWGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    tr = M.DCWGANTrainer(model, loader, loader, loader)
    tr.train(num_epochs=1, G_lr=5e-5, D_lr=5e-5, D_steps=5, clip=0.01)
    assert all(float(p.abs().max()) <= 0.01 for p in model.D.parameters())
    assert float(model.D.bn2.weight.abs().max()) == pytest.approx(0.01)           # BatchNorm's scale starts near 1: clamped

    class Hinge(M.DCWGANTrainer):
        def train_D(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            return torch.mean(torch.relu(1 + self.model.D(self.model.G(noise).detach()))) + torch.mean(torch.relu(1 - self.model.D(images)))

    torch.manual_seed(2)
    model = M.DCWGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    tr = Hinge(model, loader, loader, loader)
    tr.train(num_epochs=1, G_lr=5e-5, D_lr=5e-5, D_steps=1, clip=0.02)
    assert len(tr.Dlosses) == 4 and all(np.isfinite(tr.Dlosses))
    assert all(float(p.abs().max()) <= 0.02 for p in model.D.parameters())
    assert float(model.D.bn3.weight.abs().max()) == pytest.approx(0.02)


# ------------------------------------------------------------------ the f-GAN method switch
def test_f_gan_method_switch_keeps_weights_and_running_statistics():
    import dc_f_gan as M
    imgs, loader = _loader()
    torch.manual_seed(4)
    model = M.DCfGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    tr = M.DCfGANTrainer(model, loader, loader, loader)
    tr.train(num_epochs=1, method="jensen_shannon")
    old = tr._engine
    sd = {k: v.clone() for k, v in model.state_dict().items()}
    assert float(sd["D.bn2.running_var"].sub(1).abs().max()) > 1e-3                  # the statistics moved away from their init
    tr.train(num_epochs=0, method="pearson")
    assert tr._engine is not old and tr._engine.variant == "f_pearson" and tr.variant == "f_pearson"
    for k, v in model.state_dict().items():
        assert torch.equal(v, sd[k]), k
    tw = tr._engine.torch_weights()
    assert all(torch.equal(tw[k], sd[k]) for k in tw)
    assert torch.equal(tr._engine.run_D[2][1].cpu(), sd["D.bn3.running_var"]) and torch.equal(tr._engine.run_G[0][0].cpu(), sd["G.bn1.running_mean"])
    # the loss changed with the method: the same weights, images and noise under the old divergence and the new one
    import gm_b200
    js = gm_b200.DcganEngine(hidden_dim=16, z_dim=100, variant="f_jensen_shannon")
    js.load_torch_weights(tw)
    z = torch.randn(8, 100).cuda()
    L_js = js.d_grad(js.stage_images(imgs[:8].reshape(8, -1).cuda()), 8, noise=z).item()
    L_p = tr._engine.d_grad(tr._engine.stage_images(imgs[:8].reshape(8, -1).cuda()), 8, noise=z).item()
    s = tr._engine.scores_.double().cpu()
    dx, dg = torch.sigmoid(s[:8]), torch.sigmoid(s[8:])
    assert L_p == pytest.approx(float(RO.d_rows("f_pearson", dx, dg)), rel=1e-4)
    assert L_js == pytest.approx(float(RO.d_rows("f_jensen_shannon", dx, dg)), rel=1e-4)
    assert abs(L_p - L_js) > 1e-2


# ------------------------------------------------------------------ the autoencoder's latent kernels
def _padded(rows, ld, dtype, fill):
    """a [rows + 2, ld] buffer of fill: the kernel's block is rows [1, rows + 1), rows 0 and rows + 1 must stay untouched"""
    return torch.full((rows + 2, ld), fill, device="cuda", dtype=dtype)


@pytest.mark.parametrize("n,z,ldm", [(37, 20, 48), (5, 32, 32), (300, 7, 9)])
def test_ae_latent_rows_match_float64(n, z, ldm):
    L, h = _lib()
    ldz = (z + 1 + 7) // 8 * 8
    g = torch.Generator(device="cuda").manual_seed(n)
    hb = _padded(n, ldm, torch.float32, float("nan"))
    hb[1:n + 1, :z] = torch.randn(n, z, device="cuda", generator=g)
    hb[1, :z:3] = 0.0                                                                  # codes exactly 0 from h == 0
    out = _padded(n, ldz, torch.bfloat16, float("nan"))
    L.check(h, L.lib().gm_ae_latent_rows(h, L._ptr(hb[1:]), ldm, L._ptr(out[1:]), ldz, n, z, L._stream()))
    ref = torch.relu(hb[1:n + 1, :z].double())
    got = out[1:n + 1].double()
    assert float(((got[:, :z] - ref).abs() / ref.abs().clamp_min(1e-30)).max()) <= BF
    assert bool((got[:, :z][ref == 0] == 0).all())
    assert bool((got[:, z] == 1).all()) and bool((got[:, z + 1:] == 0).all())
    assert bool(out[0].isnan().all()) and bool(out[n + 1].isnan().all())


@pytest.mark.parametrize("n,z,ld", [(37, 20, 32), (5, 32, 32), (300, 7, 16)])
def test_ae_dlatent_rows_match_float64(n, z, ld):
    L, h = _lib()
    g = torch.Generator(device="cuda").manual_seed(n + 1)
    hb = _padded(n, z + 3, torch.float32, float("nan"))
    hb[1:n + 1, :z] = torch.randn(n, z, device="cuda", generator=g)
    hb[1, :z:2] = 0.0
    dz = _padded(n, z + 5, torch.float32, float("nan"))
    dz[1:n + 1, :z] = 3 * torch.randn(n, z, device="cuda", generator=g)
    out = _padded(n, ld, torch.bfloat16, float("nan"))
    L.check(h, L.lib().gm_ae_dlatent_rows(h, L._ptr(hb[1:]), z + 3, L._ptr(dz[1:]), z + 5, L._ptr(out[1:]), ld, n, z, L._stream()))
    hh, dd = hb[1:n + 1, :z].double(), dz[1:n + 1, :z].double()
    ref = AO.dlatent(hh, dd)
    hg = hh.clone().requires_grad_(True)
    assert torch.equal(ref, torch.autograd.grad(torch.relu(hg), hg, dd)[0])          # torch's relu backward, 0 at h == 0
    got = out[1:n + 1].double()
    assert float(((got[:, :z] - ref).abs() / ref.abs().clamp_min(1e-30)).max()) <= BF
    assert bool((got[:, :z][hh <= 0] == 0).all()) and bool((got[:, z:] == 0).all())
    assert bool(out[0].isnan().all()) and bool(out[n + 1].isnan().all())


def test_ae_latent_kernels_refuse_bad_arguments_before_any_launch():
    from gm_b200 import launch_count
    L, h = _lib()
    n, z = 4, 20
    hb = torch.zeros(n, 32, device="cuda")
    zr = torch.zeros(n, 24, device="cuda", dtype=torch.bfloat16)
    dz = torch.zeros(n, z, device="cuda")
    lat, dlat = L.lib().gm_ae_latent_rows, L.lib().gm_ae_dlatent_rows
    P, s = L._ptr, L._stream()
    odd = C.c_void_p(zr.data_ptr() + 2)
    f_odd = C.c_void_p(hb.data_ptr() + 2)
    bad_lat = [(P(hb), 32, P(zr), 21, n, z), (P(hb), 32, P(zr), 24, n, 24), (P(hb), 19, P(zr), 24, n, z), (P(hb), 32, odd, 24, n, z),
               (f_odd, 32, P(zr), 24, n, z), (None, 32, P(zr), 24, n, z), (P(hb), 32, P(zr), 24, 0, z), (P(hb), 32, P(zr), 24, n, 0)]
    bad_dlat = [(P(hb), 32, P(dz), z, P(zr), 12, n, z), (P(hb), 32, P(dz), z, P(zr), 20, n, z), (P(hb), 19, P(dz), z, P(zr), 24, n, z),
                (P(hb), 32, P(dz), 19, P(zr), 24, n, z), (P(hb), 32, P(dz), z, odd, 24, n, z), (f_odd, 32, P(dz), z, P(zr), 24, n, z),
                (P(hb), 32, None, z, P(zr), 24, n, z), (P(hb), 32, P(dz), z, P(zr), 24, -1, z)]
    torch.cuda.synchronize()
    before = launch_count()
    for args in bad_lat:
        assert lat(h, *args, s) != 0, args
        assert b"gm_ae_latent_rows" in L.lib().gm_last_error(h)
    for args in bad_dlat:
        assert dlat(h, *args, s) != 0, args
        assert b"gm_ae_dlatent_rows" in L.lib().gm_last_error(h)
    # 2^28 rows x 64 columns = 2^31 threads: refused as unsupported (the int grid would overflow), nothing launched
    assert lat(h, P(hb), 32, P(zr), 64, 1 << 28, z, s) != 0 and b"2^31" in L.lib().gm_last_error(h)
    assert dlat(h, P(hb), 32, P(dz), z, P(zr), 64, 1 << 28, z, s) != 0 and b"2^31" in L.lib().gm_last_error(h)
    assert launch_count() == before
    assert bool((zr == 0).all())


# ------------------------------------------------------------------ ae_grad, descent, eval mode, data-parallel sums
def _ae_engine(hd=16, z=32, wstd=0.05, seed=11):
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant="ae")
    g = torch.Generator().manual_seed(seed)
    for net in eng.nets():
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.zero_padding()
    for net in eng.nets():
        net.refresh()
    E, G = AO.Encoder(hd, z), AO.Decoder(hd, z)
    AO.load_from_engine_weights(E, G, eng.torch_weights())
    for m in (E, G):
        m.train()
        m.q = staticmethod(O.bf16_points)
    return eng, E, G, g


@pytest.mark.parametrize("z", [32, 30])
def test_ae_grad_matches_the_oracle(z):
    """z = 30: the fp32 dL/dz rows and G's l1 weight-gradient rows start 120 bytes apart; bounds of the VAE's comparison"""
    n = 8
    eng, E, G, g = _ae_engine(z=z)
    x = (torch.rand(n, 3 * 4096, generator=g) < 0.3).float()
    loss_ref = AO.compute_batch(E, G, x)
    params = list(E.parameters()) + list(G.parameters())
    ref = torch.autograd.grad(loss_ref, params)
    loss = eng.ae_grad(eng.stage_images(x.cuda()), n).item()
    rep = {"recon": abs(loss - loss_ref.item()) / loss_ref.item()}
    tg = eng.torch_grads()
    names = ["D." + k for k, _ in E.named_parameters()] + ["G." + k for k, _ in G.named_parameters()]
    for name, r in zip(names, ref):
        rep["grad_" + name] = nrel(tg[name], r)
    code = eng.ae_saved_["zrows"][:, :z].float().cpu()
    rep["zero_codes"] = float((code == 0).float().mean())
    _REPORT.add("ae_step_z%d" % z, rep)
    assert 0.1 < rep["zero_codes"] < 0.9, rep                                     # the ReLU's both sides are in play
    if z < eng.mp:
        assert float(eng.D.view("l5.weight", eng.D.grads)[z:].abs().max()) == 0.0  # the head's padded rows
    assert rep["recon"] < 5e-3, rep
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.20, (k, v, rep)


def test_ae_steps_lower_the_loss_and_half_batches_sum_to_the_full_batch():
    import gm_b200
    n = 8
    eng, _, _, g = _ae_engine()
    x = eng.stage_images((torch.rand(n, 3 * 4096, generator=g) < 0.3).float().cuda())
    # a batch of two identical halves has the halves' BatchNorm statistics: its gradient is the sum of theirs (the losses
    # are sums, so data-parallel ranks add gradients without rescaling)
    l_half = eng.ae_grad(x, n).item()
    half = torch.cat([eng.G.grads, eng.D.grads]).clone()
    l_full = eng.ae_grad(torch.cat([x, x]), 2 * n).item()
    full = torch.cat([eng.G.grads, eng.D.grads])
    rel = nrel(full, 2 * half)
    _REPORT.add("ae_halves", {"grad_nrel": rel, "loss_rel": abs(l_full - 2 * l_half) / l_full})
    assert rel <= 1e-4 and abs(l_full - 2 * l_half) <= 1e-5 * l_full, (rel, l_full, l_half)
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    losses = []
    for _ in range(15):
        losses.append(eng.ae_grad(x, n).item())
        eng.apply(hp)
    assert all(np.isfinite(losses)) and losses[-1] < 0.97 * losses[0], losses


def test_ae_forward_batchnorm_modes():
    """train=True takes batch statistics and moves the running ones; train=False normalises with them and leaves them"""
    n = 8
    eng, E, G, g = _ae_engine()
    x = (torch.rand(n, 3 * 4096, generator=g) < 0.3).float()
    rows = eng.stage_images(x.cuda())
    for _ in range(3):
        eng.ae_forward(rows, n, train=True)
    runs = [r.clone() for r in list(eng.run_D.values()) + list(eng.run_G.values())]
    rec_e, code_e, loss_e = eng.ae_forward(rows, n, train=False)
    assert torch.equal(code_e, eng.encode(x.cuda(), train=False))
    assert all(torch.equal(a, b) for a, b in zip(runs, list(eng.run_D.values()) + list(eng.run_G.values())))
    with torch.no_grad():
        for i, r in eng.run_D.items():
            bn = getattr(E, "bn%d" % (i + 1))
            bn.running_mean.copy_(r[0].cpu()); bn.running_var.copy_(r[1].cpu())
        for i, r in eng.run_G.items():
            bn = getattr(G, "bn%d" % (i + 1))
            bn.running_mean.copy_(r[0].cpu()); bn.running_var.copy_(r[1].cpu())
        E.eval(); G.eval()
        ref = G(E(x))
    rec_t, _, _ = eng.ae_forward(rows, n, train=True)
    rep = {"eval_rec": nrel(rec_e, ref), "train_vs_eval": nrel(rec_t, rec_e),
           "eval_loss": abs(float(loss_e[0]) - float(((x - ref) ** 2).sum())) / float(((x - ref) ** 2).sum())}
    _REPORT.add("ae_bn_modes", rep)
    assert rep["eval_rec"] < 1e-2 and rep["eval_loss"] < 1e-2 and rep["train_vs_eval"] > 10 * rep["eval_rec"], rep


# ------------------------------------------------------------------ the drop-ins on the reference's driver lines
_GAN_DROPINS = {"mm": ("dc_mm_gan", "DCMMGAN", "DCMMGANTrainer", dict(G_lr=2e-4, D_lr=2e-4, D_steps=1, G_init=5)),
                "w": ("dc_w_gan", "DCWGAN", "DCWGANTrainer", dict(G_lr=5e-5, D_lr=5e-5, D_steps=5, clip=0.01)),
                "ls": ("dc_ls_gan", "DCLSGAN", "DCLSGANTrainer", dict(G_lr=1e-4, D_lr=1e-4, D_steps=1)),
                "f": ("dc_f_gan", "DCfGAN", "DCfGANTrainer", dict(method="jensen_shannon", G_lr=1e-4, D_lr=1e-4, D_steps=1))}


@pytest.mark.parametrize("device_dataset", [False, True], ids=["host", "pool"])
@pytest.mark.parametrize("which", sorted(_GAN_DROPINS))
def test_gan_dropins_run_the_reference_driver_lines(which, device_dataset, capsys):
    """train() with the reference's __main__ arguments, losses logged per outer step, generate_images, the discriminator's
    sigmoid scores, a save_model / load_model round trip, and train_D / train_G whose .backward() delivers gradients"""
    import importlib
    modname, model_name, trainer_name, args = _GAN_DROPINS[which]
    M = importlib.import_module(modname)
    imgs, loader = _loader()
    torch.manual_seed(3)
    model = getattr(M, model_name)(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    tr = getattr(M, trainer_name)(model, loader, loader, loader, viz=False)
    tr.device_dataset = device_dataset
    tr.train(num_epochs=2, **args)
    assert (getattr(tr, "_pool", None) is not None) == device_dataset
    steps = int(np.ceil(len(loader) / args["D_steps"]))
    assert len(tr.Dlosses) == 2 * steps and len(tr.Glosses) == 2 * steps
    assert all(np.isfinite(tr.Dlosses)) and all(np.isfinite(tr.Glosses))
    out = capsys.readouterr().out
    assert out.count("Epoch[") == 2 and (which != "mm" or "G pre-trained for 5 training steps." in out)
    after = model.state_dict()
    assert all(not torch.equal(before[k], after[k]) for k in before if k.startswith("D.l") and k.endswith("weight"))
    assert any(not torch.equal(before[k], after[k]) for k in before if k.startswith("G.") and k.endswith("weight"))
    if which == "w":
        assert all(float(p.abs().max()) <= 0.01 for p in model.D.parameters())
    gen = tr.generate_images(0, num_outputs=4)
    assert gen.shape == (4, 3, 64, 64) and float(gen.min()) >= 0 and float(gen.max()) <= 1
    d = model.D(imgs[:8])
    assert d.shape == (8, 1) and float(d.min()) > 0 and float(d.max()) < 1
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        tr.save_model(path)
        model2 = getattr(M, model_name)(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
        tr2 = getattr(M, trainer_name)(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        zz = torch.randn(4, 100)
        assert nrel(model2.G(zz), model.G(zz)) < 1e-6
    model.D.zero_grad()
    loss = tr.train_D(imgs[:16].reshape(16, -1)) if which != "ls" else tr.train_D(imgs[:16].reshape(16, -1), a=-1, b=1)
    loss.backward()
    assert model.D.l4.weight.grad is not None and float(model.D.l4.weight.grad.abs().sum()) > 0
    gl = tr.train_G(imgs[:16]) if which != "ls" else tr.train_G(imgs[:16], c=0)
    gl.backward()
    assert np.isfinite(float(gl)) and float(model.G.l2.weight.grad.abs().sum()) > 0


def test_ls_targets_reach_train_d_train_g_and_the_fused_loop():
    """train_D(a, b) / train_G(c) and loss_consts give the losses the torch expressions give on the same scores"""
    import dc_ls_gan as M
    from gm_b200 import GmError
    imgs, loader = _loader()
    torch.manual_seed(5)
    model = M.DCLSGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    tr = M.DCLSGANTrainer(model, loader, loader, loader)
    eng = tr._engine_synced()
    x = imgs[:8].reshape(8, -1).cuda()
    z = torch.randn(8, 100).cuda()
    tr.compute_noise = lambda n, zd: z[:n]
    for a, b, c in ((0.0, 1.0, 1.0), (-1.0, 1.0, 0.0)):
        Ld = float(tr.train_D(x, a=a, b=b))
        s = eng.scores_.double()
        dx, dg = torch.sigmoid(s[:8]), torch.sigmoid(s[8:])
        assert Ld == pytest.approx(float(0.5 * ((dx - b) ** 2).mean() + 0.5 * ((dg - a) ** 2).mean()), rel=1e-5)
        Lg = float(tr.train_G(x, c=c))
        assert eng.ls_c == c and np.isfinite(Lg)                                   # train_G(c) sets c; a and b are train_D's
    tr.loss_consts = dict(ls_a=-1.0, ls_b=1.0, ls_c=0.0)
    tr.train(num_epochs=1)
    assert (eng.ls_a, eng.ls_b, eng.ls_c) == (-1.0, 1.0, 0.0)
    tr.loss_consts = dict(ls_x=1.0)
    with pytest.raises(GmError):
        tr.train(num_epochs=1)


@pytest.mark.parametrize("which", ["mm", "ls", "f"])
def test_gan_dropin_overrides_train_through_the_conv_nodes(which):
    """a subclass's own train_D / train_G (the reference loop, FusedAdam) trains model.G / model.D through the conv nodes"""
    import importlib
    modname, model_name, trainer_name, args = _GAN_DROPINS[which]
    M = importlib.import_module(modname)
    _, loader = _loader()

    class Custom(getattr(M, trainer_name)):
        def train_D(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            return -torch.mean(torch.log(self.model.D(images) + 1e-8) + torch.log(1 - self.model.D(self.model.G(noise)) + 1e-8))

        def train_G(self, images):
            noise = self.compute_noise(images.shape[0], self.model.z_dim)
            return -torch.mean(torch.log(self.model.D(self.model.G(noise)) + 1e-8))

    torch.manual_seed(6)
    model = getattr(M, model_name)(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    tr = Custom(model, loader, loader, loader)
    tr.train(num_epochs=1, **args)
    assert len(tr.Dlosses) == 4 and all(np.isfinite(tr.Dlosses)) and all(np.isfinite(tr.Glosses))
    after = model.state_dict()
    assert all(not torch.equal(before[k], after[k].cpu()) for k in before if k.endswith("weight") and ".l" in k)


@pytest.mark.parametrize("device_dataset", [False, True], ids=["host", "pool"])
def test_dc_ae_runs_the_reference_driver_lines(device_dataset, capsys):
    """src/ae.py's __main__ on the conv autoencoder: train() with early stopping, the epoch line, the reconstruction, the
    encoder / decoder calls, compute_batch's backward and a save_model / load_model round trip in eval mode"""
    import dc_ae
    imgs, loader = _loader()
    torch.manual_seed(7)
    model = dc_ae.DCAutoencoder(image_size=64 * 64 * 3, hidden_dim=16, z_dim=32)
    tr = dc_ae.DCAutoencoderTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    tr.device_dataset = device_dataset
    tr.train(num_epochs=3, lr=1e-3, weight_decay=1e-5)
    assert (getattr(tr, "_pool", None) is not None) == device_dataset
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("Epoch[")]
    assert len(lines) == 3 and lines[0].startswith("Epoch[1/3], Train Loss: ") and ", Val Loss: " in lines[0]
    assert len(tr.recon_loss) == 3 * len(loader) and tr.recon_loss[-1] < tr.recon_loss[0]
    assert tr.best_val_loss < 1e10 and isinstance(tr.best_model, dc_ae.DCAutoencoder)
    model.eval()
    rec = tr.reconstruct_images(imgs[:4], 0)
    assert rec.shape == (4, 3, 64, 64) and float(rec.min()) >= 0 and float(rec.max()) <= 1
    code = model.encoder(imgs[:4].reshape(4, -1))
    assert code.shape == (4, 32) and float(code.min()) == 0.0
    assert model.decoder(code).shape == (4, 3 * 4096)
    assert nrel(tr.best_model(imgs[:4].reshape(4, -1)), tr.best_model(imgs[:4].reshape(4, -1))) == 0.0
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "ae.ckpt")
        tr.save_model(path)
        model2 = dc_ae.DCAutoencoder(image_size=64 * 64 * 3, hidden_dim=16, z_dim=32)
        tr2 = dc_ae.DCAutoencoderTrainer(model2, loader, loader, loader)
        tr2.load_model(path)
        model2.eval()
        assert list(model2.state_dict()) == list(model.state_dict())
        x = imgs[:4].reshape(4, -1)
        assert nrel(model2(x), model(x)) < 1e-6
    model.train()
    model.zero_grad()
    loss = tr.compute_batch((imgs[:16], torch.zeros(16)))
    loss.backward()
    assert float(model.encoder.l4.weight.grad.abs().sum()) > 0 and float(model.decoder.l2.weight.grad.abs().sum()) > 0
