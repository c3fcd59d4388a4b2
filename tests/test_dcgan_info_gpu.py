"""InfoGAN on the DCGAN conv path on the GPU: the on-device code sampler (gm_info_noise_rows) and the MI loss on Q's rows
(gm_info_loss_rows) against torch, one D, G and MI step against fp32 autograd at the CUDA path's bf16 storage points
(tests/dcgan_info_oracle.py), MI_optimizer's separate Adam state against torch.optim.Adam, descent of the MI loss and the
dc_info_gan drop-in on the reference's driver lines.  With GM_PARITY_DIR set, the measured errors are written to
$GM_PARITY_DIR/parity_dcgan_info.json."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

import dcgan_harness as H
import dcgan_info_oracle as IO
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_info")
CH = 3


def _engine(hd=16, z=100, nd=10, nc=10, wstd=0.05, seed=11):
    """DcganEngine(variant="info") with N(0, wstd) conv weights (as dcgan_harness.setup) and the oracle G, D and Q holding the
    same weights at the bf16 storage points"""
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant="info", disc_dim=nd, cont_dim=nc)
    g = torch.Generator().manual_seed(seed)
    for net in eng.nets():
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.zero_padding()
    for net in eng.nets():
        net.refresh()
    G, D, Qn = O.Generator(hd, z + nd + nc), O.Discriminator(hd), IO.QNet(hd, nd, nc)
    IO.load_from_engine_weights(G, D, Qn, eng.torch_weights())
    for m in (G, D, Qn):
        m.train()
        m.q = staticmethod(O.bf16_points)
    return eng, G, D, Qn, g


def _noise(n, z, nd, nc, g):
    onehot = torch.zeros(n, nd)
    onehot[range(n), torch.randint(0, nd, (n,), generator=g)] = 1
    return torch.cat([torch.randn(n, z, generator=g), onehot, torch.randn(n, nc, generator=g)], 1)


def _draw(n, zd, nd, nc, seed, stream, ld=None):
    from gm_b200 import _lib
    K = zd + nd + nc
    ld = ld or (K + 1 + 7) // 8 * 8
    rows = torch.full((n, ld), 7.0, device="cuda", dtype=torch.bfloat16)          # garbage: the kernel writes every column
    codes = torch.full((n, K), 7.0, device="cuda")
    h = _lib.ctx()
    _lib.check(h, _lib.lib().gm_info_noise_rows(h, _lib._ptr(rows), ld, _lib._ptr(codes), n, zd, nd, nc, seed, stream, _lib._stream()))
    return rows, codes


# ------------------------------------------------------------------ kernel units
def test_info_noise_rows_sampler():
    """one seeded draw at n = 2^20, nd = 10: one-hot rows with the index in range, the bf16 operand equal to the fp32 copy
    bit for bit with the ones column and zero padding, reproducible per (seed, stream), uniform categories and N(0, 1) codes"""
    n, zd, nd, nc = 1 << 20, 100, 10, 10
    K = zd + nd + nc
    rows, codes = _draw(n, zd, nd, nc, 1234, 5)
    oh = codes[:, zd:zd + nd]
    assert bool(((oh == 0) | (oh == 1)).all()) and bool((oh.sum(1) == 1).all())
    assert torch.equal(rows[:, :K].float(), codes)
    assert bool((rows[:, K] == 1).all()) and bool((rows[:, K + 1:] == 0).all())
    rows2, codes2 = _draw(n, zd, nd, nc, 1234, 5)
    assert torch.equal(rows2, rows) and torch.equal(codes2, codes)
    counts = torch.bincount(oh.argmax(1), minlength=nd).double().cpu()
    sigma = (n * 0.1 * 0.9) ** 0.5
    gauss = torch.cat([codes[:, :zd], codes[:, zd + nd:]], 1).double()
    N = gauss.numel()
    mean, var = float(gauss.mean()), float(gauss.var())
    col_mean = gauss.mean(0)
    rep = {"count_dev_sigma": float((counts - n / nd).abs().max()) / sigma, "mean_se": abs(mean) / (1 / N) ** 0.5,
           "var_se": abs(var - 1) / (2 / N) ** 0.5, "col_mean_se_max": float(col_mean.abs().max()) * n ** 0.5}
    _REPORT.add("sampler", rep)
    assert rep["count_dev_sigma"] < 5 and rep["mean_se"] < 5 and rep["var_se"] < 5 and rep["col_mean_se_max"] < 5, rep
    # a row that crosses 8-column groups inside the one-hot block, nd = 1, and no z columns: still one 1 per row
    for zd2, nd2, nc2 in ((5, 7, 3), (3, 1, 1), (0, 12, 2)):
        r2, c2 = _draw(4096, zd2, nd2, nc2, 9, 2)
        oh2 = c2[:, zd2:zd2 + nd2]
        assert bool((oh2.sum(1) == 1).all()) and torch.equal(r2[:, :zd2 + nd2 + nc2].float(), c2), (zd2, nd2, nc2)
        assert bool((r2[:, zd2 + nd2 + nc2] == 1).all()) and bool((r2[:, zd2 + nd2 + nc2 + 1:] == 0).all())


def test_d_g_and_mi_draws_of_one_step_differ():
    """the engine's D (stream 2 step), G (2 step + 1) and MI (MI_STREAM + step) draws of one step are pairwise different"""
    eng, _, _, _, _ = _engine()
    n, step, seed = 64, 3, 77
    out = []
    for stream in (2 * step, 2 * step + 1, eng.MI_STREAM + step):
        eng.g_forward(n, None, seed, stream)
        out.append(eng.codes_["g"].clone())
    for a in range(3):
        for b in range(a + 1, 3):
            assert not torch.equal(out[a][:, :100], out[b][:, :100]) and not torch.equal(out[a][:, 110:], out[b][:, 110:]), (a, b)
            assert int((out[a][:, 100:110] != out[b][:, 100:110]).any(1).sum()) > n // 2, (a, b)


def test_info_loss_rows_match_float64_torch():
    """gm_info_loss_rows at nd = 7, nc = 3 on fp32 Q rows: the loss to 1e-5, the gradient to one bf16 rounding, zero padding"""
    from gm_b200 import _lib
    n, zd, nd, nc, ld = 1000, 20, 7, 3, 16
    g = torch.Generator(device="cuda").manual_seed(4)
    _, codes = _draw(n, zd, nd, nc, 3, 1)
    q = torch.randn(n, ld, device="cuda", generator=g) * 2
    inv, lam = 1.0 / 4096, 0.7
    grad = torch.full((n, ld), 9.0, device="cuda", dtype=torch.bfloat16)
    loss = torch.zeros(1, device="cuda")
    h = _lib.ctx()
    _lib.check(h, _lib.lib().gm_info_loss_rows(h, _lib._ptr(q), ld, _lib._ptr(codes), zd + nd + nc, zd, n, nd, nc, inv * lam, _lib._ptr(grad),
                                               ld, _lib._ptr(loss), _lib._stream()))
    q64, c64 = q.double().cpu(), codes.double().cpu()
    d, c = IO.mi_terms(q64[:, :nd], q64[:, nd:nd + nc], c64, zd)
    want = float(d + c)
    ref = IO.mi_rows_grad(q64, c64, zd, nd, nc, inv, lam)
    got = grad.double().cpu()
    rel = ((got[:, :nd + nc] - ref).abs() / ref.abs().clamp_min(1e-30)).max()
    rep = {"loss_rel": abs(float(loss[0]) - want) / want, "grad_rel_max": float(rel)}
    _REPORT.add("loss_rows", rep)
    assert rep["loss_rel"] < 1e-5 and rep["grad_rel_max"] <= 2.0 ** -8, rep
    assert bool((got[:, nd + nc:] == 0).all())


# ------------------------------------------------------------------ one D, G and MI step (hidden 16, batch 8)
def _step_report(seed=11):
    n, z, nd, nc = 8, 100, 10, 10
    eng, G, D, Qn, g = _engine(seed=seed)
    imgs = torch.rand(n, CH * 4096, generator=g)
    z1, z2, z3 = (_noise(n, z, nd, nc, g) for _ in range(3))
    rep = {}
    Ld_ref = O.d_loss(G, D, imgs, z1)
    gd = torch.autograd.grad(Ld_ref, list(D.parameters()))
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z1.cuda()).item()
    rep["D_loss"] = abs(Ld - Ld_ref.item()) / abs(Ld_ref.item())
    tg = eng.torch_grads()
    for (name, _), gref in zip(D.named_parameters(), gd):
        rep["gradD_" + name] = nrel(tg["D." + name], gref)
    Lg_ref = O.g_loss(G, D, z2)
    gg = torch.autograd.grad(Lg_ref, list(G.parameters()))
    Lg = eng.g_grad(n, noise=z2.cuda()).item()
    rep["G_loss"] = abs(Lg - Lg_ref.item()) / abs(Lg_ref.item())
    tg = eng.torch_grads()
    for (name, _), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(tg["G." + name], gref)
    # MI step: the gradient reaches Q and, through Q's input, G
    Lm_ref = IO.mi_loss(G, Qn, z3, z)
    gm = torch.autograd.grad(Lm_ref, list(Qn.parameters()) + list(G.parameters()))
    Lm = eng.q_grad(n, noise=z3.cuda()).item()
    rep["MI_loss"] = abs(Lm - Lm_ref.item()) / abs(Lm_ref.item())
    tg = eng.torch_grads()
    names = ["Q." + k for k, _ in Qn.named_parameters()] + ["G." + k for k, _ in G.named_parameters()]
    for name, gref in zip(names, gm):
        rep["gradMI_" + name] = nrel(tg[name], gref)
    assert float(eng.Q.view("l5.weight", eng.Q.grads)[nd + nc:].abs().max()) == 0.0          # Q's padded head rows
    return rep


def test_info_d_g_and_mi_step_match_the_oracle():
    rep = _step_report()
    _REPORT.add("step", rep)
    # 2e-2 on the G loss and 20 % on the gradients, not the 1e-2 / 12 % of test_dcgan_train_step_matches_the_torch_oracle.
    # The G step here is that test's code path, but at hidden 16 and batch 8 both bounds depend on the operating point: the
    # device and this oracle evaluate at slightly different forward points (their bf16 roundings differ where the
    # accumulation orders do), a few per mille of the (Leaky)ReLU units take the other slope, and BatchNorm over 8 images
    # amplifies that.  Over weight seeds 11-18 the G-step gradients are 1.3-18 % from the oracle and the MI-step gradients
    # 1-22 %; at this seed the G loss is 1.25 %, the G step 11-14 % and the MI step 1-12 %.  The arithmetic is held to 2 % by
    # test_g_and_mi_backward_match_float64_at_the_device_forward_points, at the device's own activations (DESIGN.md §6b).
    assert rep["D_loss"] < 5e-3 and rep["MI_loss"] < 5e-3 and rep["G_loss"] < 2e-2, rep
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.20, (k, v, rep)


def test_g_and_mi_backward_match_float64_at_the_device_forward_points():
    """The compositions the device runs for the G step (D's input-gradient chain from the NS rows, sigmoid', G's backward)
    and for the MI step (Q's backward from the MI rows' gradient, with weight gradients, down to the image, sigmoid', G's
    backward), restated in float64 with torch.nn.grad at the device's OWN stored activations, masks and BatchNorm inputs
    (the BEGAN test's restatement of the two stacks).  Both sides then differentiate the same function, so what remains is
    the bf16 rounding of the device's backward tensors.  (z, nd, nc) = (20, 7, 3) gives G 30 input columns, so G's l1
    weight gradient is an fp32 output whose rows start 120 bytes apart (not on 16 bytes)."""
    from test_dcgan_began_gpu import _at, _stack_backward, _trunk_backward, _tw
    n = 8
    for z, nd, nc in ((100, 10, 10), (20, 7, 3)):
        eng, _, _, _, g = _engine(z=z, nd=nd, nc=nc)
        tw = _tw(eng)
        w = {tag: {k[2:]: v for k, v in tw.items() if k.startswith(tag + ".")} for tag in "GDQ"}
        rep = {}
        # G step: the body of DcganEngine.g_grad, keeping its saved tensors
        fake, gsv = eng.g_forward(n, _noise(n, z, nd, nc, g).cuda())
        logits = torch.zeros(16, n, device="cuda")
        sf = eng.d_forward(fake, n, logits, "df")
        ds = torch.zeros(n, device="cuda")
        eng._loss_rows(logits, n, 1, 1.0 / n, ds, C.c_void_p(eng.loss_buf.data_ptr() + 4))
        dpre = eng.d_backward(sf, ds, None, need_wgrad=False, need_dimg=True, tag="df")
        eng.g_backward(gsv, dpre)
        dy = ds.to(torch.bfloat16).double().cpu().view(n, 1)                  # the bf16 column d_backward packs
        _, T = _trunk_backward(eng, sf, dy, w["D"], "")
        f = _at(fake, 64, CH)
        rep["Gstep_dpre"] = nrel(_at(dpre, 64, CH), T * f * (1 - f))
        gref, _ = _stack_backward(eng, gsv, T * f * (1 - f), w["G"], "")
        tg = eng.torch_grads()
        for name, r in gref.items():
            rep["Gstep_G." + name] = nrel(tg["G." + name], r)
        # MI step
        eng.q_grad(n, noise=_noise(n, z, nd, nc, g).cuda())
        s = eng.q_saved_
        qref, T = _trunk_backward(eng, s["qsv"], s["dq"][:, :nd + nc].double().cpu(), w["Q"], "")
        f = _at(s["fake"], 64, CH)
        rep["MI_dpre"] = nrel(_at(s["dpre"], 64, CH), T * f * (1 - f))
        gref, _ = _stack_backward(eng, s["gsv"], T * f * (1 - f), w["G"], "")
        tg = eng.torch_grads()
        for name, r in qref.items():
            rep["MI_Q." + name] = nrel(tg["Q." + name], r)
        for name, r in gref.items():
            rep["MI_G." + name] = nrel(tg["G." + name], r)
        # Q.l1's weight gradient sums 8 x 1024 output positions of an upstream whose signs alternate, so the bf16 rounding of
        # that upstream (which the chain above does not model) reads larger there than anywhere else; from the device's own
        # stored upstream the same GEMM agrees to fp32 accumulation
        from torch.nn.grad import conv2d_weight
        d0 = _at(eng._bufs["qdprev1"][:n * 1024], 32, eng.dc[0])
        rep["MI_Q.l1.weight_from_stored_upstream"] = nrel(tg["Q.l1.weight"], conv2d_weight(_at(s["fake"], 64, CH), w["Q"]["l1.weight"].shape, d0, 2, 1))
        _REPORT.add("float64_at_device_points" + ("" if z == 100 else "_z%d_nd%d_nc%d" % (z, nd, nc)), rep)
        assert len([k for k in rep if k.startswith("MI_Q.")]) == 12 and len([k for k in rep if k.startswith("MI_G.")]) == 13
        assert rep["MI_Q.l1.weight_from_stored_upstream"] < 1e-4, rep
        for k, v in rep.items():
            assert v < (0.04 if k == "MI_Q.l1.weight" else 0.02), (k, v, rep)


def test_apply_mi_keeps_its_own_g_moments():
    """apply(0) then apply_mi on given gradients == torch.optim.Adam as G_optimizer, then a separate Adam(G + Q)"""
    import gm_b200
    eng, _, _, _, _ = _engine()
    g = torch.Generator(device="cuda").manual_seed(8)
    gG1, gG2 = (torch.randn(eng.G.total, device="cuda", generator=g) for _ in range(2))
    gQ = torch.randn(eng.Q.total, device="cuda", generator=g)
    pG, pQ = eng.G.params.clone(), eng.Q.params.clone()
    lr = 1e-3
    hp = gm_b200.AdamHP.make(lr)
    eng.G.grads.copy_(gG1)
    eng.apply(0, hp)
    eng.G.grads.copy_(gG2)
    eng.Q.grads.copy_(gQ)
    eng.apply_mi(hp)
    tG, tQ = pG.clone().requires_grad_(), pQ.clone().requires_grad_()
    optG, optMI = torch.optim.Adam([tG], lr=lr), torch.optim.Adam([tG, tQ], lr=lr)
    tG.grad = gG1.clone()
    optG.step()
    tG.grad, tQ.grad = gG2.clone(), gQ.clone()
    optMI.step()
    # the alternative a shared moment state would give: G's second update from G_optimizer's moments (Adam step 2)
    sG = pG.clone().requires_grad_()
    optS = torch.optim.Adam([sG], lr=lr)
    for gr in (gG1, gG2):
        sG.grad = gr.clone()
        optS.step()
    rep = {"G": nrel(eng.G.params - pG, tG.detach() - pG), "Q": nrel(eng.Q.params - pQ, tQ.detach() - pQ),
           "shared_moments_would_give": nrel(sG.detach() - pG, tG.detach() - pG)}
    _REPORT.add("apply_mi", rep)
    assert rep["G"] < 1e-5 and rep["Q"] < 1e-5 and rep["shared_moments_would_give"] > 1e-2, rep
    assert eng.G.step == 1 and eng.Q.step == 1


# ------------------------------------------------------------------ behaviour
def test_mi_steps_lower_the_mi_loss():
    import gm_b200
    n = 16
    eng, _, _, _, g = _engine()
    noise = _noise(n, 100, 10, 10, g).cuda()
    hp = gm_b200.AdamHP.make(2e-4)
    losses = []
    for _ in range(30):
        losses.append(eng.q_grad(n, noise=noise).item())
        eng.apply_mi(hp)
    _REPORT.add("descent", {"first": losses[0], "last": losses[-1]})
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses


def test_engine_arguments():
    import gm_b200
    from gm_b200 import GmError
    for kw in (dict(variant="ns", disc_dim=10), dict(variant="be", cont_dim=3), dict(variant="info", disc_dim=0),
               dict(variant="info", cont_dim=0)):
        with pytest.raises(GmError):
            gm_b200.DcganEngine(hidden_dim=16, **kw)
    eng = gm_b200.DcganEngine(hidden_dim=16, z_dim=20, variant="info", disc_dim=7, cont_dim=3)
    assert (eng.zin, eng.qp) == (30, 16) and eng.G.shapes["l1.weight"] == (16 * 128, 30)
    assert tuple(eng.torch_weights()["Q.l5.weight"].shape) == (10, 128, 4, 4)
    with pytest.raises(GmError):
        gm_b200.DcganEngine(hidden_dim=16).q_grad(4)


# ------------------------------------------------------------------ the drop-in on the reference's driver lines
def test_dc_info_gan_runs_the_reference_driver_code(capsys):
    import dc_info_gan as M
    g = torch.Generator().manual_seed(0)
    imgs = (torch.rand(64, 3, 64, 64, generator=g) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(64)), batch_size=16, shuffle=True)
    torch.manual_seed(3)
    model = M.DCInfoGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100, disc_dim=10, cont_dim=10)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    trainer = M.DCInfoGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=2, G_lr=2e-4, D_lr=2e-4, D_steps=1)
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("Epoch[")]
    assert len(lines) == 2 and all(", MI Loss: " in ln for ln in lines), lines
    assert len(trainer.Dlosses) == 8 and len(trainer.Glosses) == 8 and len(trainer.MIlosses) == 8
    assert all(np.isfinite(trainer.Dlosses + trainer.Glosses + trainer.MIlosses))
    after = model.state_dict()
    for pfx in ("G.", "D.", "Q."):
        assert all(not torch.equal(before[k], after[k]) for k in before if k.startswith(pfx + "l") and k.endswith("weight")), pfx
    assert not torch.equal(before["Q.bn2.running_mean"], after["Q.bn2.running_mean"])
    out = trainer.generate_images(0, num_outputs=4, c=3)
    assert out.shape == (4, 3, 64, 64) and float(out.min()) >= 0 and float(out.max()) <= 1
    disc, cont = model.Q(imgs[:8].reshape(8, -1))
    assert disc.shape == (8, 10) and cont.shape == (8, 10) and bool(torch.isfinite(disc).all())
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        trainer.save_model(path)
        model2 = M.DCInfoGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100, disc_dim=10, cont_dim=10)
        tr2 = M.DCInfoGANTrainer(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        for k, v in model.state_dict().items():
            assert torch.equal(model2.state_dict()[k], v), k
        zz = tr2.compute_noise(4, 100, 10, 10)
        assert nrel(model2.G(zz), model.G(zz)) < 1e-6
    model.G.zero_grad()
    model.Q.zero_grad()
    gl = trainer.train_G(imgs[:16])
    dl = trainer.train_D(imgs[:16])
    mi = trainer.train_Q(imgs[:16].reshape(16, -1), LAMBDA=0.5)
    mi.backward()
    assert np.isfinite(gl.item()) and np.isfinite(dl.item()) and np.isfinite(mi.item())
    for p in (model.Q.l4.weight, model.G.l1.weight):
        assert p.grad is not None and p.grad.shape == p.shape and float(p.grad.abs().sum()) > 0
