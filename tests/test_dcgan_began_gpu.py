"""BEGAN on the DCGAN conv path on the GPU: gm_l1_rows against torch, the loss finalisation, K control and plateau scheduler
against a host restatement of src/be_gan.py:186-195, Adam's device lr scale, one D step and one G step against fp32 autograd
at the CUDA path's bf16 storage points (tests/dcgan_began_oracle.py), global statistics from two half batches, descent of
DX and the dc_be_gan drop-in on the reference's driver lines.  With GM_PARITY_DIR set, the measured errors are written to
$GM_PARITY_DIR/parity_dcgan_began.json."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest
import torch

import dcgan_began_oracle as BO
import dcgan_harness as H
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_began")
CH, HW = 3, 4096


def _engine(hd=16, z=100, wstd=0.05, seed=11):
    """DcganEngine(variant="be") with N(0, wstd) conv weights (as dcgan_harness.setup) and the oracle G / autoencoder holding
    the same weights at the bf16 storage points"""
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant="be")
    g = torch.Generator().manual_seed(seed)
    for net in (eng.G, eng.D):
        for name in net.names:
            if name.split(".")[-2].startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.zero_padding()
    eng.G.refresh(); eng.D.refresh()
    G, AE = O.Generator(hd, z), BO.AutoEncoder(hd, eng.e)
    BO.load_from_engine_weights(G, AE, eng.torch_weights())
    G.train(); AE.train()
    G.q = AE.q = staticmethod(O.bf16_points)
    return eng, G, AE, g


def _nchw(rows, n):
    """NHWC rows [n*4096, ch] -> flat NCHW [n, ch*4096] (the layout D reads)"""
    return rows.float().view(n, 64, 64, CH).permute(0, 3, 1, 2).reshape(n, -1).cpu()


# ------------------------------------------------------------------ kernel units
def test_l1_rows_sum_and_gradient_match_torch():
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=16, variant="be")
    n = 5
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(n * HW, CH, device="cuda", generator=g).to(torch.bfloat16)
    r = (torch.randn(n * HW, CH, device="cuda", generator=g) * 0.7).to(torch.bfloat16)
    r[:700] = x[:700]                                                    # exact zeros: sign(0) = 0
    d64 = r.double() - x.double()
    want = float(d64.abs().sum())
    coef = torch.tensor([0.37], device="cuda")
    rep = {}
    for inv, cf in ((1.0 / 16, None), (-1.0 / 16, coef)):
        grad = torch.full_like(r, 5.0)
        tot = torch.zeros(1, device="cuda", dtype=torch.float64)
        eng.l1_rows(r, x, n, inv, cf, grad, tot)
        ref = torch.sign(r.float() - x.float()) * torch.tensor(inv, dtype=torch.float32, device="cuda")
        if cf is not None:
            ref = ref * cf
        ref = ref.to(torch.bfloat16)
        key = "coef" if cf is not None else "plain"
        rep["sum_rel_" + key] = abs(float(tot[0]) - want) / want
        rep["grad_mismatches_" + key] = int((grad != ref).sum())
        assert bool((grad[:700] == 0).all())
    # rows x cols of 3001 x 1448: 543 181 16-byte groups, not a multiple of the 512 a block covers per pass and more than
    # the largest grid covers in one (8 blocks per SM), so threads run several grid-stride passes and the unrolled tail slot
    from gm_b200 import _lib
    h = _lib.ctx()
    rows, cols = 3001, 1448
    assert rows * cols // 8 % 512 and rows * cols // 8 > _lib.lib().gm_ctx_num_sms(h) * 8 * 512
    x2 = torch.rand(rows, cols, device="cuda", generator=g).to(torch.bfloat16)
    r2 = torch.rand(rows, cols, device="cuda", generator=g).to(torch.bfloat16)
    r2[-1, -5:] = x2[-1, -5:]
    grad = torch.full_like(r2, 5.0)
    tot = torch.zeros(1, device="cuda", dtype=torch.float64)
    _lib.check(h, _lib.lib().gm_l1_rows(h, _lib._ptr(r2), _lib._ptr(x2), rows, cols, 0.5, _lib._ptr(coef), _lib._ptr(grad), _lib._ptr(tot),
                                        _lib._stream()))
    want2 = float((r2.double() - x2.double()).abs().sum())
    ref2 = (torch.sign(r2.float() - x2.float()) * torch.tensor(0.5, device="cuda") * coef).to(torch.bfloat16)
    rep["sum_rel_odd"], rep["grad_mismatches_odd"] = abs(float(tot[0]) - want2) / want2, int((grad != ref2).sum())
    _REPORT.add("l1_rows", rep)
    assert rep["sum_rel_plain"] < 1e-12 and rep["sum_rel_coef"] < 1e-12 and rep["sum_rel_odd"] < 1e-12, rep
    assert rep["grad_mismatches_plain"] == 0 and rep["grad_mismatches_coef"] == 0 and rep["grad_mismatches_odd"] == 0, rep


def _dx_dg_sequence(steps=20):
    """(DX, DG) per step: K pushed up to the clip at 1, then down to the clip at 0, then a plateau of the convergence measure
    (constant, so the schedulers halve the rate every patience + 1 steps)"""
    rng = np.random.default_rng(3)
    out = []
    for s in range(steps):
        DX = float(rng.uniform(1.0, 3.0))
        if s < 5:
            DG = 0.5 * DX - 1.0                                              # gamma DX - DG = +1
        elif s < 11:
            DG = 0.5 * DX + 1.0                                              # -1
        else:
            DX, DG = 1.5, 0.5
        out.append((DX, DG))
    return out


def test_began_loss_final_control_and_plateau_follow_the_reference():
    """20 steps of given (DX, DG): the D-step loss DX - K DG, then K <- clip(K + LAMBDA (GAMMA DX - DG), 0, 1), the
    convergence measure and the two ReduceLROnPlateau(factor 0.5, threshold 0.01, patience) of src/be_gan.py:133-136,186-195
    (restated with torch's own scheduler)"""
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=16, variant="be")
    B, gamma, lam, patience = 8, 0.5, 0.4, 2
    eng.began_init(0.2, B)
    opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=1.0)
    sched = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, factor=0.50, threshold=0.01, patience=patience)
    K = 0.2
    loss = torch.zeros(1, device="cuda")
    errs = {"loss": 0.0, "K": 0.0, "conv": 0.0, "bad": 0.0, "lr": 0.0}
    clipped = set()
    for DX, DG in _dx_dg_sequence():
        sums = torch.tensor([DX * B, DG * B], device="cuda", dtype=torch.float64)
        eng.began_loss_final(sums, B, 0, loss)
        st = eng.began_state()
        errs["loss"] = max(errs["loss"], abs(float(loss[0]) - (DX - K * DG)) / abs(DX - K * DG))
        eng.began_control(gamma, lam, patience)
        st = eng.began_state()
        conv = st[3] + abs(gamma * st[3] - st[4])                              # src/be_gan.py:189, on the device's fp32 DX, DG
        K = min(max(0.0, K + lam * (gamma * st[3] - st[4])), 1.0)              # src/be_gan.py:190-191
        sched.step(st[10])                                                     # src/be_gan.py:194-195, on the device's measure
        clipped |= {K} & {0.0, 1.0}
        errs["K"] = max(errs["K"], abs(st[0] - K))
        errs["conv"] = max(errs["conv"], abs(st[10] - conv) / conv)
        errs["bad"] = max(errs["bad"], abs(st[6] - sched.num_bad_epochs))
        errs["lr"] = max(errs["lr"], abs(st[7] - opt.param_groups[0]["lr"]))
        K = st[0]
    _REPORT.add("control", dict(errs, lr_scale=opt.param_groups[0]["lr"]))
    assert clipped == {0.0, 1.0}, clipped
    assert opt.param_groups[0]["lr"] < 1.0                                     # the plateau fired at least once
    assert errs["loss"] < 1e-6 and errs["K"] < 1e-6 and errs["conv"] < 1e-6 and errs["bad"] == 0 and errs["lr"] == 0, errs


def test_adam_lr_scale_equals_adam_at_the_scaled_rate():
    import gm_b200
    from gm_b200 import _lib
    g = torch.Generator(device="cuda").manual_seed(2)
    p0 = torch.randn(1000, device="cuda", generator=g)
    grads = [torch.randn(1000, device="cuda", generator=g) for _ in range(3)]
    scale = torch.tensor([0.125], device="cuda")
    out = []
    for mode in ("scaled", "plain"):
        p, m, v = p0.clone(), torch.zeros_like(p0), torch.zeros_like(p0)
        hp = gm_b200.AdamHP.make(2e-3 if mode == "scaled" else float(np.float32(2e-3) * np.float32(0.125)))
        for s, gr in enumerate(grads):
            if mode == "scaled":
                _lib.adam_step(p, gr, m, v, hp, s + 1, lr_scale=scale)
            else:
                h = _lib.ctx()
                _lib.check(h, _lib.lib().gm_adam_step(h, _lib._ptr(p), _lib._ptr(gr), _lib._ptr(m), _lib._ptr(v), p.numel(), C.byref(hp),
                                                      s + 1, _lib._stream()))
        out.append(p)
    assert torch.equal(out[0], out[1])
    assert not torch.equal(out[0], p0)


# ------------------------------------------------------------------ one D step and one G step (hidden 16, batch 8)
def test_began_d_and_g_step_match_the_oracle():
    n, z, K = 8, 100, 0.3
    eng, G, AE, g = _engine()
    imgs = torch.rand(n, CH * HW, generator=g)
    z1, z2 = torch.randn(n, z, generator=g), torch.randn(n, z, generator=g)
    eng.began_init(K, n)
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z1.cuda()).item()
    st = eng.began_state()
    s_real = torch.sign(_nchw(eng.be_dr_[0], n))
    s_fake = -torch.sign(_nchw(eng.be_dr_[1], n))                          # the fake half carries -K inv
    x = O.bf16_points(imgs)
    with torch.no_grad():
        fake = G(z1)
        flips = [int((torch.sign(AE(v) - v) != s).sum()) for v, s in ((x, s_real), (fake, s_fake))]
    Ld_ref, DX_ref, DG_ref = BO.d_loss(AE, x, fake, K, (s_real, s_fake))
    gd = torch.autograd.grad(Ld_ref, list(AE.parameters()))
    rep = {"D_loss": abs(Ld - Ld_ref.item()) / abs(Ld_ref.item()), "DX": abs(st[3] - DX_ref.item()) / DX_ref.item(),
           "DG": abs(st[4] - DG_ref.item()) / DG_ref.item(), "sign_flips_real": flips[0], "sign_flips_fake": flips[1],
           "values_per_half": n * CH * HW}
    tg = eng.torch_grads()
    for (name, _), gref in zip(AE.named_parameters(), gd):
        rep["gradD_" + name] = nrel(tg["D." + name], gref)
    # G step: the gradient reaches G(z) through D and directly
    Lg = eng.g_grad(n, noise=z2.cuda()).item()
    s_g = torch.sign(_nchw(eng.be_drg_, n))
    with torch.no_grad():
        fg = G(z2)
        rep["sign_flips_g"] = int((torch.sign(AE(fg) - fg) != s_g).sum())
    Lg_ref = BO.g_loss(AE, G, z2, s_g)
    gg = torch.autograd.grad(Lg_ref, list(G.parameters()))
    rep["G_loss"] = abs(Lg - Lg_ref.item()) / abs(Lg_ref.item())
    tg = eng.torch_grads()
    for (name, _), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(tg["G." + name], gref)
    _REPORT.add("step", rep)
    assert rep["D_loss"] < 5e-3 and rep["DX"] < 5e-3 and rep["DG"] < 5e-3 and rep["G_loss"] < 5e-3, rep
    # 20 %, not the 12 % of the DCGAN steps.  The device and this oracle differentiate at slightly different forward points
    # (their bf16 roundings differ where the accumulation orders do), so a few per mille of the (Leaky)ReLU units take the
    # other slope; each flip swaps a whole term of the gradient, so the relative error grows like the square root of the
    # flipped fraction, a few per cent per layer, over up to 9 BatchNorm layers below the L1 term (4 in NSGAN's D).  bf16
    # storage alone moves these gradients 20 - 46 % from exact fp32 at the same L1 signs.  The arithmetic itself is held to
    # 2 % by test_began_backward_matches_float64_at_the_device_forward_points, at the device's own activations (DESIGN.md §6b).
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.20, (k, v, rep)


def _at(t, hw, C):
    """stored NHWC rows [n*hw*hw, >= C] -> NCHW float64 on the CPU"""
    return t[:, :C].double().reshape(-1, hw, hw, C).permute(0, 3, 1, 2).cpu()


def _tw(eng):
    """the device's bf16 operand copies of every weight in torch's layout (float64), BatchNorm vectors as they are"""
    return {k: (v.to(torch.bfloat16) if ".l" in k else v).double() for k, v in eng.torch_weights().items()}


def _bn_parts(g, c, gamma_eps):
    """(dL/dc, dgamma, dbeta) of BatchNorm2d in training mode at its input c, for g = dL/d(BatchNorm output)"""
    gamma, eps = gamma_eps
    bn = torch.nn.BatchNorm2d(c.shape[1], eps=eps).double()
    with torch.no_grad():
        bn.weight.copy_(gamma)
    dims = (0, 2, 3)
    xh = (c - c.mean(dims, keepdim=True)) * (c.var(dims, unbiased=False, keepdim=True) + eps).rsqrt()
    return BO._bn_backward(g, c, bn), (g * xh).sum(dims), g.sum(dims)


def _stack_backward(eng, sv, d, w, pfx):
    """backward of the transposed-conv stack (G, or BEGAN's decoder) in float64 at the device's stored forward tensors sv:
    d = dL/d(output before its activation) NCHW -> ({torch name: gradient}, dL/d(input rows) [n, K])"""
    from torch.nn.grad import conv2d_weight
    import torch.nn.functional as F
    gc, out, hw = eng.gc, {}, 64
    for i in (3, 2, 1, 0):
        hw //= 2
        a, c = _at(sv["a%d" % i], hw, gc[i]), _at(sv["c%d" % i], hw, gc[i])
        W = w[pfx + "l%d.weight" % (i + 2)]
        out[pfx + "l%d.weight" % (i + 2)] = conv2d_weight(d, W.shape, a, 2, 1)
        g = F.conv2d(d, W, None, 2, 1) * (a > 0).double()
        d, out[pfx + "bn%d.weight" % (i + 1)], out[pfx + "bn%d.bias" % (i + 1)] = _bn_parts(g, c, (w[pfx + "bn%d.weight" % (i + 1)], 1e-5))
    W1 = w[pfx + "l1.weight"]
    zin = sv["z"][:, :W1.shape[0]].double().cpu().view(-1, W1.shape[0], 1, 1)
    out[pfx + "l1.weight"] = conv2d_weight(d, W1.shape, zin, 1, 0)
    return out, F.conv2d(d, W1, None, 1, 0).view(-1, W1.shape[0])


def _trunk_backward(eng, sv, demb, w, pfx):
    """backward of BEGAN's encoder (the D trunk) in float64 at the device's stored forward tensors sv, from demb [n, e] ->
    ({torch name: gradient}, dL/d(image) NCHW)"""
    from torch.nn.grad import conv2d_input, conv2d_weight
    dc, out = eng.dc, {}
    y = [_at(sv["y%d" % i], 32 >> i, dc[i]) for i in range(4)]
    img = _at(sv["img"], 64, CH)
    dh = demb.view(-1, demb.shape[1], 1, 1)
    W5 = w[pfx + "l5.weight"]
    out[pfx + "l5.weight"] = conv2d_weight(y[3], W5.shape, dh, 1, 0)
    d = conv2d_input(y[3].shape, W5, dh, 1, 0)
    for i in (3, 2, 1):
        c = _at(sv["c%d" % i], 32 >> i, dc[i])
        dcv, out[pfx + "bn%d.weight" % (i + 1)], out[pfx + "bn%d.bias" % (i + 1)] = _bn_parts(
            d * O._lrelu_grad(y[i]), c, (w[pfx + "bn%d.weight" % (i + 1)], 1e-5))
        W = w[pfx + "l%d.weight" % (i + 1)]
        out[pfx + "l%d.weight" % (i + 1)] = conv2d_weight(y[i - 1], W.shape, dcv, 2, 1)
        d = conv2d_input(y[i - 1].shape, W, dcv, 2, 1)
    g = d * O._lrelu_grad(y[0])
    out[pfx + "l1.weight"] = conv2d_weight(img, w[pfx + "l1.weight"].shape, g, 2, 1)
    return out, conv2d_input(img.shape, w[pfx + "l1.weight"], g, 2, 1)


def test_began_backward_matches_float64_at_the_device_forward_points():
    """The composition the device runs - decoder backward to the embedding gradient, encoder backward, T - dr through
    sigmoid', G's backward - restated in float64 with torch.nn.grad at the device's OWN stored activations, masks and
    BatchNorm inputs.  Unlike the oracle step test, both sides then differentiate the same function, so what remains is the
    bf16 rounding of the device's backward tensors."""
    n, K = 8, 0.3
    eng, G, AE, g = _engine()
    eng.began_init(K, n)
    w = {k[2:]: v for k, v in _tw(eng).items()}
    rep = {}
    # D step, one half at a time (d_grad runs exactly these calls per half): the real images, then a generated batch with K
    fake, _ = eng.g_forward(n, torch.randn(n, 100, generator=g).cuda())
    halves = ((eng.stage_images(torch.rand(n, CH * HW, generator=g).cuda()), 1.0 / n, None),
              (fake.clone(), -1.0 / n, eng.be_state[0:1]))
    for k, (x, inv, coef) in enumerate(halves):
        rec, sve, svd = eng.autoencode(x, n, "t")
        dr = torch.empty_like(rec)
        eng.l1_rows(rec, x, n, inv, coef, dr, torch.zeros(1, device="cuda", dtype=torch.float64))
        eng.D.grads.zero_()
        eng._autoencoder_backward(sve, svd, dr, eng.D.grads, tag="t")
        got = {k2[2:]: v.double().cpu() for k2, v in eng.torch_grads().items() if k2.startswith("D.")}
        ref, demb = _stack_backward(eng, svd, _at(dr, 64, CH), w, "decoder.")
        ref2, _ = _trunk_backward(eng, sve, demb[:, :eng.e], w, "encoder.")
        ref.update(ref2)
        for name, r in ref.items():
            rep["half%d_%s" % (k, name)] = nrel(got[name], r)
    # G step: T at the device's forward points, dpre = (T - dr) f (1 - f), then G's backward
    eng.g_grad(n, noise=torch.randn(n, 100, generator=g).cuda())
    s = eng.be_g_saved_
    drg = _at(eng.be_drg_, 64, CH)
    _, demb = _stack_backward(eng, s["svd"], drg, w, "decoder.")
    rep["G_demb"] = nrel(s["demb"][:, :eng.e].cpu(), demb)
    _, T = _trunk_backward(eng, s["sve"], demb, w, "encoder.")
    rep["G_T"] = nrel(_at(s["T"], 64, CH), T)
    f = _at(s["fake"], 64, CH)
    dpre = (T - drg) * f * (1 - f)
    rep["G_dpre"] = nrel(_at(s["dpre"], 64, CH), dpre)
    gref, _ = _stack_backward(eng, s["gsv"], dpre, {k[2:]: v for k, v in _tw(eng).items() if k.startswith("G.")}, "")
    tg = eng.torch_grads()
    for name, r in gref.items():
        rep["G_" + name] = nrel(tg["G." + name], r)
    _REPORT.add("float64_at_device_points", rep)
    assert len([k for k in rep if k.startswith("half0")]) == 24 and len([k for k in rep if k.startswith("G_l")]) == 5
    for k, v in rep.items():
        assert v < 0.02, (k, v, rep)


def test_began_padding_stays_zero_and_state_is_on_device():
    """the padded embedding rows / columns get zero gradients (so Adam keeps them zero), and the lr scale reaches Adam"""
    import gm_b200
    n = 4
    eng, G, AE, g = _engine()
    x = eng.stage_images(torch.rand(n, CH * HW, generator=g).cuda())
    eng.began_init(0.5, n)
    eng.d_grad(x, n, seed=1)
    assert float(eng.D.view("encoder.l5.weight", eng.D.grads)[eng.e:].abs().max()) == 0.0
    assert float(eng.D.view("decoder.l1.weight", eng.D.grads)[:, eng.e:].abs().max()) == 0.0
    p = eng.D.params.clone()
    eng.be_state[7] = 0.0                                                  # lr scale 0: Adam leaves D unchanged
    eng.apply(1, gm_b200.AdamHP.make(1e-3))
    assert torch.equal(eng.D.params, p)


# ------------------------------------------------------------------ data-parallel statistics
def test_two_half_batches_through_stats_reduce_equal_the_full_batch():
    """two ranks' halves on one GPU: their L1 sums, summed by stats_reduce, give the full batch's DX, DG and loss"""
    import gm_b200
    n = 4
    g = torch.Generator(device="cuda").manual_seed(7)
    x = [torch.rand(2 * n * HW, CH, device="cuda", generator=g).to(torch.bfloat16) for _ in range(2)]      # real, fake
    r = [(v.float() + 0.3 * torch.randn(v.shape, device="cuda", generator=g)).to(torch.bfloat16) for v in x]
    eng = gm_b200.DcganEngine(hidden_dim=16, variant="be")
    eng.began_init(0.4, 2 * n)
    grad = torch.empty(2 * n * HW, CH, device="cuda", dtype=torch.bfloat16)

    def sums_of(rows):
        s = torch.zeros(2, device="cuda", dtype=torch.float64)
        for k in range(2):
            eng.l1_rows(r[k][rows].contiguous(), x[k][rows].contiguous(), (rows.stop - rows.start) // HW, 1.0, None, grad, s[k:k + 1])
        return s

    loss_full = torch.zeros(1, device="cuda")
    eng.began_loss_final(sums_of(slice(0, 2 * n * HW)), 2 * n, 0, loss_full)
    full = eng.began_state()
    halves = [sums_of(slice(k * n * HW, (k + 1) * n * HW)) for k in range(2)]
    total = halves[0] + halves[1]
    eng.stats_reduce = lambda buf: buf.copy_(total)
    out = []
    for k in range(2):
        loss = torch.zeros(1, device="cuda")
        eng.began_loss_final(halves[k].clone(), 2 * n, 0, loss)
        st = eng.began_state()
        out.append((float(loss[0]), st[3], st[4]))
    eng.stats_reduce = None
    rep = {"loss": max(abs(o[0] - float(loss_full[0])) for o in out) / abs(float(loss_full[0])),
           "DX": max(abs(o[1] - full[3]) for o in out) / full[3], "DG": max(abs(o[2] - full[4]) for o in out) / full[4]}
    _REPORT.add("split_stats", rep)
    assert rep["loss"] < 1e-6 and rep["DX"] < 1e-6 and rep["DG"] < 1e-6, rep


# ------------------------------------------------------------------ behaviour
def test_d_steps_at_k0_lower_the_reconstruction_error():
    import gm_b200
    n = 16
    eng, G, AE, g = _engine()
    x = eng.stage_images(torch.rand(n, CH * HW, generator=g).cuda())
    zc = torch.randn(n, 100, generator=g).cuda()
    eng.began_init(0.0, n)
    hp = gm_b200.AdamHP.make(1e-4)
    dx = []
    for _ in range(30):
        eng.d_grad(x, n, noise=zc)
        dx.append(eng.began_state()[3])
        eng.apply(1, hp)
    _REPORT.add("descent", {"first": dx[0], "last": dx[-1]})
    assert all(np.isfinite(dx)) and dx[-1] < dx[0], dx


# ------------------------------------------------------------------ the drop-in on the reference's driver lines
def test_dc_be_gan_runs_the_reference_driver_code(capsys):
    import dc_be_gan as M
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(64, 3, 64, 64, generator=g)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(64)), batch_size=16, shuffle=True)
    torch.manual_seed(3)
    model = M.DCBEGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    trainer = M.DCBEGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=2, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("Epoch[")]
    assert len(lines) == 2 and all(", K: " in ln and ", Convergence Measure: " in ln for ln in lines), lines
    assert len(trainer.Dlosses) == 8 and len(trainer.Glosses) == 8
    assert all(np.isfinite(trainer.Dlosses)) and all(np.isfinite(trainer.Glosses))
    after = model.state_dict()
    dw = [k for k in before if k.startswith("D.") and ".l" in k and k.endswith("weight")]
    assert len(dw) == 10 and all(not torch.equal(before[k], after[k]) for k in dw)
    assert any(not torch.equal(before[k], after[k]) for k in before if k.startswith("G.") and k.endswith("weight"))
    assert not torch.equal(before["D.decoder.bn1.running_mean"], after["D.decoder.bn1.running_mean"])
    out = trainer.generate_images(0, num_outputs=4)
    assert out.shape == (4, 3, 64, 64)
    rec = model.D(imgs[:8].reshape(8, -1))
    assert rec.shape == (8, 64 * 64 * 3) and bool(torch.isfinite(rec).all())
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        trainer.save_model(path)
        model2 = M.DCBEGAN(image_size=64 * 64 * 3, hidden_dim=16, z_dim=100)
        tr2 = M.DCBEGANTrainer(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        for k, v in model.state_dict().items():
            assert torch.equal(model2.state_dict()[k], v), k
        zz = torch.randn(4, 100)
        assert nrel(model2.G(zz), model.G(zz)) < 1e-6
    model.D.zero_grad()
    loss, DX, DG = trainer.train_D(imgs[:16].reshape(16, -1), 0.25)
    assert abs(loss.item() - (DX.item() - 0.25 * DG.item())) <= 1e-4 * abs(DX.item())
    loss.backward()
    for name in ("encoder.l4.weight", "decoder.l2.weight"):
        p = model.D.get_parameter(name)
        assert p.grad is not None and p.grad.shape == p.shape and float(p.grad.abs().sum()) > 0, name
    gl = trainer.train_G(imgs[:16])
    gl.backward()
    assert np.isfinite(float(gl))
