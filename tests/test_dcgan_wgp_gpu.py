"""WGAN-GP on the DCGAN conv path on the GPU: the new kernels against torch (interpolation, masked im2col, penalty), one
critic step against autograd's double backward and against the closed-form oracle at the CUDA path's bf16 storage points
(oracle/dcgan_torch.py), the generator step, the data-parallel split, the penalty's descent, and the dc_w_gp_gan drop-in
on the reference's driver lines.  With GM_PARITY_DIR set, the measured errors are written to
$GM_PARITY_DIR/parity_dcgan_wgp.json."""
import pytest
import torch

import dcgan_harness as H
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_wgp")


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
    rep = {"norm": nrel(norms, nref), "r": nrel(r.view(n, -1), rref), "loss": abs(float(loss[0]) - lref) / lref}
    _REPORT.add("penalty_kernel", rep)
    assert float(norms[4]) == 0.0 and bool((r[4 * 4096:5 * 4096] == 0).all())
    assert rep["norm"] < 1e-6 and rep["loss"] < 1e-6 and rep["r"] < 4e-3, rep        # r: bf16 rounding of the stored seed
    assert float(loss[1]) == 0.25


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_wgp_d_step_matches_autograd_and_the_closed_form_oracle(out_act):
    n = 8
    eng, G, D, imgs, z, (eps,) = H.critic_setup("wgp", out_act, n=n)
    lam = 10.0
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z.cuda(), gp_lambda=lam, eps=eps.cuda()).item()
    norms = eng.gp_norms_.cpu().double()
    gp = lam * float(((norms - 1) ** 2).mean())
    tg = eng.torch_grads()
    got = [tg["D.l%d.weight" % (i + 1)].cpu() for i in range(5)]
    assert torch.equal(eng.gp_eps_.cpu(), eps)
    # exact: fp32 autograd double backward (generator and critic in fp32)
    with torch.no_grad():
        fake = G(z)
    ex = O.autograd_d_step(D, imgs, fake, O.interpolate(imgs, fake, eps), lam)
    # closed form at the CUDA path's bf16 storage points
    Gq = O.Generator(D.l1.weight.shape[0], z.shape[1])
    Gq.load_state_dict(G.state_dict())
    Gq.q = staticmethod(O.bf16_points)
    Gq.train()
    with torch.no_grad():
        fake_q = Gq(z)
    cf = O.closed_form_d_step(D, imgs, fake_q, O.interpolate(imgs, fake_q, eps, O.bf16_points), lam, q=O.bf16_points)
    live = int((norms > 0).sum())
    rep = {"live_rows": live, "D_loss": abs(Ld - float(ex["loss"])) / abs(float(ex["loss"])),
           "GP": abs(gp - float(ex["gp"])) / abs(float(ex["gp"])),
           "W_part": abs((Ld - gp) - float(ex["rows"])) / max(abs(float(ex["rows"])), 1e-30),
           "norms_vs_exact": nrel(norms, ex["norms"])}
    for i in range(5):
        rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] = nrel(got[i], cf["grads"][i])
        rep["gradD_l%d_vs_exact" % (i + 1)] = nrel(got[i], ex["grads"][i])
        # the gradient is a sum of three parts (real rows, fake rows, penalty) of which the first two nearly cancel: the
        # bf16 rounding of each part shows against the size of the parts, not of their sum
        scale = sum(float(cf["parts"][k][i].norm()) for k in ("real", "fake", "penalty"))
        rep["gradD_l%d_cancellation" % (i + 1)] = scale / float(cf["grads"][i].norm())
        rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] = float((got[i].double() - cf["grads"][i].double()).norm()) / scale
    _REPORT.add("d_step_" + out_act, rep)
    if out_act == "relu":
        assert live >= n // 2, rep
    assert rep["D_loss"] < 5e-3 and rep["GP"] < 5e-3, rep
    # the W part is a difference of two means of similar size; measured against the scale of its terms
    with torch.no_grad():
        w_scale = float(D(imgs).abs().mean() + D(fake).abs().mean())
    assert abs((Ld - gp) - float(ex["rows"])) < 5e-3 * w_scale, (rep, w_scale)
    for i in range(5):
        assert rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] < 3e-2, rep
        assert rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] < 5e-2, rep


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_wgp_g_step_matches_the_oracle(out_act):
    n = 8
    eng, G, D, imgs, z, _ = H.critic_setup("wgp", out_act, n=n, live="fake")
    Lg = eng.g_grad(n, noise=z.cuda()).item()
    G.q = staticmethod(O.bf16_points)
    zq = z.clone()
    s, _ = D.trace(G(zq), O.bf16_points)
    loss = -D.out(s).mean()                                             # src/w_gp_gan.py:237
    gg = torch.autograd.grad(loss, list(G.parameters()))
    live = int((s > 0).sum())
    rep = {"live_rows": live, "G_loss": abs(Lg - loss.item()) / abs(loss.item())}
    assert live >= n // 2 or out_act == "none", rep
    tg = eng.torch_grads()
    for (name, p), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(tg["G." + name], gref)
    _REPORT.add("g_step_" + out_act, rep)
    assert rep["G_loss"] < 5e-3, rep
    # as in test_dcgan_gpu: the upstream gradient is one number per sample (-1/n), BatchNorm's backward removes that common
    # mode and the bf16 rounding of what is left reads as several percent
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.12, (k, v, rep)


def test_wgp_split_batch_sums_to_the_full_batch():
    H.split_batch_sums_to_the_full_batch("wgp", _REPORT, "split_batch")


@pytest.mark.parametrize("out_act", ["relu", "none"])
def test_the_penalty_pulls_gradient_norms_to_one(out_act):
    H.penalty_pulls_gradient_norms_to_one("wgp", out_act, _REPORT, "penalty_descent_" + out_act)


def test_dc_w_gp_gan_runs_the_reference_driver_code():
    """src/w_gp_gan.py's __main__ lines on the conv model at hidden 16 and 64x64x3 synthetic images"""
    H.run_reference_driver_lines("wgp")
