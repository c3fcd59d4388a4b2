"""RaNSGAN, Fisher GAN and DRAGAN on the DCGAN conv path on the GPU: the new kernels against torch (image std sums, DRAGAN's
x_hat, the sigmoid / K penalty, the split batch-statistic loss passes), one D and one G step per variant against fp32
autograd at the CUDA path's bf16 storage points, global statistics from two half batches, DRAGAN's penalty descent,
Fisher's multiplier update and the drop-ins on the reference's driver lines.  With GM_PARITY_DIR set, the measured errors
are written to $GM_PARITY_DIR/parity_dcgan_stats.json."""
import pytest
import torch

import dcgan_harness as H
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_stats")


def _L():
    from gm_b200 import _lib
    return _lib, _lib.ctx()


# ------------------------------------------------------------------ kernel units
def test_std_sums_and_dragan_xhat_rows_match_torch():
    L, h = _L()
    n, cols, C = 5, 3 * 4096, 0.7
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(n, cols, device="cuda", generator=g).to(torch.bfloat16)
    sums = torch.zeros(2, device="cuda", dtype=torch.float64)
    L.check(h, L.lib().gm_dra_std_sums(h, L._ptr(x), n, cols, cols, L._ptr(sums), L._stream()))
    xd = x.double()
    want = torch.stack([xd.sum(), (xd * xd).sum()])
    assert float(((sums - want).abs() / want).max()) < 1e-12
    delta = torch.rand(n, device="cuda", generator=g)
    u = torch.rand(n, cols, device="cuda", generator=g)
    rnd = torch.cat([delta, u.reshape(-1)])
    out = torch.empty_like(x)
    L.check(h, L.lib().gm_dra_xhat_rows(h, L._ptr(x), n, cols, cols, L._ptr(sums), float(n * cols), C, L._ptr(rnd), 0, 0, L._ptr(out), cols,
                                        L._stream()))
    xf = x.float()
    sd = float(xd.std())
    ref = delta.view(n, 1) * xf + (1 - delta.view(n, 1)) * (xf + C * sd * u)
    err = (out.float() - ref).abs() / ref.abs().clamp_min(1e-3)
    _REPORT.add("xhat_rows", {"max_rel": float(err.max()), "std": sd})
    assert float(err.max()) <= 2 ** -8 * 1.01, float(err.max())                 # one bf16 rounding of the fp32 value
    # Philox: keyed by (seed, stream), delta per row and u per element in [0, 1]
    draws = []
    for seed, sid in ((7, 2), (7, 2), (7, 4), (8, 2)):
        L.check(h, L.lib().gm_dra_xhat_rows(h, L._ptr(x), n, cols, cols, L._ptr(sums), float(n * cols), C, None, seed, sid, L._ptr(out),
                                            cols, L._stream()))
        draws.append(out.clone())
    assert torch.equal(draws[0], draws[1]) and not torch.equal(draws[0], draws[2]) and not torch.equal(draws[0], draws[3])
    lo, hi = xf.min(dim=1, keepdim=True)[0], (xf + C * sd).max(dim=1, keepdim=True)[0]
    assert bool((draws[0].float() >= lo - 1e-2).all()) and bool((draws[0].float() <= hi + 1e-2).all())


def test_dragan_penalty_kernel_seed_norm_and_loss():
    L, h = _L()
    n, C, lam, K, inv = 6, 3, 10.0, 0.5, 1.0 / 16
    g = torch.Generator(device="cuda").manual_seed(3)
    J = (torch.randn(n * 4096, C, device="cuda", generator=g) * torch.tensor([0.001, 0.01, 0.1, 1.0, 0.05, 0.3], device="cuda")
         .repeat_interleave(4096).view(-1, 1)).to(torch.bfloat16)
    J[4 * 4096:5 * 4096] = 0                                               # ||J|| = 0: seed 0, loss term K^2
    xh = torch.rand(n * 4096, C, device="cuda", generator=g).to(torch.bfloat16)
    s = torch.tensor([0.3, -1.2, 2.0, 0.0, 0.7, 40.0], device="cuda")     # the last one saturated
    r = torch.full_like(J, 7.0)
    norms = torch.zeros(n, device="cuda")
    loss = torch.full((2,), 0.25, device="cuda")
    L.check(h, L.lib().gm_dra_penalty(h, L._ptr(J), C, L._ptr(xh), C, L._ptr(s), n, 4096, C, lam, K, inv, 1.0 / n, L._ptr(r), C,
                                      L._ptr(norms), L._ptr(loss), L._stream()))
    Jd, xd, sdv = J.double().view(n, -1), xh.double().view(n, -1), s.double()
    nJ = Jd.norm(dim=1)
    sg = torch.sigmoid(sdv)
    sp = sg * (1 - sg)
    ng = sp * nJ
    k = 2 * lam * inv * (ng - K) * sp
    rref = torch.where((nJ > 0).view(n, 1), k.view(n, 1) * (Jd / nJ.clamp_min(1e-300).view(n, 1) + ((1 - 2 * sg) * nJ).view(n, 1) * xd),
                       torch.zeros_like(Jd))
    lref = 0.25 + lam * float(((ng - K) ** 2).mean())
    rep = {"norm": nrel(norms, ng), "r": nrel(r.view(n, -1), rref), "loss": abs(float(loss[0]) - lref) / lref}
    _REPORT.add("penalty_kernel", rep)
    assert float(norms[4]) == 0.0 and bool((r[4 * 4096:5 * 4096] == 0).all())
    assert float(norms[5]) < 1e-15 and float(r[5 * 4096:].float().abs().max()) < 1e-12
    assert rep["norm"] < 1e-6 and rep["loss"] < 1e-6 and rep["r"] < 4e-3, rep            # r: bf16 rounding of the stored seed
    assert float(loss[1]) == 0.25


def _stat_loss_torch(variant, s, n, lam=0.0, rho=0.0):
    """the reference's D loss on logits s [real n | fake n] (float64 autograd): (loss, ds, Omega)"""
    s = s.double().detach().requires_grad_(True)
    d = torch.sigmoid(s)
    DX, DG = d[:n], d[n:]
    omega = None
    if variant == "ra":                                                  # src/ra_gan.py:204-205
        loss = -torch.mean(torch.log(torch.sigmoid(DX - DG.mean()) + 1e-8) + torch.log(torch.sigmoid(1 - DG) + 1e-8)) / 2
    else:                                                                # src/fisher_gan.py:214-223
        omega = 1 - (0.5 * (DX ** 2).mean() + 0.5 * (DG ** 2).mean())
        loss = -((DX.mean() - DG.mean()) + lam * omega - (rho / 2) * omega ** 2)
    ds, = torch.autograd.grad(loss, s)
    return loss.item(), ds, (omega.item() if omega is not None else None)


def _stat_engine(variant):
    import gm_b200
    return gm_b200.DcganEngine(hidden_dim=16, z_dim=100, variant=variant)


def _stat_call(eng, logits, n, stat_batch, inv, stats=None):
    stats = torch.zeros(8, device="cuda", dtype=torch.float64) if stats is None else stats
    ds = torch.zeros(2 * n, device="cuda")
    loss = torch.zeros(4, device="cuda")
    eng.loss_stats(logits, n, stat_batch, stats)
    eng.loss_rows_stats(logits, n, stat_batch, stats, inv, ds, loss)
    return stats, ds, loss


@pytest.mark.parametrize("variant", ["ra", "fisher"])
def test_batch_statistic_loss_passes_match_torch(variant):
    n = 37
    eng = _stat_engine(variant)
    g = torch.Generator(device="cuda").manual_seed(4)
    logits = torch.randn(2 * n, device="cuda", generator=g) * 2
    lam, rho = 0.3, 0.5
    eng.fisher_state(lam, rho)
    _, ds, loss = _stat_call(eng, logits, n, n, 1.0 / n)
    lref, dsref, omega = _stat_loss_torch(variant, logits, n, lam, rho)
    rep = {"loss": abs(float(loss[0]) - lref) / abs(lref), "ds": nrel(ds, dsref)}
    if variant == "fisher":
        rep["omega"] = abs(float(loss[2]) - omega)
        rep["lambda"] = abs(eng.fisher_state()[0] - (lam - rho * omega))
    _REPORT.add("loss_pass_" + variant, rep)
    assert rep["loss"] < 1e-5 and rep["ds"] < 1e-5, rep
    if variant == "fisher":
        assert rep["omega"] < 1e-6 and rep["lambda"] < 1e-6, rep
        assert eng.fisher_state()[1] == pytest.approx(rho)


@pytest.mark.parametrize("variant", ["ra", "fisher"])
def test_batch_statistics_of_two_halves_equal_the_full_batch(variant):
    """two ranks' halves on one GPU: their statistic buffers summed between the passes give the full batch's ds, loss and
    LAMBDA to fp32 rounding"""
    n = 16
    g = torch.Generator(device="cuda").manual_seed(5)
    logits = torch.randn(4 * n, device="cuda", generator=g)              # [real 2n | fake 2n]
    eng = _stat_engine(variant)
    eng.fisher_state(0.2, 0.1)
    _, ds_full, loss_full = _stat_call(eng, logits, 2 * n, 2 * n, 1.0 / (2 * n))
    lam_full = eng.fisher_state()[0]
    halves = [torch.cat([logits[k * n:(k + 1) * n], logits[2 * n + k * n:2 * n + (k + 1) * n]]).contiguous() for k in range(2)]
    engs = [_stat_engine(variant) for _ in range(2)]
    for e in engs:
        e.fisher_state(0.2, 0.1)
    st = [torch.zeros(8, device="cuda", dtype=torch.float64) for _ in range(2)]
    L, h = _L()
    from gm_b200._lib import VARIANTS
    v = VARIANTS[variant]
    for k in range(2):
        L.check(h, L.lib().gm_loss_stats(h, v, 0, L._ptr(halves[k]), n, 2 * n, 0, None, L._ptr(st[k]), L._stream()))
    tot = st[0] + st[1]
    if variant == "ra":
        for k in range(2):
            st[k][:4] = tot[:4]
            L.check(h, L.lib().gm_loss_stats(h, v, 0, L._ptr(halves[k]), n, 2 * n, 1, L._ptr(st[k]), L._ptr(st[k][4:]), L._stream()))
        tot[4:] = st[0][4:] + st[1][4:]
    out = []
    for k in range(2):
        ds = torch.zeros(2 * n, device="cuda")
        loss = torch.zeros(4, device="cuda")
        engs[k].loss_rows_stats(halves[k], n, 2 * n, tot.clone(), 1.0 / (2 * n), ds, loss)
        out.append((ds, loss))
    ds_split = torch.cat([out[0][0][:n], out[1][0][:n], out[0][0][n:], out[1][0][n:]])
    loss_split = 0.5 * (float(out[0][1][0]) + float(out[1][1][0]))
    rep = {"ds": nrel(ds_split, ds_full), "loss": abs(loss_split - float(loss_full[0])) / abs(float(loss_full[0]))}
    if variant == "fisher":
        rep["lambda"] = [abs(e.fisher_state()[0] - lam_full) for e in engs]
    _REPORT.add("split_stats_" + variant, rep)
    assert rep["ds"] < 1e-6 and rep["loss"] < 1e-5, rep
    if variant == "fisher":
        assert max(rep["lambda"]) < 1e-7, rep


# ------------------------------------------------------------------ one D step and one G step (hidden 16, batch 8)
@pytest.mark.parametrize("variant", ["ra", "fisher"])
def test_ra_fisher_d_and_g_step_match_the_oracle(variant):
    n, z = 8, 100
    eng, G, D, _ = H.setup(variant)
    lam, rho = 0.4, 0.3
    eng.fisher_state(lam, rho)
    g = torch.Generator().manual_seed(5)
    imgs = torch.rand(n, 3 * 64 * 64, generator=g)
    z1, z2 = torch.randn(n, z, generator=g), torch.randn(n, z, generator=g)
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z1.cuda()).item()
    DX, DG = D(imgs).view(-1), D(G(z1)).view(-1)
    if variant == "ra":
        Ld_ref = -torch.mean(torch.log(torch.sigmoid(DX - DG.mean()) + 1e-8) + torch.log(torch.sigmoid(1 - DG) + 1e-8)) / 2
    else:
        omega = 1 - (0.5 * (DX ** 2).mean() + 0.5 * (DG ** 2).mean())
        Ld_ref = -((DX.mean() - DG.mean()) + lam * omega - (rho / 2) * omega ** 2)
    gd = torch.autograd.grad(Ld_ref, list(D.parameters()))
    rep = {"D_loss": abs(Ld - Ld_ref.item()) / abs(Ld_ref.item())}
    tg = eng.torch_grads()
    for (name, p), gref in zip(D.named_parameters(), gd):
        rep["gradD_" + name] = nrel(tg["D." + name], gref)
    if variant == "fisher":
        rep["lambda"] = abs(eng.fisher_state()[0] - (lam - rho * float(omega)))
    # G step: NS for RaNS (as the conv NSGAN), -mean(D(G(z))) for Fisher
    Lg = eng.g_grad(n, noise=z2.cuda()).item()
    dg = D(G(z2)).view(-1)
    Lg_ref = -torch.mean(torch.log(dg + 1e-8)) if variant == "ra" else -dg.mean()
    gg = torch.autograd.grad(Lg_ref, list(G.parameters()))
    rep["G_loss"] = abs(Lg - Lg_ref.item()) / abs(Lg_ref.item())
    tg = eng.torch_grads()
    for (name, p), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(tg["G." + name], gref)
    _REPORT.add("step_" + variant, rep)
    assert rep["D_loss"] < 5e-3 and rep["G_loss"] < 1e-2, rep
    if variant == "fisher":
        assert rep["lambda"] < 5e-3 * rho * abs(float(omega)), rep        # Omega of the device's scores vs the oracle's
    # the BatchNorm-D step bounds of test_dcgan_gpu (a common-mode upstream gradient that BatchNorm's backward removes)
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.12, (k, v, rep)


def test_dra_d_step_matches_autograd_and_the_closed_form_oracle():
    n, lam, K, Cc = 8, 10.0, 1.0, 1.0
    eng, G, D, imgs, z, (delta, u) = H.critic_setup("dra", n=n)
    Ld = eng.d_grad(eng.stage_images(imgs.cuda()), n, noise=z.cuda(), gp_lambda=lam, gp_k=K, dra_c=Cc, delta=delta.cuda(),
                    u=u.cuda()).item()
    norms = eng.gp_norms_.cpu().double()
    gp = lam * float(((norms - K) ** 2).mean())
    tg = eng.torch_grads()
    got = [tg["D.l%d.weight" % (i + 1)].cpu() for i in range(5)]
    with torch.no_grad():
        fake = G(z)
    xh = O.make_xhat(imgs, delta, u, Cc)
    ex = O.autograd_d_step(D, imgs, fake, xh, lam, K)
    Gq = O.Generator(D.l1.weight.shape[0], z.shape[1])
    Gq.load_state_dict(G.state_dict())
    Gq.q = staticmethod(O.bf16_points)
    Gq.train()
    with torch.no_grad():
        fake_q = Gq(z)
    rq = O.bf16_points(imgs)
    xh_q = O.bf16_points(O.make_xhat(rq, delta, u, Cc))
    cf = O.closed_form_d_step(D, rq, fake_q, xh_q, lam, K, q=O.bf16_points)
    rep = {"D_loss": abs(Ld - float(ex["loss"])) / abs(float(ex["loss"])), "GP": abs(gp - float(ex["gp"])) / abs(float(ex["gp"])),
           "NS_part": abs((Ld - gp) - float(ex["rows"])) / abs(float(ex["rows"])), "norms_vs_exact": nrel(norms, ex["norms"]),
           "norms_vs_bf16_oracle": nrel(norms, cf["norms"]), "xhat_logits_vs_bf16_oracle": nrel(eng.gp_logits_, cf["s"])}
    for i in range(5):
        rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] = nrel(got[i], cf["grads"][i])
        rep["gradD_l%d_vs_exact" % (i + 1)] = nrel(got[i], ex["grads"][i])
        scale = sum(float(cf["parts"][k][i].norm()) for k in ("real", "fake", "penalty"))
        rep["gradD_l%d_cancellation" % (i + 1)] = scale / float(cf["grads"][i].norm())
        rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] = float((got[i].double() - cf["grads"][i].double()).norm()) / scale
    _REPORT.add("d_step_dra", rep)
    assert rep["D_loss"] < 5e-3 and rep["GP"] < 5e-3, rep
    # the WGAN-GP critic bounds of test_dcgan_wgp_gpu
    for i in range(5):
        assert rep["gradD_l%d_vs_bf16_oracle_of_parts" % (i + 1)] < 3e-2, rep
        assert rep["gradD_l%d_vs_bf16_oracle" % (i + 1)] < 5e-2, rep


def test_dra_g_step_matches_the_oracle():
    n = 8
    eng, G, D, imgs, z, _ = H.critic_setup("dra", n=n)
    Lg = eng.g_grad(n, noise=z.cuda()).item()
    G.q = staticmethod(O.bf16_points)
    s, _ = D.trace(G(z), O.bf16_points)
    loss = -torch.mean(torch.log(torch.sigmoid(s) + 1e-8))               # src/dra_gan.py:245
    gg = torch.autograd.grad(loss, list(G.parameters()))
    rep = {"G_loss": abs(Lg - loss.item()) / abs(loss.item())}
    tg = eng.torch_grads()
    for (name, p), gref in zip(G.named_parameters(), gg):
        rep["gradG_" + name] = nrel(tg["G." + name], gref)
    _REPORT.add("g_step_dra", rep)
    assert rep["G_loss"] < 5e-3, rep
    for k, v in rep.items():
        if k.startswith("grad"):
            assert v < 0.12, (k, v, rep)


def test_dra_split_batch_sums_to_the_full_batch():
    """data-parallel contract on one GPU: with std(x) summed over both halves through stats_reduce, the D gradient of 2n
    images equals the SUM of the two n-image gradients at inv_global_batch = 1/(2n)"""
    H.split_batch_sums_to_the_full_batch("dra", _REPORT, "dra_split_batch")


# ------------------------------------------------------------------ behaviour
def test_dra_penalty_pulls_gradient_norms_to_k():
    H.penalty_pulls_gradient_norms_to_one("dra", None, _REPORT, "dra_penalty_descent")


def test_fisher_lambda_follows_rho_omega_step_by_step():
    import gm_b200
    n = 8
    eng, G, D, _ = H.setup("fisher")
    g = torch.Generator().manual_seed(6)
    x = eng.stage_images(torch.rand(n, 3 * 64 * 64, generator=g).cuda())
    rho = 0.05
    eng.fisher_state(0.0, rho)
    hp = gm_b200.AdamHP.make(1e-3)
    lam = 0.0
    errs = []
    for s in range(6):
        eng.d_grad(x, n, seed=3, step=s)
        omega = float(eng.fisher_omega_)
        new = eng.fisher_state()[0]
        errs.append(abs(new - (lam - rho * omega)))
        lam = new
        eng.apply(1, hp)
    _REPORT.add("fisher_lambda", {"max_err": max(errs), "lambda": lam})
    assert max(errs) < 1e-7 and lam != 0.0, errs


# ------------------------------------------------------------------ the drop-ins on the reference's driver lines
@pytest.mark.parametrize("which", ["ra", "fisher", "dra"])
def test_dropins_run_the_reference_driver_code(which):
    H.run_reference_driver_lines(which)
