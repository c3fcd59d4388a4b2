"""north_star's bound in the fp32-grade operand mode (gm_prec GM_PREC_SPLIT, SURVEY.md 8b dtype_mode):
every output of the CUDA path — losses, D scores, EVERY gradient tensor, the weights and Adam moments after
three optimizer steps — within 1e-3 (norm-relative for tensors) of the reference's fp32 CPU path
(src/ns_gan.py:138,155 autograd; golden fixtures made by the unmodified reference) and of the exact
numpy oracle, for every loss variant, the gradient-penalty variants, BEGAN, InfoGAN and the VAE.

Measured errors are written to gpurun_out/parity_split.json."""
import json
import os

import numpy as np
import pytest
import torch

from inputs import (GAN_SHAPES, INFO_SHAPES, BEGAN_SHAPES, VAE_SHAPES, STEPS, B, gm_init_weights, params_dict, load_case,
                    unpack_draws, images_from_bits)
from oracle import ref_math as R
from mlp_harness import DeviceReluSides, aux_from as _aux_from, gan_engine, nrel as _nrel

pytestmark = pytest.mark.gpu
TOL = 1e-3          # north_star: "within 1e-3 relative fp32"
_REPORT = {}

ROW_VARIANTS = ["ns", "mm", "ls", "w", "ra", "fisher", "f_total_variation", "f_forward_kl", "f_reverse_kl",
                "f_pearson", "f_hellinger", "f_jensen_shannon"]
GP_VARIANTS = ["wgp", "dra"]
KW = {"wgp": dict(G_lr=1e-4, D_lr=1e-4), "dra": dict(G_lr=1e-4, D_lr=1e-4), "ns": dict(G_lr=2e-4, D_lr=2e-4),
      "mm": dict(G_lr=2e-4, D_lr=2e-4, G_init=2), "ls": dict(G_lr=1e-4, D_lr=1e-4),
      "w": dict(G_lr=5e-5, D_lr=5e-5, D_steps=2, clip=0.01), "ra": dict(G_lr=2e-4, D_lr=2e-4),
      "fisher": dict(G_lr=1e-4, D_lr=1e-4, RHO=1e-6)}
for _m in ROW_VARIANTS:
    KW.setdefault(_m, dict(G_lr=1e-4, D_lr=1e-4))
G_NAMES = ["G.linear.weight", "G.linear.bias", "G.generate.weight", "G.generate.bias"]
D_NAMES = ["D.linear.weight", "D.linear.bias", "D.discriminate.weight", "D.discriminate.bias"]


def _dump():
    os.makedirs("gpurun_out", exist_ok=True)
    with open("gpurun_out/parity_split.json", "w") as f:
        json.dump(_REPORT, f, indent=1, sort_keys=True)


def _engine(variant, batch=B):
    return gan_engine(variant, max_batch=batch, precision="split")


@pytest.mark.parametrize("case", ROW_VARIANTS + GP_VARIANTS)
def test_step1_every_output_within_1e3(case):
    fx = load_case("gan_" + case)
    eng = _engine(case)
    x = images_from_bits(fx)
    draws = unpack_draws(fx, "step1_")
    z1, z2 = draws[0], draws[-1]
    aux_o, aux_d = _aux_from(iter(draws[1:]), case)
    P = params_dict(gm_init_weights(GAN_SHAPES, 1234), np.float64)
    st = dict(LAMBDA=0.0, RHO=1e-6) if case == "fisher" else None
    if case == "fisher":
        eng.fisher_state(0.0, 1e-6)
    Ld = eng.d_grad(torch.from_numpy(x).cuda(), noise=torch.from_numpy(z1).cuda(), aux=aux_d).item()
    sc = eng.scores(2 * B).cpu().numpy()
    gD = [v.cpu().numpy() for v in eng.views(1, eng.grads[1])]
    # D hidden rows: real, fake, xhat (WGAN-GP keeps the x_hat rows only in mask form, in the U region of DHall)
    regions = [("Aall", 0, True), ("Aall", 1, True), ("DHall", 2)] if case == "wgp" else [0, 1, 2]
    with DeviceReluSides(eng, d_regions=regions, g_hidden=False) as sides_d:
        Lo, go, _ = R.gan_d_step(P, case, x.astype(np.float64), z1.astype(np.float64), aux_o, st)
    rep = {"D_loss_vs_golden": abs(Ld - float(fx["step1_D_loss"])) / max(abs(float(fx["step1_D_loss"])), 1e-3),
           "D_loss_vs_oracle": abs(Ld - Lo) / max(abs(Lo), 1e-3),
           "DX_score": _nrel(sc[:B], fx["step1_score_0"]), "DG_score": _nrel(sc[B:], fx["step1_score_1"])}
    for nme, g in zip(D_NAMES, gD):
        rep["grad_" + nme] = _nrel(g, go[nme])
    Lg = eng.g_grad(B, noise=torch.from_numpy(z2).cuda()).item()
    with DeviceReluSides(eng, d_regions=[1]) as sides_g:                         # the G step's D rows are the fake region
        Lgo, ggo, _ = R.gan_g_step(P, case, z2.astype(np.float64))
    rep["G_loss_vs_golden"] = abs(Lg - float(fx["step1_G_loss"])) / max(abs(float(fx["step1_G_loss"])), 1e-3)
    for nme, g in zip(G_NAMES, [v.cpu().numpy() for v in eng.views(0, eng.grads[0])]):
        rep["grad_" + nme] = _nrel(g, ggo[nme])
    rep["relu_units_at_boundary"] = sides_d.count + sides_g.count
    _REPORT["step1_" + case] = rep
    _dump()
    assert rep["relu_units_at_boundary"] <= 8, rep
    for k, v in rep.items():
        if k != "relu_units_at_boundary":
            assert v < TOL, (k, v, rep)


@pytest.mark.parametrize("case", ROW_VARIANTS + GP_VARIANTS)
def test_three_steps_losses_and_final_weights_within_1e3(case):
    import gm_b200
    fx = load_case("gan_" + case)
    kw = KW[case]
    eng = _engine(case)
    x = torch.from_numpy(images_from_bits(fx)).cuda()
    raw = iter(unpack_draws(fx))
    it = (torch.from_numpy(d).cuda() for d in raw)
    hpG = gm_b200.AdamHP.make(kw["G_lr"])
    hpD = gm_b200.AdamHP.make(kw["D_lr"], clamp=kw.get("clip", 0.0) or 0.0)
    if case == "fisher":
        eng.fisher_state(0.0, kw["RHO"])
    for _ in range(kw.get("G_init", 0)):
        eng.g_grad(B, noise=next(it))
        eng.apply(0, hpG)
    Dl, Gl = [], []
    for _ in range(STEPS):
        acc = []
        for _ in range(kw.get("D_steps", 1)):
            zd = next(it)
            acc.append(eng.d_grad(x, noise=zd, aux=_aux_from(raw, case)[1]).item())
            eng.apply(1, hpD)
        Dl.append(np.mean(acc))
        Gl.append(eng.g_grad(B, noise=next(it)).item())
        eng.apply(0, hpG)
    rep = {"D": [abs(a - b) / max(abs(b), 0.5) for a, b in zip(Dl, fx["D_loss"])],
           "G": [abs(a - b) / max(abs(b), 0.5) for a, b in zip(Gl, fx["G_loss"])]}
    finals = [v.cpu().numpy() for v in eng.views(0)] + [v.cpu().numpy() for v in eng.views(1)]
    for nme, w in zip(G_NAMES + D_NAMES, finals):
        key = "final_" + nme
        got = w.reshape(-1).astype(np.float64)
        if key in fx:
            ref = fx[key].astype(np.float64).reshape(-1)
        else:
            ref, got = fx[key + "__samp"].astype(np.float64), got[fx[key + "__idx"]]
        rep["w_" + nme] = float(np.linalg.norm(got - ref) / max(np.linalg.norm(ref), 1e-30))
    _REPORT["traj_" + case] = rep
    _dump()
    assert max(rep["D"]) < TOL and max(rep["G"]) < TOL, rep
    # Adam's first steps are sign-like (|update| = lr whatever the gradient's size), so an fp32-rounding-level
    # difference in a near-zero gradient entry can flip one weight by 2 lr; norm-relative that stays far below 1e-3
    for k, v in rep.items():
        if k.startswith("w_"):
            assert v < TOL, (k, v, rep)


def test_infogan_q_step_within_1e3():
    import gm_b200
    fx = load_case("gan_info")
    W = gm_init_weights(INFO_SHAPES, 1234)
    eng = gm_b200.InfoGanEngine(784, 400, 20, 10, 10, max_batch=B, precision="split")
    eng.load(0, [W["G.linear"][0], W["G.linear"][1], W["G.generate"][0], W["G.generate"][1]])
    eng.load(1, [W["D.linear"][0], W["D.linear"][1], W["D.discriminator"][0], W["D.discriminator"][1]])
    eng.load_q([W["Q.linear"][0], W["Q.linear"][1], W["Q.inference"][0], W["Q.inference"][1]])
    x = torch.from_numpy(images_from_bits(fx)).cuda()
    d1 = unpack_draws(fx, "step1_")
    P = {k.replace("D.discriminator", "D.discriminate"): v for k, v in params_dict(W, np.float64).items()}
    rep = {}
    rep["D_loss"] = abs(eng.d_grad(x, noise=torch.from_numpy(d1[0]).cuda()).item() - float(fx["step1_D_loss"])) / abs(float(fx["step1_D_loss"]))
    rep["G_loss"] = abs(eng.g_grad(B, noise=torch.from_numpy(d1[1]).cuda()).item() - float(fx["step1_G_loss"])) / abs(float(fx["step1_G_loss"]))
    rep["MI_loss"] = abs(eng.q_grad(B, torch.from_numpy(d1[2]).cuda()).item() - float(fx["step1_MI_loss"])) / abs(float(fx["step1_MI_loss"]))
    _, gq = R.info_q_step(P, d1[2].astype(np.float64))
    for nme, g in zip(G_NAMES, eng.views(0, eng.grads[0])):
        rep["grad_" + nme] = _nrel(g.cpu().numpy(), gq[nme])
    for nme, g in zip(["Q.linear.weight", "Q.linear.bias", "Q.inference.weight", "Q.inference.bias"], eng.q_views(eng.q_grads)):
        rep["grad_" + nme] = _nrel(g.cpu().numpy(), gq[nme])
    _REPORT["step1_info"] = rep
    _dump()
    for k, v in rep.items():
        assert v < TOL, (k, v, rep)


def test_began_steps_within_1e3():
    import gm_b200
    fx = load_case("gan_began")
    W = gm_init_weights(BEGAN_SHAPES, 1234)
    eng = gm_b200.GanEngine(784, 400, 20, max_batch=B, variant="began", precision="split")
    eng.load(0, [W["G.linear"][0], W["G.linear"][1], W["G.generate"][0], W["G.generate"][1]])
    eng.load(1, [W["D.encoder"][0], W["D.encoder"][1], W["D.decoder"][0], W["D.decoder"][1]])
    x = torch.from_numpy(images_from_bits(fx)).cuda()
    d1 = unpack_draws(fx, "step1_")
    P = params_dict(W, np.float64)
    eng.began_init(0.3, B)
    rep = {}
    Ld = eng.d_grad(x, noise=torch.from_numpy(d1[0]).cuda()).item()
    rep["D_loss"] = abs(Ld - float(fx["step1_D_loss"])) / abs(float(fx["step1_D_loss"]))
    _, ge, _, _ = R.began_d_step(P, images_from_bits(fx).astype(np.float64), d1[0].astype(np.float64), 0.3)
    for nme, g in zip(["D.encoder.weight", "D.encoder.bias", "D.decoder.weight", "D.decoder.bias"], eng.views(1, eng.grads[1])):
        rep["grad_" + nme] = _nrel(g.cpu().numpy(), ge[nme])
    Lg = eng.g_grad(B, noise=torch.from_numpy(d1[1]).cuda()).item()
    rep["G_loss"] = abs(Lg - float(fx["step1_G_loss"])) / abs(float(fx["step1_G_loss"]))
    _, gge = R.began_g_step(P, d1[1].astype(np.float64))
    for nme, g in zip(G_NAMES, eng.views(0, eng.grads[0])):
        rep["grad_" + nme] = _nrel(g.cpu().numpy(), gge[nme])
    _REPORT["step1_began"] = rep
    _dump()
    for k, v in rep.items():
        # sign(r - x) is discontinuous: where |r - x| is at fp32 rounding level a single sign can differ from the
        # float64 oracle; norm-relative that stays below the bound (measured value in the report)
        assert v < TOL, (k, v, rep)


def test_vae_step_and_trajectory_within_1e3():
    import gm_b200
    fx = load_case("vae")
    eng = gm_b200.VaeEngine(784, 400, 20, max_batch=B, precision="split")
    Wt = gm_init_weights(VAE_SHAPES, 4321)
    t = {}
    for k, (w, b) in Wt.items():
        t[k + ".weight"], t[k + ".bias"] = w, b
    eng.load(t)
    x = images_from_bits(fx)
    eps = unpack_draws(fx, "step1_")[0]
    P = params_dict(Wt, np.float64)
    _, _, g_o, _ = R.vae_step(P, x.astype(np.float64), eps.astype(np.float64))
    xd = torch.from_numpy(x).cuda()
    ls = eng.grad(xd, eps=torch.from_numpy(eps).cuda()).cpu().numpy()
    gv = {k: v.cpu().numpy() for k, v in eng.views(eng.grads).items()}
    rep = {"recon_vs_golden": float(abs(ls[0] - float(fx["step1_recon"])) / float(fx["step1_recon"])),
           "kl_vs_golden": float(abs(ls[1] - float(fx["step1_kl"])) / float(fx["step1_kl"]))}
    for k in g_o:
        rep["grad_" + k] = _nrel(gv[k], g_o[k])
    draws = unpack_draws(fx)
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    eng.reset_optimizer()
    Rl, Kl = [], []
    for s in range(STEPS):
        l2 = eng.grad(xd, eps=torch.from_numpy(draws[s]).cuda()).cpu().numpy()
        eng.apply(hp)
        Rl.append(l2[0])
        Kl.append(l2[1])
    rep["recon_traj"] = [float(abs(a - b) / b) for a, b in zip(Rl, fx["recon_loss"])]
    rep["kl_traj"] = [float(abs(a - b) / b) for a, b in zip(Kl, fx["kl_loss"])]
    _REPORT["vae"] = rep
    _dump()
    for k, v in rep.items():
        assert (max(v) if isinstance(v, list) else v) < TOL, (k, v, rep)


def test_split_and_bf16_engines_agree_on_bf16_scale():
    """the two operand modes are the same algorithm: their gradients differ by the bf16 operand rounding only"""
    import gm_b200
    fx = load_case("gan_ns")
    x = torch.from_numpy(images_from_bits(fx)).cuda()
    z = torch.from_numpy(unpack_draws(fx, "step1_")[0]).cuda()
    eng_s = _engine("ns")
    eng_b = gm_b200.GanEngine(784, 400, 20, max_batch=B, variant="ns")
    for net in (0, 1):
        eng_b.load(net, eng_s.views(net))
    ls, lb = eng_s.d_grad(x, noise=z).item(), eng_b.d_grad(x, noise=z).item()
    assert abs(ls - lb) < 1e-3 * abs(ls)
    assert 1e-5 < _nrel(eng_b.grads[1].cpu().numpy(), eng_s.grads[1].cpu().numpy()) < 6e-2


def _torch_step_grads(eng, x, zd, zg, variant, consts, aux=None):
    """fp32 autograd (TF32 off) of the reference's formulas with explicit loss constants -> (Ld, gD flat, Lg, gG flat)."""
    torch.backends.cuda.matmul.allow_tf32 = False
    Wg1, bg1, Wg2, bg2 = [t.clone().requires_grad_() for t in eng.views(0)]
    Wd1, bd1, Wd2, bd2 = [t.clone().requires_grad_() for t in eng.views(1)]
    relu_out = variant == "wgp"

    def Gf(zz):
        return torch.sigmoid(torch.relu(zz @ Wg1.t() + bg1) @ Wg2.t() + bg2)

    def Df(xx):
        s = torch.relu(xx @ Wd1.t() + bd1) @ Wd2.t() + bd2
        return torch.relu(s) if relu_out else torch.sigmoid(s)
    n = x.shape[0]
    fake = Gf(zd)
    DX, DG = Df(x), Df(fake)
    if variant == "ls":                                                          # src/ls_gan.py:192-193,213
        Ld = 0.5 * torch.mean((DX - consts["b"]) ** 2) + 0.5 * torch.mean((DG - consts["a"]) ** 2)
    elif variant == "ns":
        Ld = -torch.mean(torch.log(DX + 1e-8) + torch.log(1 - DG + 1e-8))
    else:
        if variant == "wgp":                                                     # src/w_gp_gan.py:197-218
            eps = aux.view(-1, 1)
            xh = (eps * x + (1 - eps) * fake.detach()).requires_grad_()
            base = torch.mean(DG) - torch.mean(DX)
        else:                                                                    # src/dra_gan.py:195-220
            delta, u = aux[:n].view(-1, 1), aux[n:].view(n, -1)
            xh = (delta * x + (1 - delta) * (x + consts["C"] * x.std() * u)).requires_grad_()
            base = -torch.mean(torch.log(DX + 1e-8) + torch.log(1 - DG + 1e-8))
        gr = torch.autograd.grad(Df(xh), xh, torch.ones(n, 1, device="cuda"), create_graph=True, retain_graph=True)[0]
        Ld = base + consts["LAMBDA"] * torch.mean((gr.norm(2, dim=1) - consts.get("K", 1.0)) ** 2)
    gD = torch.cat([t.reshape(-1) for t in torch.autograd.grad(Ld, [Wd1, bd1, Wd2, bd2])])
    DGg = Df(Gf(zg))
    if variant == "ls":
        Lg = 0.5 * torch.mean((DGg - consts["c"]) ** 2)
    elif variant == "wgp":
        Lg = -torch.mean(DGg)
    else:
        Lg = -torch.mean(torch.log(DGg + 1e-8))
    gG = torch.cat([t.reshape(-1) for t in torch.autograd.grad(Lg, [Wg1, bg1, Wg2, bg2])])
    return Ld.item(), gD, Lg.item(), gG


@pytest.mark.parametrize("case", ["ls_abc", "wgp_lambda5", "dra_lkc", "ns_h256_z128"])
def test_loss_constants_and_notebook_shapes(case):
    """The loss constants the reference passes as train_D / train_G kwargs (a, b, c of src/ls_gan.py:173,197; LAMBDA of
    src/w_gp_gan.py:177; LAMBDA, K, C of src/dra_gan.py:174) at non-default values, and the shapes of notebooks 11 / 13 / 14
    (hidden 256, z 128): losses and flat D / G gradients within 1e-3 of fp32 autograd (split operand mode, batch 128)."""
    import gm_b200
    import torch.nn as nn
    variant = case.split("_")[0]
    Hh, Zz = (256, 128) if case == "ns_h256_z128" else (400, 20)
    n = 128
    eng = gm_b200.GanEngine(784, Hh, Zz, max_batch=n, variant=variant, d_out_act="relu" if variant == "wgp" else "sigmoid",
                            precision="split")
    torch.manual_seed(4321)
    g1, g2, d1, d2 = nn.Linear(Zz, Hh), nn.Linear(Hh, 784), nn.Linear(784, Hh), nn.Linear(Hh, 1)
    eng.load(0, [g1.weight.data, g1.bias.data, g2.weight.data, g2.bias.data])
    eng.load(1, [d1.weight.data, d1.bias.data, d2.weight.data, d2.bias.data])
    g = torch.Generator(device="cuda").manual_seed(17)
    x = (torch.rand(n, 784, device="cuda", generator=g) < 0.1307).float()
    zd, zg = torch.randn(n, Zz, device="cuda", generator=g), torch.randn(n, Zz, device="cuda", generator=g)
    consts, aux = {}, None
    if case == "ls_abc":
        consts = dict(a=0.1, b=0.9, c=0.8)
        eng.set_loss_consts(ls_a=0.1, ls_b=0.9, ls_c=0.8)
    elif case == "wgp_lambda5":
        consts = dict(LAMBDA=5.0)
        eng.set_loss_consts(gp_lambda=5.0)
        aux = torch.rand(n, device="cuda", generator=g)
    elif case == "dra_lkc":
        consts = dict(LAMBDA=5.0, K=0.7, C=0.5)
        eng.set_loss_consts(gp_lambda=5.0, gp_k=0.7, dra_c=0.5)
        aux = torch.cat([torch.rand(n, device="cuda", generator=g), torch.rand(n * 784, device="cuda", generator=g)])
    Ld_ref, gD, Lg_ref, gG = _torch_step_grads(eng, x, zd, zg, variant, consts, aux)
    Ld = eng.d_grad(x, noise=zd, aux=aux).item()
    flatD = eng.grads[1].clone()
    Lg = eng.g_grad(n, noise=zg).item()
    flatG = eng.grads[0].clone()
    rep = {"D_loss": abs(Ld - Ld_ref) / max(abs(Ld_ref), 0.5), "G_loss": abs(Lg - Lg_ref) / max(abs(Lg_ref), 0.5),
           "gD": _nrel(flatD.cpu().numpy(), gD.cpu().numpy()), "gG": _nrel(flatG.cpu().numpy(), gG.cpu().numpy())}
    _REPORT["consts_" + case] = rep
    _dump()
    for k, v in rep.items():
        assert v < TOL, (k, v, rep)
