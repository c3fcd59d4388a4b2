"""The VAE on the DCGAN conv path on the GPU: the SSE-through-sigmoid loss (gm_sse_sigmoid_rows), the latent kernels
(gm_vae_latent_rows, gm_vae_dlatent_rows) and inference-mode BatchNorm (gm_bn_forward_eval) against float64 torch, one
vae_grad against fp32 autograd at the CUDA path's bf16 storage points (tests/dcgan_vae_oracle.py), the backward restated in
float64 at the device's own stored tensors, Adam with weight decay against torch.optim.Adam, descent, the train / eval
BatchNorm modes and the dc_vae drop-in on the reference's driver lines.  With GM_PARITY_DIR set, the measured errors are
written to $GM_PARITY_DIR/parity_dcgan_vae.json."""
import os
import tempfile

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import dcgan_harness as H
import dcgan_vae_oracle as VO
from dcgan_harness import nrel
from oracle import dcgan_torch as O

pytestmark = pytest.mark.gpu
_REPORT = H.Report("dcgan_vae")
CH = 3
BF = 2.0 ** -8                                   # one bf16 rounding, relative


def _lib():
    from gm_b200 import _lib
    return _lib, _lib.ctx()


def _engine(hd=16, z=20, wstd=0.05, seed=11):
    """DcganEngine(variant="vae") with N(0, wstd) conv weights (as dcgan_harness.setup) and the oracle encoder and decoder
    holding the same weights at the bf16 storage points"""
    import gm_b200
    eng = gm_b200.DcganEngine(hidden_dim=hd, z_dim=z, variant="vae")
    g = torch.Generator().manual_seed(seed)
    for net in eng.nets():
        for name in net.names:
            if name.startswith("l"):
                net.view(name).copy_(wstd * torch.randn(net.view(name).shape, generator=g))
    eng.zero_padding()
    for net in eng.nets():
        net.refresh()
    E, G = VO.Encoder(hd, z), VO.Decoder(hd, z)
    VO.load_from_engine_weights(E, G, eng.torch_weights())
    for m in (E, G):
        m.train()
        m.q = staticmethod(O.bf16_points)
    return eng, E, G, g


# ------------------------------------------------------------------ kernel units
def test_sse_sigmoid_rows_match_float64():
    """non-binary targets, 5 images: the sum to double precision, the gradient to one bf16 rounding"""
    L, h = _lib()
    n, cols, scale = 5, 4096 * CH, 0.75
    g = torch.Generator(device="cuda").manual_seed(2)
    out = torch.sigmoid(2 * torch.randn(n, cols, device="cuda", generator=g)).to(torch.bfloat16)
    x = torch.rand(n, cols, device="cuda", generator=g).to(torch.bfloat16)
    grad = torch.full((n, cols), 9.0, device="cuda", dtype=torch.bfloat16)
    total = torch.zeros(1, device="cuda", dtype=torch.float64)
    L.check(h, L.lib().gm_sse_sigmoid_rows(h, L._ptr(out), L._ptr(x), n, cols, scale, L._ptr(grad), L._ptr(total), L._stream()))
    o64, x64 = out.double().cpu(), x.double().cpu()
    want = float(((x64 - o64) ** 2).sum())
    ref = VO.dpre(o64, x64, scale)
    err = (grad.double().cpu() - ref).abs()
    rep = {"sum_rel": abs(float(total) - want) / want, "grad_rel_max": float((err / ref.abs().clamp_min(1e-30))[ref.abs() > 1e-30].max()),
           "grad_abs_at_zero": float(err[ref.abs() <= 1e-30].max()) if bool((ref.abs() <= 1e-30).any()) else 0.0}
    _REPORT.add("sse_rows", rep)
    assert rep["sum_rel"] < 1e-12 and rep["grad_rel_max"] <= BF and rep["grad_abs_at_zero"] == 0.0, rep


def _latent(mulv, n, z, eps=None, seed=0, stream=0, ldz=None):
    L, h = _lib()
    ldz = ldz or (z + 1 + 7) // 8 * 8
    rows = torch.full((n, ldz), 7.0, device="cuda", dtype=torch.bfloat16)          # garbage: the kernel writes every column
    eps_out = torch.full((n, z), 7.0, device="cuda")
    kl = torch.zeros(1, device="cuda", dtype=torch.float64)
    L.check(h, L.lib().gm_vae_latent_rows(h, L._ptr(mulv), mulv.stride(0), L._ptr(eps), L._ptr(eps_out), L._ptr(rows), ldz, n, z, seed, stream,
                                          L._ptr(kl), L._stream()))
    return rows, eps_out, kl


def test_vae_latent_rows_with_a_caller_eps():
    """rows = bf16(mu + eps e^(lv/2)), the ones column and zero padding in place, eps_out = eps, KL against float64"""
    n, z, mp = 37, 20, 48
    g = torch.Generator(device="cuda").manual_seed(5)
    mulv = torch.randn(n, mp, device="cuda", generator=g)
    mulv[:, z:2 * z] *= 0.5
    eps = torch.randn(n, z, device="cuda", generator=g)
    rows, eps_out, kl = _latent(mulv, n, z, eps)
    m64, l64, e64 = mulv[:, :z].double().cpu(), mulv[:, z:2 * z].double().cpu(), eps.double().cpu()
    ref = VO.reparameterize(m64, l64, e64)
    # relative to one bf16 rounding, with a floor for the few values where mu and eps e^(lv/2) cancel
    rep = {"z_rel_max": float(((rows[:, :z].double().cpu() - ref).abs() / (ref.abs() + 1e-4)).max()),
           "kl_rel": abs(float(kl) - float(VO.kl_divergence(m64, l64))) / float(VO.kl_divergence(m64, l64))}
    _REPORT.add("latent_caller_eps", rep)
    assert rep["z_rel_max"] <= BF and rep["kl_rel"] < 1e-10, rep
    assert torch.equal(eps_out, eps)
    assert bool((rows[:, z] == 1).all()) and bool((rows[:, z + 1:] == 0).all())


def test_vae_latent_rows_philox():
    """Philox eps: N(0, 1) moments, the same (seed, step) gives identical bits, another step differs, eps_out holds the draws"""
    n, z = 1 << 15, 100
    mulv = torch.zeros(n, 208, device="cuda")                                      # mu = 0, log_var = 0: z = eps
    rows, eps, _ = _latent(mulv, n, z, seed=77, stream=3)
    rows2, eps2, _ = _latent(mulv, n, z, seed=77, stream=3)
    _, eps3, _ = _latent(mulv, n, z, seed=77, stream=4)
    assert torch.equal(rows, rows2) and torch.equal(eps, eps2)
    assert float((eps3 != eps).float().mean()) > 0.99
    assert torch.equal(rows[:, :z], eps.to(torch.bfloat16))
    e = eps.double()
    N = e.numel()
    rep = {"mean_se": abs(float(e.mean())) / (1 / N) ** 0.5, "var_se": abs(float(e.var()) - 1) / (2 / N) ** 0.5,
           "col_mean_se_max": float(e.mean(0).abs().max()) * n ** 0.5}
    _REPORT.add("latent_philox", rep)
    assert rep["mean_se"] < 5 and rep["var_se"] < 5 and rep["col_mean_se_max"] < 5, rep


def test_vae_dlatent_rows_match_float64():
    L, h = _lib()
    n, z, mp = 37, 20, 48
    g = torch.Generator(device="cuda").manual_seed(6)
    mulv = torch.randn(n, mp, device="cuda", generator=g)
    dz = torch.randn(n, z, device="cuda", generator=g) * 3
    eps = torch.randn(n, z, device="cuda", generator=g)
    out = torch.full((n, mp), 9.0, device="cuda", dtype=torch.bfloat16)
    L.check(h, L.lib().gm_vae_dlatent_rows(h, L._ptr(mulv), mp, L._ptr(dz), z, L._ptr(eps), L._ptr(out), mp, n, z, 0.5, L._stream()))
    dmu, dlv = VO.dlatent(mulv[:, :z].double().cpu(), mulv[:, z:2 * z].double().cpu(), eps.double().cpu(), dz.double().cpu(), 0.5)
    ref = torch.cat([dmu, dlv], 1)
    got = out.double().cpu()
    rel = float(((got[:, :2 * z] - ref).abs() / (ref.abs() + 1e-4)).max())          # floor: the two dlv terms may cancel
    _REPORT.add("dlatent", {"rel_max": rel})
    assert rel <= BF, rel
    assert bool((got[:, 2 * z:] == 0).all())


@pytest.mark.parametrize("act", [1, 2])
def test_bn_forward_eval_matches_torch(act):
    """gm_bn_forward_eval == F.batch_norm(training=False) + ReLU / LeakyReLU(0.2) to one bf16 rounding; the running
    statistics are read, not changed"""
    L, h = _lib()
    rows, C = 3000, 64
    g = torch.Generator(device="cuda").manual_seed(act)
    x = (torch.randn(rows, C, device="cuda", generator=g) * 2 + 0.5).to(torch.bfloat16)
    gamma, beta = 1 + 0.1 * torch.randn(C, device="cuda", generator=g), 0.1 * torch.randn(C, device="cuda", generator=g)
    running = torch.stack([0.3 * torch.randn(C, device="cuda", generator=g), 0.5 + torch.rand(C, device="cuda", generator=g)])
    before = running.clone()
    y = torch.empty(rows, C, device="cuda", dtype=torch.bfloat16)
    L.check(h, L.lib().gm_bn_forward_eval(h, L._ptr(x), rows, C, C, L._ptr(gamma), L._ptr(beta), L._ptr(running), 1e-5, act, 0.2, L._ptr(y), C,
                                          L._stream()))
    ref = F.batch_norm(x.double(), running[0].double(), running[1].double(), gamma.double(), beta.double(), training=False, eps=1e-5)
    ref = torch.relu(ref) if act == 1 else F.leaky_relu(ref, 0.2)
    err = float(((y.double() - ref).abs() / (ref.abs() + 1e-3)).max())
    _REPORT.add("bn_eval_act%d" % act, {"rel_max": err})
    assert err <= 2 * BF, err
    assert torch.equal(running, before)


# ------------------------------------------------------------------ one vae_grad (hidden 16, batch 8)
def test_vae_grad_matches_the_oracle():
    # z = 30: the fp32 dL/dz rows and G's l1 weight-gradient rows start 120 bytes apart (not on 16 bytes)
    n = 8
    for z in (20, 30):
        eng, E, G, g = _engine(z=z)
        x = (torch.rand(n, CH * 4096, generator=g) < 0.3).float()
        eps = torch.randn(n, z, generator=g)
        recon_ref, kl_ref = VO.compute_batch(E, G, x, eps)
        params = list(E.parameters()) + list(G.parameters())
        ref = torch.autograd.grad(recon_ref + kl_ref, params)
        losses = eng.vae_grad(eng.stage_images(x.cuda()), n, eps=eps.cuda()).tolist()
        rep = {"recon": abs(losses[0] - recon_ref.item()) / recon_ref.item(), "kl": abs(losses[1] - kl_ref.item()) / kl_ref.item()}
        tg = eng.torch_grads()
        names = ["D." + k for k, _ in E.named_parameters()] + ["G." + k for k, _ in G.named_parameters()]
        for name, r in zip(names, ref):
            rep["grad_" + name] = nrel(tg[name], r)
        _REPORT.add("step" + ("" if z == 20 else "_z%d" % z), rep)
        assert float(eng.D.view("l5.weight", eng.D.grads)[2 * z:].abs().max()) == 0.0               # the head's padded rows
        # the bounds of the BEGAN and InfoGAN oracle comparisons (DESIGN.md §6b): device and oracle evaluate at slightly different
        # forward points (their bf16 roundings differ where the accumulation orders do), a few per mille of the (Leaky)ReLU units
        # take the other slope, and 7 BatchNorm layers over 8 images amplify that; the arithmetic itself is held to 2 % by
        # test_vae_backward_matches_float64_at_the_device_forward_points
        assert rep["recon"] < 5e-3 and rep["kl"] < 2e-2, rep
        for k, v in rep.items():
            if k.startswith("grad"):
                assert v < 0.20, (k, v, rep)


def test_vae_backward_matches_float64_at_the_device_forward_points():
    """The composition vae_grad runs - closed-form dpre, the decoder backward to dz, (dmu, dlv), the encoder backward - restated
    in float64 with torch.nn.grad at the device's OWN stored activations, masks and BatchNorm inputs (the BEGAN test's
    restatement of the two stacks), so that what remains is the bf16 rounding of the device's backward tensors."""
    from test_dcgan_began_gpu import _at, _stack_backward, _trunk_backward, _tw
    n, z = 8, 20
    eng, _, _, g = _engine()
    x = (torch.rand(n, CH * 4096, generator=g) < 0.3).float()
    eng.vae_grad(eng.stage_images(x.cuda()), n, eps=torch.randn(n, z, generator=g).cuda())
    s = eng.vae_saved_
    tw = _tw(eng)
    w = {tag: {k[2:]: v for k, v in tw.items() if k.startswith(tag + ".")} for tag in "GD"}
    rep = {}
    out, x64 = _at(s["out"], 64, CH), _at(eng.stage_images(x.cuda()), 64, CH)
    dp = VO.dpre(out, x64)
    rep["dpre"] = nrel(_at(s["dpre"], 64, CH), dp)
    gref, dz = _stack_backward(eng, s["svd"], dp, w["G"], "")
    rep["dz"] = nrel(s["dz"], dz)
    mulv, eps = s["mulv"].double().cpu(), s["eps"].double().cpu()
    dmu, dlv = VO.dlatent(mulv[:, :z], mulv[:, z:2 * z], eps, dz)
    rep["dlatent"] = nrel(s["dml"][:, :2 * z], torch.cat([dmu, dlv], 1))
    eref, _ = _trunk_backward(eng, s["sve"], torch.cat([dmu, dlv], 1), w["D"], "")
    tg = eng.torch_grads()
    for name, r in gref.items():
        rep["G." + name] = nrel(tg["G." + name], r)
    for name, r in eref.items():
        rep["D." + name] = nrel(tg["D." + name], r)
    _REPORT.add("float64_at_device_points", rep)
    assert len([k for k in rep if k.startswith("G.")]) == 13 and len([k for k in rep if k.startswith("D.")]) == 11
    for k, v in rep.items():
        assert v < 0.02, (k, v, rep)


def test_apply_is_one_adam_with_weight_decay_over_all_parameters():
    """apply(hp) == torch.optim.Adam(all parameters, lr, weight_decay=1e-5) for two steps on given gradients"""
    import gm_b200
    eng, _, _, _ = _engine()
    g = torch.Generator(device="cuda").manual_seed(9)
    grads = [(torch.randn(eng.G.total, device="cuda", generator=g), torch.randn(eng.D.total, device="cuda", generator=g)) for _ in range(2)]
    pG, pD = eng.G.params.clone(), eng.D.params.clone()
    lr = 1e-3
    hp = gm_b200.AdamHP.make(lr, weight_decay=1e-5)
    tG, tD = pG.clone().requires_grad_(), pD.clone().requires_grad_()
    opt = torch.optim.Adam([tD, tG], lr=lr, weight_decay=1e-5)
    for gG, gD in grads:
        eng.G.grads.copy_(gG)
        eng.D.grads.copy_(gD)
        eng.apply(hp)
        tG.grad, tD.grad = gG.clone(), gD.clone()
        opt.step()
    rep = {"G": nrel(eng.G.params - pG, tG.detach() - pG), "D": nrel(eng.D.params - pD, tD.detach() - pD)}
    _REPORT.add("apply", rep)
    assert rep["G"] < 1e-5 and rep["D"] < 1e-5, rep
    assert eng.G.step == 2 and eng.D.step == 2


def test_vae_steps_lower_the_loss():
    """about 20 steps at hidden 16 on one binarised batch lower recon + KL"""
    import gm_b200
    n = 16
    eng, _, _, g = _engine()
    x = eng.stage_images((torch.rand(n, CH * 4096, generator=g) < 0.3).float().cuda())
    hp = gm_b200.AdamHP.make(1e-3, weight_decay=1e-5)
    losses = []
    for s in range(20):
        losses.append(float(eng.vae_grad(x, n, seed=5, step=s).sum()))
        eng.apply(hp)
    _REPORT.add("descent", {"first": losses[0], "last": losses[-1]})
    assert all(np.isfinite(losses)) and losses[-1] < 0.9 * losses[0], losses


def test_vae_forward_batchnorm_modes():
    """train=False equals the oracle in eval() mode and leaves the running statistics unchanged; train=True takes batch
    statistics and updates the running statistics as torch's training-mode forward does"""
    n, z = 8, 20
    eng, E, G, g = _engine()
    for r in list(eng.run_G.values()) + list(eng.run_D.values()):                # non-trivial running statistics
        r[0].copy_(0.1 * torch.randn(r.shape[1], generator=g))
        r[1].copy_(0.5 + torch.rand(r.shape[1], generator=g))
    for t, mod in (("G", G), ("D", E)):
        for i, r in (eng.run_G if t == "G" else eng.run_D).items():
            bn = getattr(mod, "bn%d" % (i + 1))
            bn.running_mean.copy_(r[0].cpu()); bn.running_var.copy_(r[1].cpu())
    x = (torch.rand(n, CH * 4096, generator=g) < 0.3).float()
    eps = torch.randn(n, z, generator=g)
    runs = lambda: [r.clone() for r in list(eng.run_G.values()) + list(eng.run_D.values())]    # noqa: E731
    before = runs()
    rec, mu, lv, losses = eng.vae_forward(eng.stage_images(x.cuda()), n, eps=eps.cuda(), train=False)
    E.eval(); G.eval()
    with torch.no_grad():
        mu_r, lv_r = E(x)
        out_r = G(VO.reparameterize(mu_r, lv_r, eps))
    rep = {"eval_mu": nrel(mu, mu_r), "eval_lv": nrel(lv, lv_r), "eval_out": nrel(rec, out_r)}
    assert all(torch.equal(a, b) for a, b in zip(runs(), before))
    E.train(); G.train()
    rec, mu, lv, _ = eng.vae_forward(eng.stage_images(x.cuda()), n, eps=eps.cuda(), train=True)
    with torch.no_grad():
        mu_r, lv_r = E(x)
        out_r = G(VO.reparameterize(mu_r, lv_r, eps))
    rep.update({"train_mu": nrel(mu, mu_r), "train_out": nrel(rec, out_r)})
    for t, mod in (("G", G), ("D", E)):
        for i, r in (eng.run_G if t == "G" else eng.run_D).items():
            bn = getattr(mod, "bn%d" % (i + 1))
            rep["run_%s%d" % (t, i)] = max(nrel(r[0], bn.running_mean), nrel(r[1], bn.running_var))
    _REPORT.add("forward_modes", rep)
    assert not all(torch.equal(a, b) for a, b in zip(runs(), before))
    # about ten times the measured values (DESIGN.md §6b): a wrong momentum or variance convention is far outside them
    bound = {"eval": 4e-3, "run": 2e-3, "train": 2.5e-2}
    for k, v in rep.items():
        assert v < bound[k.split("_")[0]], (k, v, rep)


def test_compute_batch_loop_keeps_the_running_statistics():
    """the reference's loop body in a user's own loop - compute_batch, (recon + kl).backward(), torch.optim.Adam - three
    times: the modules' running statistics follow torch's training-mode forwards (the oracle run at the same weights,
    batches and eps), the saved checkpoint holds them, and a model.eval() forward normalises with them"""
    import dc_vae as M
    n, z, hd = 8, 20, 16
    g = torch.Generator().manual_seed(4)
    torch.manual_seed(5)
    model = M.DCVAE(hidden_dim=hd, z_dim=z)
    it = [(torch.zeros(2, 3, 64, 64), torch.zeros(2))]
    tr = M.DCVAETrainer(model, it, it, it)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3, weight_decay=1e-5)
    E, G = VO.Encoder(hd, z), VO.Decoder(hd, z)
    for m in (E, G):
        m.q = staticmethod(O.bf16_points)

    def weights_to_oracle():
        sd = model.state_dict()
        with torch.no_grad():
            for name, p in E.named_parameters():
                p.copy_(torch.cat([sd["encoder.mu.weight"], sd["encoder.log_var.weight"]]) if name == "l5.weight" else sd["encoder." + name])
            for name, p in G.named_parameters():
                p.copy_(sd["decoder." + name])

    model.train(); E.train(); G.train()
    for _ in range(3):
        x = (torch.rand(n, CH * 4096, generator=g) < 0.3).float()
        weights_to_oracle()
        recon, kl = tr.compute_batch((x.view(n, CH, 64, 64), torch.zeros(n)))
        with torch.no_grad():
            VO.compute_batch(E, G, x, tr._engine.vae_saved_["eps"].cpu())                 # torch's running-statistics update
        opt.zero_grad()
        (recon + kl).backward()
        opt.step()
    rep = {}
    sd = model.state_dict()
    for tag, ref in (("encoder", E), ("decoder", G)):
        for name, buf in ref.named_buffers():
            if name.endswith(("running_mean", "running_var")):
                rep["%s.%s" % (tag, name)] = nrel(sd["%s.%s" % (tag, name)], buf)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        tr.save_model(path)
        saved = torch.load(path)
    for k in rep:
        assert torch.equal(saved[k], sd[k]), k
    model.eval(); E.eval(); G.eval()
    weights_to_oracle()
    x = (torch.rand(n, CH * 4096, generator=g) < 0.3).float()
    zz = torch.randn(n, z, generator=g)
    mu, lv = model.encoder(x)
    with torch.no_grad():
        mu_r, lv_r = E(x)
        out_r = G(zz)
    rep.update({"eval_mu": nrel(mu, mu_r), "eval_lv": nrel(lv, lv_r), "eval_out": nrel(model.decoder(zz), out_r)})
    _REPORT.add("compute_batch_loop", rep)
    assert len(rep) == 2 * 7 + 3
    # measured: running statistics within 2.2e-3 (decoder.bn1's running mean, the mean over the batch of a conv of z, a
    # vector near zero whose norm-relative error the bf16 rounding of z inflates; the others 1e-4 or less), eval forward
    # within 9.5e-4.  Statistics left at their previous values would be off by about 1.
    for k, v in rep.items():
        assert v < (5e-3 if k.startswith("eval") else 1e-2), (k, v, rep)


def test_engine_arguments():
    import gm_b200
    from gm_b200 import GmError
    for kw in (dict(d_out_act="sigmoid"), dict(d_out_act="none"), dict(embed_dim=8), dict(disc_dim=4), dict(cont_dim=2)):
        with pytest.raises(GmError):
            gm_b200.DcganEngine(hidden_dim=16, variant="vae", **kw)
    eng = gm_b200.DcganEngine(hidden_dim=16, z_dim=20, variant="vae")
    assert eng.mp == 48 and eng.D.shapes["l5.weight"] == (48, 16 * 128) and eng.G.shapes["l1.weight"] == (16 * 128, 20)
    assert tuple(eng.torch_weights()["D.l5.weight"].shape) == (40, 128, 4, 4)
    for call in (lambda: eng.d_grad(torch.zeros(4 * 4096, 3, device="cuda", dtype=torch.bfloat16), 4), lambda: eng.g_grad(4),
                 lambda: eng.q_grad(4)):
        with pytest.raises(GmError):
            call()
    ns = gm_b200.DcganEngine(hidden_dim=16)
    for call in (lambda: ns.vae_grad(torch.zeros(4 * 4096, 3, device="cuda", dtype=torch.bfloat16), 4), lambda: ns.encode(torch.zeros(1, 12288)),
                 lambda: ns.decode(torch.zeros(1, 100))):
        with pytest.raises(GmError):
            call()


# ------------------------------------------------------------------ the drop-in on the reference's driver lines
def test_dc_vae_runs_the_reference_driver_code(capsys):
    import dc_vae as M
    g = torch.Generator().manual_seed(0)
    imgs = (torch.rand(64, 3, 64, 64, generator=g) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(64)), batch_size=16, shuffle=True)
    torch.manual_seed(3)
    model = M.DCVAE(image_size=64 * 64 * 3, hidden_dim=16, z_dim=20)
    before = {k: v.clone() for k, v in model.state_dict().items()}
    trainer = M.DCVAETrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=2, lr=1e-3, weight_decay=1e-5)
    lines = [ln for ln in capsys.readouterr().out.splitlines() if ln.startswith("Epoch[")]
    assert len(lines) == 2 and all("Reconst Loss: " in ln and "Val Loss: " in ln for ln in lines), lines
    assert len(trainer.recon_loss) == 8 and len(trainer.kl_loss) == 8 and all(np.isfinite(trainer.recon_loss + trainer.kl_loss))
    after = model.state_dict()
    assert all(not torch.equal(before[k], after[k]) for k in before if k.endswith("weight") and ".bn" not in k)
    assert not torch.equal(before["encoder.bn2.running_mean"], after["encoder.bn2.running_mean"])
    # best_model: a detached copy that evaluates on its own engine
    best = trainer.best_model
    assert best is not model and best._owner is None and best.training is False
    x8 = imgs[:8].reshape(8, -1)
    out, mu, lv = best(x8)
    assert out.shape == (8, 3 * 64 * 64) and mu.shape == (8, 20) and lv.shape == (8, 20) and bool(torch.isfinite(out).all())
    assert float(out.min()) >= 0 and float(out.max()) <= 1
    mub, lvb = best.encoder(x8)
    assert mub.shape == (8, 20) and bool(torch.isfinite(mub).all()) and bool(torch.isfinite(lvb).all())
    model.eval()
    assert trainer.sample_images(num_images=4).shape == (4, 3, 64, 64)
    assert len(trainer.sample_interpolated_images()) == 20
    assert trainer.reconstruct_images(imgs[:4], 0).shape == (4, 3, 64, 64)
    assert np.isfinite(trainer.evaluate(loader))
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "model.ckpt")
        trainer.save_model(path)
        model2 = M.DCVAE(image_size=64 * 64 * 3, hidden_dim=16, z_dim=20)
        tr2 = M.DCVAETrainer(model2, loader, loader, loader)
        tr2.load_model(path)
        assert list(model2.state_dict()) == list(model.state_dict())
        for k, v in model.state_dict().items():
            assert torch.equal(model2.state_dict()[k], v), k
        model2.eval()
        zz = torch.randn(4, 20)
        assert nrel(model2.decoder(zz), model.decoder(zz)) < 1e-6
    # the loop body: (recon + kl).backward() puts the engine's gradients on .grad
    model.train()
    model.zero_grad()
    recon, kl = trainer.compute_batch((imgs[:16], torch.zeros(16)))
    (recon + kl).backward()
    eng = trainer._engine
    tg = trainer._torch_tensors(grads=True)
    for k, p in model.named_parameters():
        assert p.grad is not None and p.grad.shape == p.shape, k
        assert torch.equal(p.grad.cpu(), tg["%s.%s" % ("D" if k.startswith("encoder.") else "G", k.split(".", 1)[1])].cpu()), k
    assert float(model.encoder.mu.weight.grad.abs().sum()) > 0 and float(model.decoder.l1.weight.grad.abs().sum()) > 0
    assert np.isfinite(recon.item()) and np.isfinite(kl.item()) and eng.variant == "vae"
