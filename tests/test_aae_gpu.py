"""Adversarial autoencoder on the GPU: each phase of the fused step (gm_aae_recon_grad, gm_aae_d_grad, gm_aae_g_grad) and
the three Adams against the float64 oracle (tests/aae_oracle.py) at its bf16 points, the reconstruction phase against the
BIR-VAE engine with eps_std = 0 and lam = 0 bit for bit, the device prior draw, the resident draw, a user-written
train_D / train_G / compute_batch against float64 torch autograd, the per-call latent D's errors, AAETrainer.train, and
the C ABI's refusals and launch ledger.

Bounds are test_cvae_gpu.py's: losses within 1e-3 relative; gradients within 3e-3 norm-relative of the oracle evaluated
at the engine's own bf16 storage points and at the parameters the engine holds when the phase runs (the remaining error
is the fp32 accumulation order of the GEMMs and split-K partials).  Each Adam is checked against a float64 Adam applied
to the gradient the engine produced, to 1e-6 absolute (fp32 update arithmetic)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import aae
import gm_b200
from gm_b200 import GmError, AdamHP
from aae_oracle import ENC, DEC, DIS, recon_phase, d_phase, g_phase, adam
from mlp_harness import TOL_A, nrel
from oracle import ref_math as R
from test_aae_cpu import weights

pytestmark = pytest.mark.gpu

GEOMS = [(784, 400, 20), (784, 208, 13), (784, 400, 32)]


class Sides:
    """relu hook of the oracle: units with |a| < TOL_A take the side the device took (read back from its buffers, so it
    is called right after the phase it models ran on the device)"""
    BUF = {"h1": ("H1", 0), "h1d": ("H1", 0), "h3": ("H3", 0), "hd": ("AD", 0), "hg": ("AD", 1)}

    def __init__(self, eng):
        self.eng = eng

    def __call__(self, name, a):
        h = np.maximum(a, 0)
        near = np.abs(a) < TOL_A
        if near.any():
            n, c = a.shape
            buf, region = self.BUF[name]
            v = self.eng.debug_read(buf, region * n, n, c).cpu().numpy()
            act = v != 0 if name == "hg" else v > 0          # the G step stores M = w2 1[a > 0]
            h[near] = np.where(act[near], 1e-30, 0.0)
        return h


def _engine(X, H, Z, B, seed):
    eng = gm_b200.AaeEngine(X, H, Z, max_batch=B)
    P, Dp = weights(X, H, Z, seed)
    eng.load({**P, **Dp})
    return eng


def _params(eng):
    return ({k: v.double().cpu().numpy() for k, v in gm_b200.VaeEngine.views(eng).items()},
            {k: v.double().cpu().numpy() for k, v in eng.d_views().items()})


def _check_adam(before, grads, after, st, step, lr, wd=0.0):
    for k in after:
        ref = adam(before[k], grads[k], st[k], step, lr, wd)
        assert np.abs(after[k] - ref).max() < 1e-6, k


@pytest.mark.parametrize("geom", GEOMS, ids=["%dx%dx%d" % g for g in GEOMS])
def test_each_phase_and_the_step_against_the_oracle(geom):
    X, H, Z = geom
    hpR, hpD, hpG = AdamHP.make(1e-3, weight_decay=1e-5), AdamHP.make(2e-4), AdamHP.make(3e-4)
    rng = np.random.default_rng(X + H + Z)
    for b in (1, 65, 300, 4096):
        eng = _engine(X, H, Z, 4096, 11 + Z)
        sides = Sides(eng)
        st = {k: (np.zeros(s), np.zeros(s)) for k, s in [(k, v.shape) for k, v in {**_params(eng)[0], **_params(eng)[1]}.items()]}
        x = (rng.random((b, X)) < 0.13).astype(np.float32)
        prior = rng.standard_normal((b, Z)).astype(np.float32)
        xd = torch.from_numpy(x).cuda()
        # phase 1 and optimizer_R
        P, Dp = _params(eng)
        recon = eng.recon_grad(xd).item()
        r_o, g_o = recon_phase(P, x.astype(np.float64), q=R.bf16_points, relu=sides)
        assert abs(recon - r_o) <= 1e-3 * r_o, (b, recon, r_o)
        gv = {k: v.double().cpu().numpy() for k, v in eng.views(eng.grads).items()}
        for k in ENC + DEC:
            assert nrel(gv[k], g_o[k]) < 3e-3, (b, k, nrel(gv[k], g_o[k]))
        eng.apply(hpR)
        P1, _ = _params(eng)
        _check_adam(P, gv, P1, {k: st[k] for k in ENC + DEC}, 1, 1e-3, 1e-5)
        # phase 2 and optimizer_D, at the updated encoder
        dl = eng.d_grad(b, prior=torch.from_numpy(prior).cuda()).item()
        d_o, gd_o, _ = d_phase(P1, Dp, x.astype(np.float64), prior.astype(np.float64), q=R.bf16_points, relu=sides)
        assert abs(dl - d_o) <= 1e-3 * d_o, (b, dl, d_o)
        gd = {k: v.double().cpu().numpy() for k, v in eng.d_views(eng.d_grads).items()}
        for k in DIS:
            assert nrel(gd[k], gd_o[k]) < 3e-3, (b, k, nrel(gd[k], gd_o[k]))
        assert torch.equal(eng.last_prior(b).cpu(), torch.from_numpy(prior))
        eng.apply_d(hpD)
        _, Dp1 = _params(eng)
        _check_adam(Dp, gd, Dp1, {k: st[k] for k in DIS}, 1, 2e-4)
        # phase 3 and optimizer_G, at the updated discriminator, on phase 2's encoding
        gl = eng.g_grad(b).item()
        g_o3, gg_o = g_phase(P1, Dp1, x.astype(np.float64), q=R.bf16_points, relu=sides)
        assert abs(gl - g_o3) <= 1e-3 * g_o3, (b, gl, g_o3)
        gg = {k: v.double().cpu().numpy() for k, v in eng.views(eng.grads).items()}
        for k in ENC:
            assert nrel(gg[k], gg_o[k]) < 3e-3, (b, k, nrel(gg[k], gg_o[k]))
        for k in DEC:                                    # phase 3 leaves the decoder's gradient as phase 1 left it
            assert np.array_equal(gg[k], gv[k]), k
        eng.apply_g(hpG)
        P2, _ = _params(eng)
        stG = {k: (np.zeros_like(P1[k]), np.zeros_like(P1[k])) for k in ENC}
        _check_adam({k: P1[k] for k in ENC}, gg, {k: P2[k] for k in ENC}, stG, 1, 3e-4)
        for k in DEC:
            assert np.array_equal(P2[k], P1[k]), k
        # optimizer_G's moments are its own: optimizer_R's still hold phase 1's
        m = eng.exp_avg[:eng.n_enc].double().cpu().numpy()
        assert np.allclose(m, 0.1 * np.concatenate([gv[k].ravel() + 1e-5 * P[k].ravel() for k in ENC]), rtol=1e-5, atol=1e-9)


def test_recon_phase_is_the_bir_vae_with_zero_eps_and_lambda_bit_for_bit():
    """With eps_std = 0 and lam = 0 the BIR-VAE step is z = mu + 0 and dmu = dz + 0: the same kernels on the same values
    (the AAE's decoder rows come from aae_latent_rows_kernel instead of bir_latent_kernel, both bf16(mu)), so the loss and
    every gradient are bitwise equal"""
    X, H, Z = 784, 400, 20
    P, _ = weights(X, H, Z, 5)
    a = _engine(X, H, Z, 512, 5)
    bir = gm_b200.BirVaeEngine(X, H, Z, eps_std=0.0, max_batch=512)
    bir.load(P)
    rng = np.random.default_rng(3)
    for b in (1, 65, 512):
        x = torch.from_numpy((rng.random((b, X)) < 0.13).astype(np.float32)).cuda()
        zeros = torch.zeros(b, Z, device="cuda")
        lb = bir.grad(x, eps=zeros, prior=zeros, lam=0.0).clone()
        la = a.recon_grad(x).clone()
        assert torch.equal(la[0], lb[0]) and lb[1].item() == 0.0, (b, la, lb)
        ga, gb = a.views(a.grads), bir.views(bir.grads)
        for k in gb:
            assert torch.equal(ga[k], gb[k]), (b, k)


def test_device_prior_draw():
    X, H, Z, b = 784, 400, 20, 4096
    eng = _engine(X, H, Z, b, 2)
    x = (torch.rand(b, X, device="cuda") < 0.13).float()
    eng.recon_grad(x)
    l1 = eng.d_grad(b, seed=9, step=4).clone()
    g1, p1 = eng.d_grads.clone(), eng.last_prior(b)
    eng.recon_grad(x)
    eng.d_grad(b, seed=9, step=4)
    assert torch.equal(eng.last_prior(b), p1)                         # deterministic in (seed, step)
    eng.recon_grad(x)
    eng.d_grad(b, seed=9, step=5)
    p2 = eng.last_prior(b)
    assert not torch.equal(p1, p2) and (p1 - p2).abs().mean() > 0.5  # a new draw each step
    for p in (p1, p2):                                                 # N(0, 1): 81920 draws, 6-sigma bounds
        n = p.numel()
        assert abs(p.mean().item()) < 6 / n ** 0.5 and abs(p.var().item() - 1) < 6 * (2 / n) ** 0.5
        assert abs(p.double().pow(4).mean().item() - 3) < 6 * (96 / n) ** 0.5
    eng.recon_grad(x)
    l3 = eng.d_grad(b, prior=p1).clone()                              # the same draw passed as prior_dev
    assert torch.equal(l1, l3) and torch.equal(g1, eng.d_grads)


def test_resident_draw_matches_a_host_gather():
    X, H, Z, n, bs = 784, 400, 20, 1000, 300
    eng = _engine(X, H, Z, bs, 3)
    g = torch.Generator().manual_seed(2)
    imgs = (torch.rand(n, X, generator=g) < 0.13).float()
    bits = gm_b200.gan_api.DeviceDataset(imgs, bs).bits
    bpe, seed = -(-n // bs), 77
    for step in (0, 3, 5):
        rows = min(bs, n - (step % bpe) * bs)
        eng.set_sampler(n, bpe, seed, batch_size=bs)
        l1 = eng.recon_grad(bits, fmt="bits", batch=rows, step=step).clone()
        g1, xin1 = eng.grads.clone(), eng.debug_read("Xin", 0, rows, X + 1)
        eng.set_sampler(0, 0, 0)
        idx = eng.sample_indices(bs, step, bpe, n, seed)[:rows]
        assert len(set(idx.tolist())) == rows
        l2 = eng.recon_grad(imgs.cuda(), gather_idx=idx).clone()
        assert torch.equal(l1, l2) and torch.equal(g1, eng.grads)
        assert torch.equal(xin1, eng.debug_read("Xin", 0, rows, X + 1))


class _LSTrainer(aae.AAETrainer):
    """a user-written step: LS-GAN losses on z and a BCE reconstruction"""

    def compute_batch(self, batch):
        x = self._images(batch)
        out, _ = self.model(x)
        return F.binary_cross_entropy(out, x, reduction="sum")

    def train_D(self, images):
        x = self._images(images)
        with torch.no_grad():
            z_f = self.model.encoder(x)
        z_p = self.priors.pop(0).cuda()
        return 0.5 * torch.mean((self.model.discriminator(z_p) - 1) ** 2) + 0.5 * torch.mean(self.model.discriminator(z_f) ** 2)

    def train_G(self, images):
        return 0.5 * torch.mean((self.model.discriminator(self.model.encoder(self._images(images))) - 1) ** 2)


def test_user_written_steps_against_float64_autograd(capsys):
    X, H, Z, n, bs = 784, 64, 8, 192, 64
    torch.manual_seed(4)
    imgs = (torch.rand(n, 1, 28, 28) < 0.2).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(n, dtype=torch.long)), batch_size=bs)
    model = aae.AAE(X, H, Z)
    T = {k: v.detach().double().clone().requires_grad_(True) for k, v in model.state_dict().items()}
    priors = [torch.randn(bs, Z) for _ in range(2 * (n // bs))]
    tr = _LSTrainer(model, loader, loader, loader)
    tr.priors = list(priors)
    tr.train(2, lr=1e-3, D_lr=2e-4, G_lr=3e-4, weight_decay=1e-5)
    assert len(tr.recon_loss) == len(tr.Dlosses) == len(tr.Glosses) == 2 * (n // bs)
    # float64 torch: the same loop, batches and priors
    enc = lambda x: torch.relu(x @ T[ENC[0]].T + T[ENC[1]]) @ T[ENC[2]].T + T[ENC[3]]
    dec = lambda z: torch.sigmoid(torch.relu(z @ T[DEC[0]].T + T[DEC[1]]) @ T[DEC[2]].T + T[DEC[3]])
    dis = lambda z: torch.sigmoid(torch.relu(z @ T[DIS[0]].T + T[DIS[1]]) @ T[DIS[2]].T + T[DIS[3]])
    oR = torch.optim.Adam([T[k] for k in ENC + DEC], lr=1e-3, weight_decay=1e-5)
    oD, oG = torch.optim.Adam([T[k] for k in DIS], lr=2e-4), torch.optim.Adam([T[k] for k in ENC], lr=3e-4)
    ref, pri = [], list(priors)
    for _ in range(2):
        for xb, _ in loader:
            x = xb.view(xb.shape[0], -1).double()
            oR.zero_grad()
            r = F.binary_cross_entropy(dec(enc(x)), x, reduction="sum")
            r.backward()
            oR.step()
            oD.zero_grad()
            zf = enc(x).detach()
            d = 0.5 * torch.mean((dis(pri.pop(0).double()) - 1) ** 2) + 0.5 * torch.mean(dis(zf) ** 2)
            d.backward()
            oD.step()
            oG.zero_grad()
            g = 0.5 * torch.mean((dis(enc(x)) - 1) ** 2)
            g.backward()
            oG.step()
            ref.append((r.item(), d.item(), g.item()))
    got = list(zip(tr.recon_loss, tr.Dlosses, tr.Glosses))
    for a, b in zip(got, ref):
        assert np.allclose(a, b, rtol=1e-2), (a, b)
    # Adam moves each element by about lr whatever its gradient's size, so an element whose small gradient the bf16 GEMMs
    # put on the other side of zero moves the other way: the parameters agree to 1e-2, the losses above to 1e-2
    sd = model.state_dict()
    for k in T:
        assert nrel(sd[k].cpu().numpy(), T[k].detach().numpy()) < 1e-2, (k, nrel(sd[k].cpu().numpy(), T[k].detach().numpy()))
    assert tr._engine is not None and len(tr.priors) == 0
    assert "Epoch[2/2], Recon Loss:" in capsys.readouterr().out


def test_per_call_discriminator_errors():
    model = aae.AAE(784, 64, 8)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset((torch.rand(8, 784) < 0.2).float(), torch.zeros(8)), batch_size=4)
    tr = aae.AAETrainer(model, loader, loader, loader)          # the model's parameters become views of its engine
    z = torch.randn(16, 8, device="cuda", requires_grad=True)
    s0 = model.discriminator(z)
    assert tr._engine is not None and model.discriminator.linear.weight.is_cuda
    model.discriminator(z)
    model.discriminator(z)                                    # two slots: the third call takes s0's
    with pytest.raises(RuntimeError, match="overwritten"):
        s0.sum().backward()
    s = model.discriminator(z)
    s.sum().backward(retain_graph=True)                       # the backward only reads the slot: it may run again
    g1, gz1 = model.discriminator.linear.weight.grad.clone(), z.grad.clone()
    s.sum().backward()
    assert torch.equal(model.discriminator.linear.weight.grad, 2 * g1) and torch.equal(z.grad, 2 * gz1)
    s = model.discriminator(z)
    (gz,) = torch.autograd.grad(s.sum(), z, create_graph=False)
    assert gz.shape == z.shape
    s = model.discriminator(z)
    with pytest.raises(RuntimeError, match="double backward"):
        torch.autograd.grad(s.sum(), z, create_graph=True)


def test_train_on_get_data(tmp_path, capsys):
    from utils import get_data
    train_iter, val_iter, test_iter = get_data()
    model = aae.AAE(784, 400, 20)
    tr = aae.AAETrainer(model, train_iter, val_iter, test_iter)
    tr.train(1)
    out = capsys.readouterr().out
    assert "Epoch[1/1], Recon Loss: " in out and ", D Loss: " in out and ", G Loss: " in out and ", Val Loss: " in out
    nb = len(train_iter)
    assert len(tr.recon_loss) == len(tr.Dlosses) == len(tr.Glosses) == nb and tr.num_epochs == 1
    assert all(np.isfinite(v) for v in tr.recon_loss + tr.Dlosses + tr.Glosses)
    assert np.mean(tr.recon_loss[-50:]) < np.mean(tr.recon_loss[:50])
    assert tr.sample_images().shape == (36, 28, 28)
    best = tr.best_model
    assert isinstance(best, aae.AAE) and best._owner is None
    assert all(p.data_ptr() != q.data_ptr() for p, q in zip(best.parameters(), model.parameters()))
    with torch.no_grad():
        out_b, z_b = best(next(iter(test_iter))[0])
    assert out_b.shape == (100, 784) and z_b.shape == (100, 20)
    path = str(tmp_path / "aae.pt")
    tr.save_model(path)
    m2 = aae.AAE(784, 400, 20)
    tr2 = aae.AAETrainer(m2, train_iter, val_iter, test_iter)
    tr2.load_model(path)
    for (ka, va), (kb, vb) in zip(model.state_dict().items(), m2.state_dict().items()):
        assert ka == kb and torch.equal(va.cpu(), vb.cpu())
    assert abs(tr2.evaluate(val_iter) - tr.evaluate(val_iter)) < 1e-3 * tr.evaluate(val_iter)


def test_c_abi_refuses_bad_arguments_before_any_launch():
    from gm_b200._lib import ctx, VaeDesc, lib
    h = ctx()
    L = lib()
    out = C.c_void_p()
    rc_split = L.gm_aae_create(h, C.byref(VaeDesc(784, 400, 20, 64, gm_b200.PRECISIONS["split"])), C.byref(out))
    rc_z = L.gm_aae_create(h, C.byref(VaeDesc(784, 400, 33, 64, gm_b200.PRECISIONS["bf16"])), C.byref(out))
    rc_x = L.gm_aae_create(h, C.byref(VaeDesc(780, 400, 20, 64, gm_b200.PRECISIONS["bf16"])), C.byref(out))
    assert rc_split != 0 and rc_z != 0 and rc_x != 0
    eng = _engine(784, 400, 20, 64, 1)
    vae = gm_b200.VaeEngine(784, 400, 20, max_batch=64)
    bir = gm_b200.BirVaeEngine(784, 400, 20, max_batch=64)
    x = (torch.rand(64, 784, device="cuda") < 0.13).float()
    px, py = C.c_void_p(x.data_ptr()), C.c_void_p(torch.zeros(64, 20, device="cuda").data_ptr())
    hp = AdamHP.make(1e-3)
    s = None
    n0 = gm_b200.launch_count()
    g = eng.g
    bad = [("gm_aae_recon_grad", (vae.g, px, 0, None, 64, 0, None, s)), ("gm_aae_recon_grad", (g, None, 0, None, 64, 0, None, s)),
           ("gm_aae_recon_grad", (g, px, 0, None, 0, 0, None, s)), ("gm_aae_recon_grad", (g, px, 0, None, 65, 0, None, s)),
           ("gm_aae_d_grad", (g, 64, None, 0, 0, None, s)),                         # nothing staged yet
           ("gm_aae_d_grad", (bir.g, 64, None, 0, 0, None, s)), ("gm_aae_g_grad", (g, 64, None, s)),
           ("gm_aae_g_grad", (vae.g, 64, None, s)), ("gm_aae_apply_d", (g, C.byref(hp), 0, s)),
           ("gm_aae_apply_g", (vae.g, C.byref(hp), 1, s)), ("gm_aae_d_forward", (g, 2, py, 64, px, s)),
           ("gm_aae_d_forward", (g, -1, py, 64, px, s)), ("gm_aae_d_forward", (g, 0, None, 64, px, s)),
           ("gm_aae_d_forward", (vae.g, 0, py, 64, px, s)), ("gm_aae_d_backward", (g, 0, 0, px, None, s)),
           ("gm_aae_d_backward", (g, 0, 8, None, None, s)), ("gm_aae_forward", (bir.g, px, 0, 8, None, None, None, s)),
           ("gm_aae_last_prior", (vae.g, py, 8, s)), ("gm_aae_sync_shadows_d", (vae.g, s)),
           ("gm_aae_bind_d", (vae.g, py, py, None, None, None, None)),
           ("gm_vae_grad", (g, px, 0, None, 64, None, C.c_float(1.0), 0, 0, None, s)),
           ("gm_vae_forward", (g, px, 0, 8, None, 0, 0, None, None, None, s)), ("gm_vae_last_eps", (g, py, 8, s)),
           ("gm_bir_vae_grad", (g, px, 0, None, 64, None, None, C.c_float(1.0), 0, 0, None, s)),
           ("gm_bir_vae_last_latent", (g, py, None, 8, s))]
    for name, args in bad:
        assert getattr(L, name)(*args) != 0, name
    assert L.gm_aae_d_param_count(vae.g) < 0 and L.gm_aae_num_d_slots(vae.g) == 0
    assert gm_b200.launch_count() == n0
    eng.recon_grad(x)
    n1 = gm_b200.launch_count()
    assert L.gm_aae_d_grad(g, 32, None, 0, 0, None, s) != 0                       # a different batch than the staged one
    assert L.gm_aae_g_grad(g, 64, None, s) != 0                                   # not encoded by a D step yet
    assert gm_b200.launch_count() == n1
    with pytest.raises(GmError, match="bf16 only"):
        gm_b200.AaeEngine(784, 400, 20, max_batch=8, precision="split")


def test_launch_ledger_of_the_new_kernels():
    eng = _engine(784, 400, 20, 64, 6)
    x = (torch.rand(64, 784, device="cuda") < 0.13).float()
    gm_b200.prof_enable(2)
    try:
        eng.recon_grad(x)
        eng.apply(AdamHP.make(1e-3))
        eng.d_grad(64)
        eng.apply_d(AdamHP.make(2e-4))
        eng.g_grad(64)
        eng.apply_g(AdamHP.make(2e-4))
        eng.d_forward(0, torch.randn(64, 20, device="cuda"))
        eng.d_backward(0, torch.ones(64, device="cuda"), True)
        torch.cuda.synchronize()
        names = {n: c for n, c, _ in gm_b200.prof_report()}
    finally:
        gm_b200.prof_enable(0)
    assert names.get("aae_latent_rows_kernel", 0) == 3, names       # recon's decoder rows, the D rows, the per-call rows
    assert names.get("bir_dlatent_kernel", 0) == 2, names           # recon's and the G step's latent upstream
    assert names.get("loss_pass_kernel<2>", 0) == 2, names
    assert names.get("dh_kernel", 0) == 2 and names.get("custom_ds_kernel", 0) == 1, names
    assert names.get("adam_kernel", 0) >= 3, names
