"""Bayesian GAN on the GPU: the D and per-sample G gradients of the Bayes-mode GAN engine against the float64 step
(tests/bayes_gan_oracle.py) at the engine's bf16 points, J = 1 against an NS engine bit for bit, SGHMC against a float64
update of the engine's own gradient and xi, the refreshed operand copies of every sample, the xi draws, BayesGANTrainer.train
on get_data(), and the C ABI's refusals (nothing launched).

Bounds are test_aae_gpu.py's: losses within 1e-3 relative, gradients within 3e-3 norm-relative of the float64 step
evaluated at the engine's bf16 storage points (near-kink ReLU units take the device's side, the fake images are the
device's stored values); SGHMC to 1e-6 absolute (fp32 update arithmetic)."""
import ctypes as C

import numpy as np
import pytest
import torch

import bayes_gan
import gm_b200
from gm_b200 import GmError, SghmcHP, AdamHP
from bayes_gan_oracle import G_KEYS, D_KEYS, d_step, g_step, sghmc
from mlp_harness import TOL_A, nrel, gan_engine
from oracle import ref_math as R
from test_bayes_gan_cpu import weights

pytestmark = pytest.mark.gpu

GEOMS = [(784, 400, 20), (784, 208, 13), (784, 400, 32)]
G, D = 0, 1


class DeviceSides:
    """patches ref_math's g_forward / d_forward for one oracle call: hidden units with |a| < TOL_A take the side the
    device took, and each sample's fake images are the device's stored bf16 values (checked to lie within one ulp).
    d_regions / g_samples: the Aall row region (units of B) and the generator sample of successive calls."""

    def __init__(self, eng, B, d_regions, g_samples):
        self.eng, self.B, self.d_regions, self.g_samples = eng, B, list(d_regions), list(g_samples)

    def _side(self, fw, key, buf, row0):
        near = np.abs(fw["a1"]) < TOL_A
        if near.any():
            n, c = fw["a1"].shape
            act = self.eng.debug_read(buf, row0, n, c).cpu().numpy() != 0
            for k in key:
                v = fw[k].copy()
                v[near] = np.where(act[near], 1e-30, 0.0)
                fw[k] = v

    def __enter__(self):
        self._d, self._g = R.d_forward, R.g_forward

        def d_forward(P, x, *a, **k):
            fw = self._d(P, x, *a, **k)
            self._side(fw, ("h", "hq"), "Aall", self.d_regions.pop(0) * self.B)
            return fw

        def g_forward(P, z, *a, **k):
            fw = self._g(P, z, *a, **k)
            j = self.g_samples.pop(0)
            self._side(fw, ("h",), "Hg", j * self.B)
            n, x = fw["out"].shape
            dev = self.eng.debug_read("Xall", (1 + j) * self.B, n, x).cpu().numpy().astype(np.float64)
            assert not (np.abs(dev - fw["out"]) > 2.0 ** -7 * np.abs(fw["out"])).any(), "stored fake rows beyond one bf16 ulp"
            fw["out"] = dev
            return fw
        R.d_forward, R.g_forward = d_forward, g_forward
        return self

    def __exit__(self, *exc):
        R.d_forward, R.g_forward = self._d, self._g
        return False


def _engine(X, H, Z, J, B, seed):
    eng = gm_b200.BayesGanEngine(X, H, Z, num_g=J, max_batch=B)
    PG, PD = weights(X, H, Z, J, seed)
    for j in range(J):
        eng.load(G, [PG[j][k] for k in G_KEYS], sample=j)
    eng.load(D, [PD[k] for k in D_KEYS])
    return eng


def _params(eng):
    PG = [{k: v.double().cpu().numpy() for k, v in zip(G_KEYS, eng.views(G, sample=j))} for j in range(eng.num_g)]
    PD = {k: v.double().cpu().numpy() for k, v in zip(D_KEYS, eng.views(D))}
    return PG, PD


@pytest.mark.parametrize("J", [1, 3, 10])
@pytest.mark.parametrize("geom", GEOMS, ids=["%dx%dx%d" % g for g in GEOMS])
def test_gradients_against_the_oracle(geom, J):
    X, H, Z = geom
    rng = np.random.default_rng(X + H + Z + J)
    eng = _engine(X, H, Z, J, 4096, 5 + Z)
    PG, PD = _params(eng)
    for b in (1, 65, 4096):
        x = (rng.random((b, X)) < 0.13).astype(np.float32)
        z = rng.standard_normal((J * b, Z)).astype(np.float32)
        zs = [z[j * b:(j + 1) * b].astype(np.float64) for j in range(J)]
        ld = eng.d_grad(torch.from_numpy(x).cuda(), noise=torch.from_numpy(z).cuda()).item()
        with DeviceSides(eng, b, [0] + list(range(1, J + 1)), range(J)):
            l_o, g_o, _ = d_step(PG, PD, x.astype(np.float64), zs, q=R.bf16_points)
        assert abs(ld - l_o) <= 1e-3 * abs(l_o), (b, ld, l_o)
        gd = {k: v.double().cpu().numpy() for k, v in zip(D_KEYS, eng.views(D, eng.grads[D]))}
        for k in D_KEYS:
            assert nrel(gd[k], g_o[k].reshape(gd[k].shape)) < 3e-3, (b, k, nrel(gd[k], g_o[k].reshape(gd[k].shape)))
        z2 = rng.standard_normal((J * b, Z)).astype(np.float32)
        lg = eng.g_grad(b, noise=torch.from_numpy(z2).cuda()).item()
        with DeviceSides(eng, b, range(1, J + 1), range(J)):
            lg_o, gg_o, _ = g_step(PG, PD, [z2[j * b:(j + 1) * b].astype(np.float64) for j in range(J)], q=R.bf16_points)
        assert abs(lg - lg_o) <= 1e-3 * abs(lg_o), (b, lg, lg_o)
        for j in range(J):
            gg = {k: v.double().cpu().numpy() for k, v in zip(G_KEYS, eng.views(G, eng.grads[G], sample=j))}
            for k in G_KEYS:
                e = nrel(gg[k], gg_o[j][k].reshape(gg[k].shape))
                assert e < 3e-3, (b, j, k, e)


def test_one_sample_is_the_ns_engine_bit_for_bit():
    X, H, Z = 784, 400, 20
    bay = _engine(X, H, Z, 1, 512, 9)
    ns = gan_engine("ns", X, H, Z, max_batch=512)
    for net in (G, D):
        ns.load(net, [t.clone() for t in bay.views(net)])
    rng = np.random.default_rng(4)
    for b in (1, 65, 512):
        x = torch.from_numpy((rng.random((b, X)) < 0.13).astype(np.float32)).cuda()
        for noise in (torch.randn(b, Z, device="cuda"), None):
            la = bay.d_grad(x, noise=noise, seed=7, step=3).clone()
            lb = ns.d_grad(x, noise=noise, seed=7, step=3).clone()
            assert torch.equal(la, lb) and torch.equal(bay.grads[D], ns.grads[D]), (b, noise is None)
            la = bay.g_grad(b, noise=noise, seed=7, step=3).clone()
            lb = ns.g_grad(b, noise=noise, seed=7, step=3).clone()
            assert torch.equal(la, lb) and torch.equal(bay.grads[G][:ns.n[G]], ns.grads[G]), (b, noise is None)


@pytest.mark.parametrize("prior_std", [1.0, 0.01])
def test_sghmc_against_float64_and_the_refreshed_samples(prior_std):
    X, H, Z, J, b = 784, 400, 20, 3, 256
    eng = _engine(X, H, Z, J, b, 12)
    hp = dict(lr=2e-4, alpha=0.1, prior_std=prior_std, data_size=100.0)
    x = (torch.rand(b, X, device="cuda") < 0.13).float()
    v = [np.zeros(n) for n in eng.n]
    for step in range(2):
        eng.d_grad(x, seed=1, step=step)
        eng.g_grad(b, seed=1, step=step)
        for net in (D, G):
            th, gr = eng.params[net].double().cpu().numpy(), eng.grads[net].double().cpu().numpy()
            xi = eng.sghmc_noise(net, 5, step).double().cpu().numpy()
            eng.apply(net, SghmcHP(**hp), seed=5, step=step)
            t_ref, v[net] = sghmc(th, v[net], gr, xi, **hp)
            if net == G:                       # alignment padding between samples is left alone
                keep = np.zeros(eng.n[G], bool)
                for j in range(J):
                    keep[j * eng.stride:j * eng.stride + H * Z + H + X * H + X] = True
                t_ref, v[net] = np.where(keep, t_ref, th), np.where(keep, v[net], 0.0)
            assert np.abs(eng.params[net].double().cpu().numpy() - t_ref).max() < 1e-6, (step, net)
            assert np.abs(eng.momentum[net].double().cpu().numpy() - v[net]).max() < 1e-6, (step, net)
    if prior_std < 0.1:                        # the prior dominates: every weight shrank towards 0
        PG, _ = _params(eng)
        PG0, _ = weights(X, H, Z, J, 12)
        assert np.abs(PG[1][G_KEYS[2]]).mean() < 0.999 * np.abs(PG0[1][G_KEYS[2]]).mean()
    PG, _ = _params(eng)
    z = torch.randn(100, Z, device="cuda")
    for j in range(J):                         # every sample's operand copies were refreshed by the update
        img = eng.generate(j, z).double().cpu().numpy()
        ref = R.g_forward(PG[j], z.double().cpu().numpy(), q=R.bf16_points)["out"]
        assert np.abs(img - ref).max() < 4e-3, j


def test_xi_draws():
    eng = _engine(784, 400, 20, 10, 64, 3)
    a = eng.sghmc_noise(G, 11, 4)
    assert torch.equal(a, eng.sghmc_noise(G, 11, 4))                      # reproducible
    assert not torch.equal(a, eng.sghmc_noise(G, 11, 5))                  # per step
    assert not torch.equal(a, eng.sghmc_noise(G, 12, 4))                  # per seed
    d = eng.sghmc_noise(D, 11, 4)
    assert not torch.equal(a[:d.numel()], d)                              # per net
    s = eng.stride
    assert (a[:s] - a[s:2 * s]).abs().mean() > 0.5                        # per sample
    assert abs(a.mean().item()) < 5e-3 and abs(a.var().item() - 1) < 1e-2
    assert abs(d.mean().item()) < 5e-3 and abs(d.var().item() - 1) < 1e-2


def test_train_on_get_data(tmp_path, capsys):
    from utils import get_data
    train_iter, val_iter, test_iter = get_data()
    model = bayes_gan.BayesGAN(784, 400, 20, num_g_samples=10)
    tr = bayes_gan.BayesGANTrainer(model, train_iter, val_iter, test_iter)
    before = [g.generate.weight.detach().clone() for g in model.G]
    tr.train(1)
    out = capsys.readouterr().out
    assert "Epoch[1/1], G Loss: " in out and ", D Loss: " in out
    assert len(tr.Glosses) == len(tr.Dlosses) == len(train_iter) and tr.num_epochs == 1
    assert all(np.isfinite(v) for v in tr.Glosses + tr.Dlosses)
    after = [g.generate.weight.detach() for g in model.G]
    for j in range(10):
        assert not torch.equal(before[j].cuda(), after[j]), j                # every sample moved
        for k in range(j):
            assert (after[j] - after[k]).abs().mean() > 1e-3, (j, k)        # and they stay apart
    imgs = tr.generate_images(1, save=False)
    assert imgs.shape == (36, 28, 28) and float(imgs.min()) >= 0 and float(imgs.max()) <= 1
    path = str(tmp_path / "bayes_gan.pt")
    tr.save_model(path)
    m2 = bayes_gan.BayesGAN(784, 400, 20, num_g_samples=10)
    tr2 = bayes_gan.BayesGANTrainer(m2, train_iter, val_iter, test_iter)
    tr2.load_model(path)
    for (ka, va), (kb, vb) in zip(model.state_dict().items(), m2.state_dict().items()):
        assert ka == kb and torch.equal(va.cpu(), vb.cpu())
    z = torch.randn(8, 20, device="cuda")
    with torch.no_grad():
        assert torch.equal(model.G[3](z), m2.G[3](z)) and torch.equal(model.D(model.G[3](z)), m2.D(m2.G[3](z)))


def test_c_abi_refuses_before_any_launch():
    from gm_b200._lib import ctx, GanDesc, lib, SghmcHP as HP
    h, L = ctx(), lib()
    out = C.c_void_p()
    P = gm_b200.PRECISIONS
    desc = lambda v=0, act=0, prec=P["bf16"], mb=64: GanDesc(784, 400, 20, mb, v, act, prec)
    assert L.gm_bgan_create(h, C.byref(desc()), 0, C.byref(out)) == -1
    assert L.gm_bgan_create(h, C.byref(desc()), 17, C.byref(out)) == -1
    assert L.gm_bgan_create(h, C.byref(desc(v=2)), 2, C.byref(out)) == -1                # not NS
    assert L.gm_bgan_create(h, C.byref(desc(act=1)), 2, C.byref(out)) == -1              # not a sigmoid D
    assert L.gm_bgan_create(h, C.byref(desc(prec=P["split"])), 2, C.byref(out)) == -4
    assert L.gm_bgan_create(h, C.byref(desc(mb=1 << 20)), 16, C.byref(out)) == -4        # row indices overflow
    bay = _engine(784, 400, 20, 2, 64, 1)
    ns = gan_engine("ns", max_batch=64)
    x = (torch.rand(64, 784, device="cuda") < 0.13).float()
    px, pz = C.c_void_p(x.data_ptr()), C.c_void_p(torch.zeros(128, 20, device="cuda").data_ptr())
    adam, hp, s, g = AdamHP.make(1e-3), HP(2e-4, 0.1, 1.0, 100.0), None, bay.g
    f = C.c_float(1.0 / 64)
    buf = (C.c_float * 11)()
    n0 = gm_b200.launch_count()
    bad = [("gm_gan_apply", (g, 0, C.byref(adam), 1, s)), ("gm_gan_apply_allreduce", (g, 0, C.byref(adam), 1, None, s)),
           ("gm_gan_exchange_begin", (g, 0, None, s)),
           ("gm_gan_d_grad", (g, px, 0, None, 64, None, None, f, 0, 0, None, s)), ("gm_gan_d_stage", (g, px, 0, None, 64, 0, s)),
           ("gm_gan_g_grad", (g, 64, None, f, 0, 0, None, s)), ("gm_gan_g_forward_stage", (g, 64, None, 0, 0, s)),
           ("gm_gan_g_grad_staged", (g, 64, f, None, s)), ("gm_gan_set_lazy_grads", (g, 1, s)),
           ("gm_gan_use_device_step", (g, 1, None, s)), ("gm_gan_attach_comm", (g, None)),
           ("gm_gan_d_forward", (g, 0, px, 64, pz, s)), ("gm_gan_d_backward", (g, 0, 64, pz, None, s)),
           ("gm_gan_g_forward", (g, pz, 64, px, s)), ("gm_gan_g_backward", (g, 64, px, s)),
           ("gm_gan_ae_forward", (g, 0, px, 64, px, s)), ("gm_gan_ae_backward", (g, 0, 64, px, None, s)),
           ("gm_gan_generate", (g, pz, 64, px, s)), ("gm_gan_bind_q", (g, pz, pz, None, None, None, None)),
           ("gm_gan_sync_shadows_q", (g, s)), ("gm_gan_q_grad", (g, 64, pz, 0, f, None, s)), ("gm_gan_apply_mi", (g, C.byref(adam), 1, s)),
           ("gm_gan_q_forward", (g, 0, px, 64, pz, s)), ("gm_gan_q_backward", (g, 0, 64, pz, None, s)),
           ("gm_gan_began_state", (g, buf, 0, s)), ("gm_gan_began_control", (g, C.c_float(0.5), C.c_float(1e-3), C.c_float(1.0), s)),
           # the gm_bgan_* entries refuse a point-estimate engine, and bad arguments
           ("gm_bgan_d_grad", (ns.g, px, 0, None, 64, None, 0, 0, None, s)), ("gm_bgan_g_grad", (ns.g, 64, None, 0, 0, None, s)),
           ("gm_bgan_apply", (ns.g, 0, C.byref(hp), 0, 0, s)), ("gm_bgan_generate", (ns.g, 0, pz, 8, px, s)),
           ("gm_bgan_sghmc_noise", (ns.g, 0, 0, 0, px, s)),
           ("gm_bgan_d_grad", (g, None, 0, None, 64, None, 0, 0, None, s)), ("gm_bgan_d_grad", (g, px, 0, None, 65, None, 0, 0, None, s)),
           ("gm_bgan_g_grad", (g, 0, None, 0, 0, None, s)), ("gm_bgan_generate", (g, 2, pz, 8, px, s)),
           ("gm_bgan_apply", (g, 2, C.byref(hp), 0, 0, s)), ("gm_bgan_apply", (g, 0, C.byref(HP(2e-4, 0.1, 0.0, 100.0)), 0, 0, s))]
    for name, args in bad:
        assert getattr(L, name)(*args) == -1, name
    assert L.gm_bgan_g_stride(ns.g) == -1 and L.gm_bgan_num_samples(ns.g) == 0 and L.gm_bgan_num_samples(g) == 2
    assert gm_b200.launch_count() == n0
    with pytest.raises(GmError):
        bay.d_forward(0, x)
