"""Bayesian GAN without a GPU: the float64 step (tests/bayes_gan_oracle.py) against float64 torch autograd of the
energies, its J = 1 case against oracle.ref_math's NSGAN step, SGHMC against a hand-written loop, the drop-in's surface
and state_dict, and the refusals that come before any engine or launch."""
import numpy as np
import pytest
import torch

import bayes_gan
from bayes_gan_oracle import G_KEYS, D_KEYS, d_step, g_step, sghmc
from gm_b200 import GmError, BayesGanEngine
from gm_b200 import parallel as par
from inputs import gm_init_weights
from oracle import ref_math as R


def weights(X, H, Z, J, seed):
    """J generator dicts and one discriminator dict (gm_init_weights, float64), each generator from its own seed"""
    PG = []
    for j in range(J):
        W = gm_init_weights([("G.linear", (H, Z)), ("G.generate", (X, H))], seed + 101 * j)
        PG.append({k + s: v.astype(np.float64) for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))})
    W = gm_init_weights([("D.linear", (H, X)), ("D.discriminate", (1, H))], seed + 7)
    PD = {k + s: v.astype(np.float64) for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))}
    return PG, PD


def _torch_energies(PG, PD, x, zs):
    TG = [{k: torch.tensor(v, requires_grad=True) for k, v in P.items()} for P in PG]
    TD = {k: torch.tensor(v, requires_grad=True) for k, v in PD.items()}

    def G(T, z):
        return torch.sigmoid(torch.relu(z @ T[G_KEYS[0]].T + T[G_KEYS[1]]) @ T[G_KEYS[2]].T + T[G_KEYS[3]])

    def D(x):
        return torch.sigmoid(torch.relu(x @ TD[D_KEYS[0]].T + TD[D_KEYS[1]]) @ TD[D_KEYS[2]].T + TD[D_KEYS[3]])
    xt = torch.from_numpy(x)
    fakes = [G(T, torch.from_numpy(z)) for T, z in zip(TG, zs)]
    U_D = -torch.mean(torch.log(D(xt) + 1e-8)) - torch.mean(torch.log(1 - D(torch.cat([f.detach() for f in fakes])) + 1e-8))
    U_D.backward()
    U = [-torch.mean(torch.log(D(f) + 1e-8)) for f in fakes]
    gG = [torch.autograd.grad(u, [T[k] for k in G_KEYS]) for u, T in zip(U, TG)]
    return U_D.item(), {k: TD[k].grad.numpy() for k in D_KEYS}, [u.item() for u in U], gG


@pytest.mark.parametrize("geom", [(64, 32, 5, 3), (784, 48, 20, 2)])
def test_oracle_against_torch_autograd(geom):
    X, H, Z, J = geom
    PG, PD = weights(X, H, Z, J, 11 + Z)
    rng = np.random.default_rng(X + J)
    x = (rng.random((13, X)) < 0.2).astype(np.float64)
    zs = [rng.standard_normal((13, Z)) for _ in range(J)]
    ud, gd, U, gG = _torch_energies(PG, PD, x, zs)
    L, g, outs = d_step(PG, PD, x, zs)
    assert np.isclose(L, ud, rtol=1e-12) and outs.shape == ((1 + J) * 13, 1)
    for k in D_KEYS:
        assert np.allclose(g[k].reshape(gd[k].shape), gd[k], rtol=1e-10, atol=1e-14), k
    Lg, grads, losses = g_step(PG, PD, zs)
    assert np.allclose(losses, U, rtol=1e-12) and np.isclose(Lg, np.mean(U), rtol=1e-12)
    for j in range(J):
        for k, t in zip(G_KEYS, gG[j]):
            assert np.allclose(grads[j][k].reshape(t.shape), t.numpy(), rtol=1e-10, atol=1e-14), (j, k)


def test_one_sample_is_nsgan():
    X, H, Z = 784, 64, 20
    PG, PD = weights(X, H, Z, 1, 3)
    rng = np.random.default_rng(1)
    x = (rng.random((17, X)) < 0.2).astype(np.float64)
    z = rng.standard_normal((17, Z))
    P = {**PG[0], **PD}
    for q in (R._exact, R.bf16_points):
        L0, g0, _ = R.gan_d_step(P, "ns", x, z, q=q)
        L1, g1, _ = d_step(PG, PD, x, [z], q=q)
        assert np.isclose(L0, L1, rtol=1e-14, atol=0) and all(np.allclose(g0[k], g1[k], rtol=1e-14, atol=0) for k in D_KEYS)
        L0, g0, _ = R.gan_g_step(P, "ns", z, q=q)
        L1, g1, _ = g_step(PG, PD, [z], q=q)
        assert np.isclose(L0, L1, rtol=1e-14, atol=0) and all(np.allclose(g0[k], g1[0][k], rtol=1e-14, atol=0) for k in G_KEYS)


def test_sghmc_against_a_loop():
    rng = np.random.default_rng(2)
    theta, v = rng.standard_normal(50), np.zeros(50)
    t_ref, v_ref = theta.copy(), v.copy()
    lr, alpha, ps, N = 2e-4, 0.1, 0.05, 1000.0
    for _ in range(3):
        g, xi = rng.standard_normal(50), rng.standard_normal(50)
        theta, v = sghmc(theta, v, g, xi, lr, alpha, ps, N)
        for i in range(50):
            prior = t_ref[i] / (ps * ps * N)
            v_ref[i] = (1 - alpha) * v_ref[i] - lr * (g[i] + prior) + (2 * alpha * lr / N) ** 0.5 * xi[i]
            t_ref[i] = t_ref[i] + v_ref[i]
    assert np.allclose(theta, t_ref, rtol=1e-14, atol=0) and np.allclose(v, v_ref, rtol=1e-14, atol=0)
    # the prior term pulls every weight towards 0: with g = xi = 0 a weight shrinks
    t1, _ = sghmc(np.ones(1), np.zeros(1), np.zeros(1), np.zeros(1), lr, alpha, ps, N)
    assert t1[0] == 1 - lr / (ps * ps * N)


def test_surface_and_state_dict():
    m = bayes_gan.BayesGAN(784, 400, 20, num_g_samples=3)
    assert isinstance(m.G, torch.nn.ModuleList) and len(m.G) == 3 and m.num_g_samples == 3 and m.shape == 28
    keys = list(m.state_dict())
    want = ["G.%d.%s.%s" % (j, l, t) for j in range(3) for l in ("linear", "generate") for t in ("weight", "bias")]
    want += ["D.linear.weight", "D.linear.bias", "D.discriminate.weight", "D.discriminate.bias"]
    assert keys == want
    assert m.state_dict()["G.2.generate.weight"].shape == (784, 400) and m.state_dict()["D.discriminate.weight"].shape == (1, 400)
    w = [g.linear.weight for g in m.G]
    assert not torch.equal(w[0], w[1]) and not torch.equal(w[1], w[2])      # the chains start apart
    assert bayes_gan.BayesGAN(784, 400, 20).num_g_samples == 10
    import inspect
    sig = inspect.signature(bayes_gan.BayesGANTrainer.train)
    assert [(p.name, p.default) for p in list(sig.parameters.values())[1:]] == [
        ("num_epochs", inspect.Parameter.empty), ("G_lr", 2e-4), ("D_lr", 2e-4), ("D_steps", 1), ("alpha", 0.1),
        ("prior_std", 1.0), ("data_size", None)]


def _loader():
    data = torch.utils.data.TensorDataset((torch.rand(16, 1, 28, 28) < 0.2).float(), torch.zeros(16))
    return torch.utils.data.DataLoader(data, batch_size=8)


def test_refusals_before_any_engine(monkeypatch):
    for n in (0, 17):
        with pytest.raises(GmError, match="num_g_samples"):
            bayes_gan.BayesGAN(784, 400, 20, num_g_samples=n)
    with pytest.raises(GmError, match="bf16 only"):
        BayesGanEngine(784, 400, 20, num_g=2, precision="split")
    with pytest.raises(GmError, match="num_g"):
        BayesGanEngine(784, 400, 20, num_g=17)

    class WithD(bayes_gan.BayesGANTrainer):
        def train_D(self, images):
            return None

    class WithG(bayes_gan.BayesGANTrainer):
        def train_G(self, images):
            return None
    for cls in (WithD, WithG):
        tr = cls(bayes_gan.BayesGAN(784, 32, 8, 2), _loader(), _loader(), _loader())
        with pytest.raises(GmError, match="cannot be overridden"):
            tr.train(1)
        assert tr._engine is None
    tr = bayes_gan.BayesGANTrainer(bayes_gan.BayesGAN(784, 32, 8, 2), _loader(), _loader(), _loader())
    monkeypatch.setattr(par, "world_size", lambda: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(1)
    assert tr._engine is None
