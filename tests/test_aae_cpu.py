"""Adversarial autoencoder without a GPU: the float64 oracle (tests/aae_oracle.py) against torch float64 autograd and
torch.optim.Adam over several steps, the drop-in's surface, state_dict and load_model, and the refusals that come
before any engine or launch."""
import inspect

import numpy as np
import pytest
import torch

import aae
from aae_oracle import ENC, DEC, DIS, aae_step, new_state, recon_phase, d_phase, g_phase
from gm_b200 import GmError, AaeEngine
from gm_b200 import parallel as par
from inputs import gm_init_weights

NAMES = list(ENC + DEC + DIS)
SHAPES = {"encoder.linear.weight": (400, 784), "encoder.linear.bias": (400,), "encoder.mu.weight": (20, 400),
          "encoder.mu.bias": (20,), "decoder.linear.weight": (400, 20), "decoder.linear.bias": (400,),
          "decoder.recon.weight": (784, 400), "decoder.recon.bias": (784,), "discriminator.linear.weight": (400, 20),
          "discriminator.linear.bias": (400,), "discriminator.discriminate.weight": (1, 400),
          "discriminator.discriminate.bias": (1,)}


def weights(X, H, Z, seed):
    """gm_init_weights for the encoder / decoder (P) and the latent discriminator (Dp), float32"""
    W = gm_init_weights([("encoder.linear", (H, X)), ("encoder.mu", (Z, H)), ("decoder.linear", (H, Z)),
                         ("decoder.recon", (X, H)), ("discriminator.linear", (H, Z)),
                         ("discriminator.discriminate", (1, H))], seed)
    flat = {k + s: v for k, (w, b) in W.items() for s, v in ((".weight", w), (".bias", b))}
    return ({k: flat[k] for k in ENC + DEC}, {k: flat[k] for k in DIS})


def _torch_step(T, opts, x, prior):
    """the three phases in torch float64 autograd on tensors T, with torch.optim.Adam"""
    def enc(x):
        return torch.relu(x @ T[ENC[0]].T + T[ENC[1]]) @ T[ENC[2]].T + T[ENC[3]]

    def dis(z):
        return torch.sigmoid(torch.relu(z @ T[DIS[0]].T + T[DIS[1]]) @ T[DIS[2]].T + T[DIS[3]])
    R, D, G = opts
    R.zero_grad()
    out = torch.sigmoid(torch.relu(enc(x) @ T[DEC[0]].T + T[DEC[1]]) @ T[DEC[2]].T + T[DEC[3]])
    recon = torch.sum((x - out) ** 2)
    recon.backward()
    R.step()
    D.zero_grad()
    z_f = enc(x).detach()
    D_loss = -torch.mean(torch.log(dis(prior) + 1e-8) + torch.log(1 - dis(z_f) + 1e-8))
    D_loss.backward()
    D.step()
    G.zero_grad()
    G_loss = -torch.mean(torch.log(dis(enc(x)) + 1e-8))
    G_loss.backward()
    G.step()
    return recon.item(), D_loss.item(), G_loss.item()


@pytest.mark.parametrize("geom", [(64, 32, 5), (784, 48, 20)])
def test_oracle_against_torch_autograd_and_adam(geom):
    X, H, Z = geom
    P, Dp = weights(X, H, Z, 7 + Z)
    P = {k: v.astype(np.float64) for k, v in P.items()}
    Dp = {k: v.astype(np.float64) for k, v in Dp.items()}
    T = {k: torch.tensor(v, requires_grad=True) for k, v in {**P, **Dp}.items()}
    lr, D_lr, G_lr, wd = 1e-3, 2e-4, 3e-4, 1e-5
    opts = (torch.optim.Adam([T[k] for k in ENC + DEC], lr=lr, weight_decay=wd), torch.optim.Adam([T[k] for k in DIS], lr=D_lr),
            torch.optim.Adam([T[k] for k in ENC], lr=G_lr))
    st = new_state(P, Dp)
    rng = np.random.default_rng(X + Z)
    for _ in range(4):
        x = (rng.random((17, X)) < 0.2).astype(np.float64)
        prior = rng.standard_normal((17, Z))
        ref = _torch_step(T, opts, torch.from_numpy(x), torch.from_numpy(prior))
        recon, dl, gl, P, Dp, _ = aae_step(P, Dp, st, x, prior, lr, D_lr, G_lr, wd)
        assert np.allclose([recon, dl, gl], ref, rtol=1e-12, atol=0), ((recon, dl, gl), ref)
        for k in NAMES:
            got = P[k] if k in P else Dp[k]
            assert np.allclose(got, T[k].detach().numpy(), rtol=1e-10, atol=1e-13), k


def test_phase_gradients_against_autograd():
    """each phase's gradients alone (no optimizer), at the exact points"""
    X, H, Z = 64, 32, 6
    P, Dp = weights(X, H, Z, 3)
    P = {k: v.astype(np.float64) for k, v in P.items()}
    Dp = {k: v.astype(np.float64) for k, v in Dp.items()}
    rng = np.random.default_rng(5)
    x = (rng.random((9, X)) < 0.3).astype(np.float64)
    prior = rng.standard_normal((9, Z))
    T = {k: torch.tensor(v, requires_grad=True) for k, v in {**P, **Dp}.items()}
    xt, pt = torch.from_numpy(x), torch.from_numpy(prior)
    enc = lambda x: torch.relu(x @ T[ENC[0]].T + T[ENC[1]]) @ T[ENC[2]].T + T[ENC[3]]
    dis = lambda z: torch.sigmoid(torch.relu(z @ T[DIS[0]].T + T[DIS[1]]) @ T[DIS[2]].T + T[DIS[3]])
    recon, g = recon_phase(P, x)
    r = torch.sum((xt - torch.sigmoid(torch.relu(enc(xt) @ T[DEC[0]].T + T[DEC[1]]) @ T[DEC[2]].T + T[DEC[3]])) ** 2)
    gt = torch.autograd.grad(r, [T[k] for k in ENC + DEC])
    assert np.isclose(recon, r.item(), rtol=1e-13)
    for k, v in zip(ENC + DEC, gt):
        assert np.allclose(g[k], v.numpy(), rtol=1e-10, atol=1e-14), k
    dl, gd, _ = d_phase(P, Dp, x, prior)
    d = -torch.mean(torch.log(dis(pt) + 1e-8) + torch.log(1 - dis(enc(xt).detach()) + 1e-8))
    for k, v in zip(DIS, torch.autograd.grad(d, [T[k] for k in DIS])):
        assert np.allclose(gd[k], v.numpy(), rtol=1e-10, atol=1e-14), k
    assert np.isclose(dl, d.item(), rtol=1e-13)
    gl, gg = g_phase(P, Dp, x)
    gx = -torch.mean(torch.log(dis(enc(xt)) + 1e-8))
    for k, v in zip(ENC, torch.autograd.grad(gx, [T[k] for k in ENC])):
        assert np.allclose(gg[k], v.numpy(), rtol=1e-10, atol=1e-14), k
    assert np.isclose(gl, gx.item(), rtol=1e-13)


def _loader(n=8, x=784):
    imgs = (torch.rand(n, 1, 28, 28) < 0.2).float() if x == 784 else (torch.rand(n, x) < 0.2).float()
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(n, dtype=torch.long)), batch_size=4)


def test_the_surface():
    assert str(inspect.signature(aae.AAE.__init__)) == "(self, image_size=784, hidden_dim=400, z_dim=20)"
    assert str(inspect.signature(aae.AAE.forward)) == "(self, x)"
    assert str(inspect.signature(aae.Encoder.__init__)) == "(self, image_size, hidden_dim, z_dim)"
    assert str(inspect.signature(aae.Decoder.__init__)) == "(self, z_dim, hidden_dim, image_size)"
    assert str(inspect.signature(aae.Discriminator.__init__)) == "(self, z_dim, hidden_dim, output_dim=1)"
    T = aae.AAETrainer
    assert str(inspect.signature(T.__init__)) == "(self, model, train_iter, val_iter, test_iter, viz=False)"
    assert str(inspect.signature(T.train)) == "(self, num_epochs, lr=0.001, D_lr=0.0002, G_lr=0.0002, weight_decay=1e-05)"
    assert str(inspect.signature(T.compute_batch)) == "(self, batch)"
    assert str(inspect.signature(T.train_D)) == "(self, images)"
    assert str(inspect.signature(T.train_G)) == "(self, images)"
    assert str(inspect.signature(T.evaluate)) == "(self, iterator)"
    assert str(inspect.signature(T.sample_images)) == "(self, epoch=-100, num_images=36, save=True)"
    for m in ["reconstruct_images", "viz_loss", "save_model", "load_model"]:
        assert callable(getattr(T, m)), m
    model = aae.AAE()
    sd = model.state_dict()
    assert list(sd) == NAMES
    assert {k: tuple(v.shape) for k, v in sd.items()} == SHAPES
    assert model.shape == 28
    loader = _loader()
    tr = T(model, loader, loader, loader)
    assert (tr.recon_loss, tr.Dlosses, tr.Glosses, tr.num_epochs, tr.best_val_loss, tr.name) == ([], [], [], 0, 1e10, "AAE")
    assert T.device_noise is True
    assert aae.EPOCH_LINE == "Epoch[%d/%d], Recon Loss: %.4f, D Loss: %.4f, G Loss: %.4f, Val Loss: %.4f"
    assert AaeEngine.NAMES == list(ENC + DEC) and AaeEngine.D_NAMES == list(DIS)


def test_load_model_of_a_saved_aae(tmp_path):
    torch.manual_seed(0)
    a = aae.AAE(784, 64, 6)
    path = str(tmp_path / "aae.pt")
    loader = _loader()
    aae.AAETrainer(a, loader, loader, loader).save_model(path)
    b = aae.AAE(784, 64, 6)
    aae.AAETrainer(b, loader, loader, loader).load_model(path)
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)


def test_model_refusals():
    with pytest.raises(GmError, match="one output"):
        aae.Discriminator(20, 400, output_dim=2)
    with pytest.raises(GmError, match="bf16 only"):
        AaeEngine(784, 400, 20, max_batch=8, precision="split")
    m = aae.AAE(784, 32, 4)                           # no trainer and no GPU: the modules refuse, there is no eager path
    if not torch.cuda.is_available():
        with pytest.raises(GmError, match="no eager/CPU path"):
            m.encoder(torch.zeros(2, 784))
        with pytest.raises(GmError, match="no eager/CPU path"):
            m.discriminator(torch.zeros(2, 4))


def _custom(*methods):
    body = {}
    if "compute_batch" in methods:
        body["compute_batch"] = lambda self, batch: torch.zeros(())
    if "train_D" in methods:
        body["train_D"] = lambda self, images: torch.zeros(())
    if "train_G" in methods:
        body["train_G"] = lambda self, images: torch.zeros(())
    return type("CustomAAETrainer", (aae.AAETrainer,), body)


@pytest.mark.parametrize("methods", [(), ("compute_batch",), ("train_D",), ("train_G",), ("train_D", "train_G")])
def test_override_detection(methods):
    loader = _loader()
    assert aae.has_custom_step(_custom(*methods)(aae.AAE(784, 32, 4), loader, loader, loader)) is bool(methods)


@pytest.mark.parametrize("methods", [(), ("train_G",)])
def test_multi_rank_training_is_refused_before_any_engine(methods, monkeypatch):
    loader = _loader()
    tr = _custom(*methods)(aae.AAE(784, 32, 4), loader, loader, loader)
    monkeypatch.setattr(par, "world_size", lambda group=None: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(1)
    assert tr._engine is None
