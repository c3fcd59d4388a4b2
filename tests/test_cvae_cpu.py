"""Conditional VAE without a GPU: the float64 oracle (tests/cvae_oracle.py) against oracle.ref_math.vae_step and the
VAE's golden fixture (a CVAE whose label weights are zero is the reference VAE), the label-column gradients, the
drop-in's surface, and the refusals that come before any engine or launch."""
import inspect

import numpy as np
import pytest
import torch

import cvae
from cvae_oracle import cvae_step
from gm_b200 import GmError, CvaeEngine
from gm_b200 import parallel as par
from gm_b200.engine import class_ids
from gm_b200.gan_api import has_custom_compute_batch
from inputs import VAE_SHAPES, STEPS, gm_init_weights, params_dict, load_case, unpack_draws, images_from_bits, check_summary
from oracle import ref_math as R

NAMES = ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.mu.bias", "encoder.log_var.weight",
         "encoder.log_var.bias", "decoder.linear.weight", "decoder.linear.bias", "decoder.recon.weight",
         "decoder.recon.bias"]


def _widen(P, C):
    """P (a VAE's parameters) as a CVAE's with zero label columns"""
    out = dict(P)
    for k in ("encoder.linear.weight", "decoder.linear.weight"):
        out[k] = np.concatenate([P[k], np.zeros((P[k].shape[0], C))], axis=1)
    return out


def _vae_case():
    fx = load_case("vae")
    P = params_dict(gm_init_weights(VAE_SHAPES, 4321), np.float64)
    x = images_from_bits(fx).astype(np.float64)
    return fx, P, x


@pytest.mark.parametrize("q", ["exact", "bf16"])
def test_zero_label_weights_equal_the_vae_step_exactly(q):
    fx, P, x = _vae_case()
    eps = unpack_draws(fx, "step1_")[0].astype(np.float64)
    y = np.arange(x.shape[0]) % 10
    hook = R.bf16_points if q == "bf16" else R._exact
    recon, kl, g, fw = R.vae_step(P, x, eps, q=hook)
    recon_c, kl_c, g_c, fw_c = cvae_step(_widen(P, 10), x, y, eps, 10, q=hook)
    assert recon_c == recon and kl_c == kl
    for k in ("out", "mu", "lv"):
        assert np.array_equal(fw_c[k], fw[k]), k
    for k in g:
        gc = g_c[k]
        if k in ("encoder.linear.weight", "decoder.linear.weight"):
            gc = gc[:, :g[k].shape[1]]
        assert np.array_equal(gc, g[k]), k


def test_zero_label_weights_reproduce_the_vae_golden_fixture():
    """the VAE golden test's own bounds (tests/test_oracle_golden.py), through the CVAE oracle and Adam"""
    fx, P0, x = _vae_case()
    y = np.arange(x.shape[0]) % 10
    d1 = [d.astype(np.float64) for d in unpack_draws(fx, "step1_")]
    recon, kl, g, _ = cvae_step(_widen(P0, 10), x, y, d1[0], 10)
    assert abs(recon - fx["step1_recon"]) <= 2e-6 * abs(fx["step1_recon"])
    assert abs(kl - fx["step1_kl"]) <= 2e-5 * abs(fx["step1_kl"])
    for k in ("encoder.linear.weight", "decoder.linear.weight"):
        g[k] = g[k][:, :-10]
    for k, v in g.items():
        check_summary(fx, "step1_grad_" + k, v, rtol=5e-5)
    P = _widen(P0, 10)
    opt = R.Adam(list(P.keys()), 1e-3, wd=1e-5)
    Rl, Kl = [], []
    for d in [d.astype(np.float64) for d in unpack_draws(fx)][:STEPS]:
        # the label columns have a gradient of their own: without it (and at zero, under Adam and weight decay) they
        # stay zero, and the model stays the reference VAE
        recon, kl, g, _ = cvae_step(P, x, y, d, 10)
        for k in ("encoder.linear.weight", "decoder.linear.weight"):
            g[k][:, -10:] = 0.0
        opt.step(P, g)
        Rl.append(recon)
        Kl.append(kl)
    np.testing.assert_allclose(Rl, fx["recon_loss"], rtol=2e-5)
    np.testing.assert_allclose(Kl, fx["kl_loss"], rtol=2e-4)


def test_label_column_gradients_are_per_class_row_sums():
    rng = np.random.default_rng(7)
    X, H, Z, C, B = 48, 32, 5, 4, 37
    P = {}
    for name, shape in [("encoder.linear.weight", (H, X + C)), ("encoder.linear.bias", (H,)), ("encoder.mu.weight", (Z, H)),
                        ("encoder.mu.bias", (Z,)), ("encoder.log_var.weight", (Z, H)), ("encoder.log_var.bias", (Z,)),
                        ("decoder.linear.weight", (H, Z + C)), ("decoder.linear.bias", (H,)),
                        ("decoder.recon.weight", (X, H)), ("decoder.recon.bias", (X,))]:
        P[name] = 0.2 * rng.standard_normal(shape)
    x = (rng.random((B, X)) < 0.3).astype(np.float64)
    y = rng.integers(0, C, B)
    y[:C] = np.arange(C)
    eps = rng.standard_normal((B, Z))
    _, _, g, fw = cvae_step(P, x, y, eps, C)
    for c in range(C):
        np.testing.assert_allclose(g["encoder.linear.weight"][:, X + c], fw["da1"][y == c].sum(0), rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(g["decoder.linear.weight"][:, Z + c], fw["da3"][y == c].sum(0), rtol=1e-12, atol=1e-15)
    # and a central difference through the label weights agrees with the closed form
    k, r, c = "decoder.linear.weight", 3, Z + 1
    h = 1e-6
    Pp, Pm = {n: v.copy() for n, v in P.items()}, {n: v.copy() for n, v in P.items()}
    Pp[k][r, c] += h
    Pm[k][r, c] -= h
    fp = sum(cvae_step(Pp, x, y, eps, C)[:2])
    fm = sum(cvae_step(Pm, x, y, eps, C)[:2])
    assert abs((fp - fm) / (2 * h) - g[k][r, c]) <= 1e-5 * max(1.0, abs(g[k][r, c]))


def _loader(n=8, bs=4, labels=None):
    y = torch.arange(n) % 10 if labels is None else labels
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(torch.rand(n, 1, 28, 28), y), batch_size=bs)


def test_the_surface():
    assert str(inspect.signature(cvae.CVAE.__init__)) == "(self, image_size=784, hidden_dim=400, z_dim=20, num_classes=10)"
    assert str(inspect.signature(cvae.CVAE.forward)) == "(self, x, y)"
    assert str(inspect.signature(cvae.Encoder.__init__)) == "(self, image_size, hidden_dim, z_dim, num_classes)"
    assert str(inspect.signature(cvae.Decoder.__init__)) == "(self, z_dim, hidden_dim, image_size, num_classes)"
    assert str(inspect.signature(cvae.Encoder.forward)) == "(self, x, y)"
    assert str(inspect.signature(cvae.Decoder.forward)) == "(self, z, y)"
    T = cvae.CVAETrainer
    assert str(inspect.signature(T.__init__)) == "(self, model, train_iter, val_iter, test_iter, viz=False)"
    assert str(inspect.signature(T.train)) == "(self, num_epochs, lr=0.001, weight_decay=1e-05)"
    assert str(inspect.signature(T.compute_batch)) == "(self, batch)"
    assert str(inspect.signature(T.reconstruct_images)) == "(self, images, labels, epoch, save=True)"
    assert str(inspect.signature(T.sample_images)) == "(self, epoch=-100, num_images=36, save=True, labels=None)"
    for m in ["kl_divergence", "evaluate", "viz_loss", "save_model", "load_model"]:
        assert callable(getattr(T, m)), m
    model = cvae.CVAE()
    sd = model.state_dict()
    assert list(sd) == NAMES
    shapes = {"encoder.linear.weight": (400, 794), "encoder.linear.bias": (400,), "encoder.mu.weight": (20, 400),
              "encoder.mu.bias": (20,), "encoder.log_var.weight": (20, 400), "encoder.log_var.bias": (20,),
              "decoder.linear.weight": (400, 30), "decoder.linear.bias": (400,), "decoder.recon.weight": (784, 400),
              "decoder.recon.bias": (784,)}
    assert {k: tuple(v.shape) for k, v in sd.items()} == shapes
    assert (model.num_classes, model.shape) == (10, 28)
    loader = _loader()
    tr = T(model, loader, loader, loader)
    assert (tr.kl_loss, tr.recon_loss, tr.num_epochs, tr.best_val_loss, tr.name) == ([], [], 0, 1e10, "CVAE")
    assert T.device_noise is True


def test_load_model_of_a_saved_cvae(tmp_path):
    torch.manual_seed(0)
    a = cvae.CVAE(784, 64, 6, 3)
    path = str(tmp_path / "cvae.pt")
    loader = _loader(labels=torch.arange(8) % 3)
    cvae.CVAETrainer(a, loader, loader, loader).save_model(path)
    b = cvae.CVAE(784, 64, 6, 3)
    cvae.CVAETrainer(b, loader, loader, loader).load_model(path)
    for (ka, va), (kb, vb) in zip(a.state_dict().items(), b.state_dict().items()):
        assert ka == kb and torch.equal(va, vb)


def test_model_refusals():
    with pytest.raises(GmError, match="num_classes must be >= 1"):
        cvae.CVAE(num_classes=0)
    with pytest.raises(GmError, match="num_classes must be >= 1"):
        cvae.CVAE(num_classes=-2)
    with pytest.raises(GmError, match="<= 63"):
        cvae.CVAE(z_dim=20, num_classes=44)
    cvae.CVAE(z_dim=20, num_classes=43)                              # z + C = 63: the widest latent row
    with pytest.raises(GmError, match="bf16 only"):
        CvaeEngine(784, 400, 20, 10, max_batch=8, precision="split")


@pytest.mark.parametrize("bad, match", [(torch.tensor([0, 10]), r"in \[0, 10\)"), (torch.tensor([-1, 3]), r"in \[0, 10\)"),
                                        (np.array([2, 11]), r"in \[0, 10\)"), (torch.tensor([1.0, 2.0]), "integer"),
                                        (np.array([0.5]), "integer"), (torch.tensor([True, False]), "integer"),
                                        (torch.tensor([], dtype=torch.long), "empty")])
def test_labels_are_refused_on_the_host(bad, match):
    with pytest.raises(GmError, match=match):
        class_ids(bad, 10, torch.device("cpu"))


def test_one_hot_and_miscounted_labels_are_refused_on_the_host():
    """a one-hot int64 matrix (what F.one_hot returns) is not a label vector, and a label vector must have one entry per
    row: neither is flattened or truncated into something the kernels would accept"""
    y = torch.tensor([3, 7, 9, 2])
    with pytest.raises(GmError, match="shape"):
        class_ids(torch.nn.functional.one_hot(y, 10), 10, torch.device("cpu"))
    with pytest.raises(GmError, match="shape"):
        class_ids(y.view(2, 2), 10, torch.device("cpu"))
    with pytest.raises(GmError, match="shape"):
        class_ids(torch.tensor(3), 10, torch.device("cpu"))
    with pytest.raises(GmError, match="5 labels for 4 rows"):
        class_ids(torch.tensor([3, 7, 9, 2, 1]), 10, torch.device("cpu"), 4)
    with pytest.raises(GmError, match="3 labels for 4 rows"):
        class_ids(torch.tensor([3, 7, 9]), 10, torch.device("cpu"), 4)
    ok = class_ids(y.view(4, 1), 10, torch.device("cpu"), 4)
    assert ok.t.tolist() == [3, 7, 9, 2]
    with pytest.raises(GmError, match="4 labels for 5 rows"):
        class_ids(ok, 10, torch.device("cpu"), 5)                         # a checked ClassIds is counted again


def test_good_labels_become_int32():
    y = class_ids(torch.tensor([[3], [0], [9]]), 10, torch.device("cpu"))
    assert y.t.dtype == torch.int32 and y.t.tolist() == [3, 0, 9] and len(y) == 3
    assert class_ids(y, 10, torch.device("cpu")) is y
    with pytest.raises(GmError, match="checked for 10 classes"):
        class_ids(y, 4, torch.device("cpu"))


def _custom():
    def compute_batch(self, batch):
        return torch.zeros(()), torch.zeros(())
    return type("CustomCVAETrainer", (cvae.CVAETrainer,), {"compute_batch": compute_batch})


def test_override_detection():
    loader = _loader()
    assert has_custom_compute_batch(cvae.CVAETrainer(cvae.CVAE(784, 32, 4), loader, loader, loader)) is False
    assert has_custom_compute_batch(_custom()(cvae.CVAE(784, 32, 4), loader, loader, loader)) is True


@pytest.mark.parametrize("custom", [False, True])
def test_multi_rank_training_is_refused_before_any_engine(custom, monkeypatch):
    loader = _loader()
    Trainer = _custom() if custom else cvae.CVAETrainer
    tr = Trainer(cvae.CVAE(784, 32, 4), loader, loader, loader)
    monkeypatch.setattr(par, "world_size", lambda group=None: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(1)
    assert tr._engine is None
