"""BIR-VAE without a GPU: the float64 oracle (tests/bir_vae_oracle.py) against the fixture the unmodified reference made
(tests/golden/bir_vae.npz), the drop-in's surface against the reference's literals, override detection, and the
refusal of data-parallel training before any engine is built."""
import inspect

import numpy as np
import pytest
import torch

import bir_vae
from bir_vae_oracle import bir_vae_step, mmd, mmd_grad
from gm_b200 import GmError
from gm_b200 import parallel as par
from gm_b200.gan_api import has_custom_compute_batch
from inputs import B, X, H, Z, gm_init_weights, images_from_bits, load_case, unpack_draws, params_dict, check_summary
from make_golden_bir_vae import BIR_SHAPES, SEED


def _loader():
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(torch.rand(8, 1, 28, 28), torch.zeros(8)), batch_size=4)


def test_oracle_reproduces_the_reference_step():
    fx = load_case("bir_vae")
    P = params_dict(gm_init_weights(BIR_SHAPES, SEED), np.float64)
    x = images_from_bits(fx).astype(np.float64)
    mse, m, g, _ = bir_vae_step(P, x, fx["step1_eps"].astype(np.float64), fx["step1_prior"].astype(np.float64))
    assert abs(mse - fx["step1_mse"]) <= 1e-5 * abs(fx["step1_mse"])
    assert abs(m - fx["step1_mmd"]) <= 1e-4 * abs(fx["step1_mmd"])      # fp32 reference: B^2 terms summed in fp32
    for name in g:
        assert check_summary(fx, "step1_grad_" + name, g[name], rtol=2e-3) < 2e-3, name


def test_oracle_reproduces_the_reference_losses_over_the_train_loop():
    """the reference's own train() over STEPS steps: its recorded eps / prior draws replayed through the oracle + Adam"""
    from oracle.ref_math import Adam
    fx = load_case("bir_vae")
    P = params_dict(gm_init_weights(BIR_SHAPES, SEED), np.float64)
    x = images_from_bits(fx).astype(np.float64)
    priors = unpack_draws(fx)
    opt = Adam(list(P.keys()), 1e-3, wd=1e-5)
    for k in range(len(fx["recon_loss"])):
        mse, m, g, _ = bir_vae_step(P, x, fx["eps"][k].astype(np.float64), priors[k].astype(np.float64))
        assert abs(mse - fx["recon_loss"][k]) <= 2e-4 * fx["recon_loss"][k], k
        assert abs(m - fx["mmd_loss"][k]) <= 2e-3 * abs(fx["mmd_loss"][k]), k
        opt.step(P, g)


def test_mmd_closed_forms():
    rng = np.random.default_rng(1)
    z, p = rng.standard_normal((5, 3)), rng.standard_normal((5, 3))
    # B = 1: lambda (2 - 2 k(p, z))
    assert np.isclose(mmd(z[:1], p[:1], 7.0), 7.0 * (2 - 2 * np.exp(-((z[0] - p[0]) ** 2).sum() / 9)))
    eps = 1e-6
    num = np.zeros_like(z)
    for i in range(5):
        for d in range(3):
            zp, zm = z.copy(), z.copy()
            zp[i, d] += eps
            zm[i, d] -= eps
            num[i, d] = (mmd(zp, p, 3.0) - mmd(zm, p, 3.0)) / (2 * eps)
    assert np.allclose(mmd_grad(z, p, 3.0), num, rtol=1e-6, atol=1e-8)


def test_the_surface_matches_the_reference():
    assert str(inspect.signature(bir_vae.BIRVAE.__init__)) == "(self, image_size=784, hidden_dim=400, z_dim=20, I=13.3)"
    assert str(inspect.signature(bir_vae.BIRVAETrainer.__init__)) == "(self, model, train_iter, val_iter, test_iter, viz=False)"
    assert str(inspect.signature(bir_vae.BIRVAETrainer.train)) == "(self, num_epochs, lr=0.001, weight_decay=1e-05)"
    assert str(inspect.signature(bir_vae.BIRVAETrainer.compute_batch)) == "(self, batch, LAMBDA=1000.0)"
    assert str(inspect.signature(bir_vae.Encoder.__init__)) == "(self, image_size, hidden_dim, z_dim)"
    assert str(inspect.signature(bir_vae.Decoder.__init__)) == "(self, z_dim, hidden_dim, image_size)"
    for m in ["train", "compute_batch", "maximum_mean_discrepancy", "compute_kernel", "evaluate", "reconstruct_images",
              "sample_images", "sample_interpolated_images", "explore_latent_space", "make_all", "viz_loss", "save_model",
              "load_model"]:
        assert callable(getattr(bir_vae.BIRVAETrainer, m)), m
    assert str(inspect.signature(bir_vae.BIRVAETrainer.explore_latent_space)) == "(self, num_epochs=3)"
    assert str(inspect.signature(bir_vae.BIRVAETrainer.sample_images)) == "(self, epoch=-100, num_images=36, save=True)"
    model = bir_vae.BIRVAE()
    assert list(model.state_dict()) == ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.mu.bias",
                                        "decoder.linear.weight", "decoder.linear.bias", "decoder.recon.weight",
                                        "decoder.recon.bias"]
    assert model.set_var == 1 / (4 ** (13.3 / 20)) and model.shape == 28 and model.I == 13.3
    loader = _loader()
    tr = bir_vae.BIRVAETrainer(model, loader, loader, loader)
    assert (tr.mmd_loss, tr.recon_loss, tr.num_epochs, tr.best_val_loss, tr.name) == ([], [], 0, 1e10, "BIRVAE")
    assert bir_vae.EPOCH_LINE == "Epoch[%d/%d], Total Loss: %.4f, MSE Loss: %.4f, MMD Loss: %.4f, Val Loss: %.4f"


def test_compute_kernel_is_the_reference_expression():
    tr = bir_vae.BIRVAETrainer(bir_vae.BIRVAE(784, 32, 4), _loader(), _loader(), _loader())
    rng = np.random.default_rng(2)
    a, b = rng.standard_normal((6, 4)), rng.standard_normal((5, 4))
    from bir_vae_oracle import gauss_kernel
    assert np.allclose(tr.compute_kernel(torch.from_numpy(a), torch.from_numpy(b)).numpy(), gauss_kernel(a, b), rtol=1e-12)


def _custom(Trainer=bir_vae.BIRVAETrainer):
    def compute_batch(self, batch):
        return torch.zeros(()), torch.zeros(())
    return type("Custom" + Trainer.__name__, (Trainer,), {"compute_batch": compute_batch})


def test_override_detection():
    loader = _loader()
    assert has_custom_compute_batch(bir_vae.BIRVAETrainer(bir_vae.BIRVAE(784, 32, 4), loader, loader, loader)) is False
    assert has_custom_compute_batch(_custom()(bir_vae.BIRVAE(784, 32, 4), loader, loader, loader)) is True


@pytest.mark.parametrize("custom", [False, True])
def test_multi_rank_training_is_refused_before_any_engine(custom, monkeypatch):
    loader = _loader()
    Trainer = _custom() if custom else bir_vae.BIRVAETrainer
    tr = Trainer(bir_vae.BIRVAE(784, 32, 4), loader, loader, loader)
    monkeypatch.setattr(par, "world_size", lambda group=None: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(1)
    assert tr._engine is None
