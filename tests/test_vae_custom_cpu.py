"""Which VAE-family trainers run a user-written compute_batch (README.md:31), without a GPU: the four shipped trainers'
compute_batch is the fused built-in one, a subclass that overrides it is detected (also below DCAutoencoderTrainer, which
overrides DCVAETrainer's itself), and an override under more than one rank stops train() before any engine is built."""
import pytest
import torch

import ae
import dc_ae
import dc_vae
import vae
from gm_b200 import GmError
from gm_b200 import parallel as par
from gm_b200.gan_api import has_custom_compute_batch


def _loader(shape):
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(torch.rand(8, *shape), torch.zeros(8)), batch_size=4)


_SHIPPED = [(lambda: vae.VAE(784, 32, 8), vae.VAETrainer, (1, 28, 28)),
            (lambda: ae.Autoencoder(784, 32), ae.AutoencoderTrainer, (1, 28, 28)),
            (lambda: dc_vae.DCVAE(hidden_dim=16, z_dim=8), dc_vae.DCVAETrainer, (3, 64, 64)),
            (lambda: dc_ae.DCAutoencoder(hidden_dim=16, z_dim=8), dc_ae.DCAutoencoderTrainer, (3, 64, 64))]
_IDS = [t.__name__ for _, t, _ in _SHIPPED]


def _override(Trainer):
    def compute_batch(self, batch):
        return torch.zeros(())
    return type("Custom" + Trainer.__name__, (Trainer,), {"compute_batch": compute_batch})


@pytest.mark.parametrize("Model,Trainer,shape", _SHIPPED, ids=_IDS)
def test_shipped_trainers_run_their_fused_step(Model, Trainer, shape):
    loader = _loader(shape)
    assert has_custom_compute_batch(Trainer(Model(), loader, loader, loader)) is False


@pytest.mark.parametrize("Model,Trainer,shape", _SHIPPED, ids=_IDS)
def test_an_override_is_detected(Model, Trainer, shape):
    loader = _loader(shape)
    assert has_custom_compute_batch(_override(Trainer)(Model(), loader, loader, loader)) is True


def test_a_subclass_of_a_shipped_subclass_keeps_the_marker():
    """DCAutoencoderTrainer overrides DCVAETrainer.compute_batch with its own built-in step: a plain subclass of it (no
    compute_batch of its own) still runs the fused step, one that overrides it does not"""
    loader = _loader((3, 64, 64))
    Plain = type("PlainAE", (dc_ae.DCAutoencoderTrainer,), {})
    assert has_custom_compute_batch(Plain(dc_ae.DCAutoencoder(hidden_dim=16, z_dim=8), loader, loader, loader)) is False
    Custom = _override(Plain)
    assert has_custom_compute_batch(Custom(dc_ae.DCAutoencoder(hidden_dim=16, z_dim=8), loader, loader, loader)) is True


@pytest.mark.parametrize("Model,Trainer,shape", _SHIPPED, ids=_IDS)
def test_a_multi_rank_override_is_refused_before_any_engine(Model, Trainer, shape, monkeypatch):
    loader = _loader(shape)
    tr = _override(Trainer)(Model(), loader, loader, loader)
    monkeypatch.setattr(par, "world_size", lambda group=None: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(num_epochs=1)
    assert tr._engine is None and tr.recon_loss == [] and tr.num_epochs == 0
