"""Which conv trainers run a user-written train_D / train_G (README.md:31) and which refuse one, without a GPU: every
shipped conv trainer's steps are the fused built-in ones, a subclass that overrides them is detected, and BEGAN / InfoGAN
overrides stop train() with GmError before anything runs."""
import pytest
import torch

import dc_be_gan
import dc_dra_gan
import dc_fisher_gan
import dc_gan
import dc_info_gan
import dc_ra_gan
import dc_w_gp_gan
from gm_b200 import GmError

_SHIPPED = [(dc_gan.DCGAN, dc_gan.DCGANTrainer), (dc_w_gp_gan.DCWGPGAN, dc_w_gp_gan.DCWGPGANTrainer),
            (dc_dra_gan.DCDRAGAN, dc_dra_gan.DCDRAGANTrainer), (dc_ra_gan.DCRaNSGAN, dc_ra_gan.DCRaNSGANTrainer),
            (dc_fisher_gan.DCFisherGAN, dc_fisher_gan.DCFisherGANTrainer), (dc_be_gan.DCBEGAN, dc_be_gan.DCBEGANTrainer),
            (dc_info_gan.DCInfoGAN, dc_info_gan.DCInfoGANTrainer)]


@pytest.mark.parametrize("Model,Trainer", _SHIPPED, ids=[t.__name__ for _, t in _SHIPPED])
def test_shipped_conv_trainers_run_their_fused_steps(Model, Trainer):
    tr = Trainer(Model(hidden_dim=16), None, None, None)
    assert tr._has_custom_step() is False


def _override(Trainer, method):
    def step(self, images, *args, **kw):
        return torch.zeros(())
    return type("Custom" + Trainer.__name__, (Trainer,), {method: step})


@pytest.mark.parametrize("method", ["train_D", "train_G"])
def test_an_override_is_detected(method):
    tr = _override(dc_w_gp_gan.DCWGPGANTrainer, method)(dc_w_gp_gan.DCWGPGAN(hidden_dim=16), None, None, None)
    assert tr._has_custom_step() is True


@pytest.mark.parametrize("Model,Trainer,method", [(dc_be_gan.DCBEGAN, dc_be_gan.DCBEGANTrainer, "train_D"),
                                                  (dc_be_gan.DCBEGAN, dc_be_gan.DCBEGANTrainer, "train_G"),
                                                  (dc_info_gan.DCInfoGAN, dc_info_gan.DCInfoGANTrainer, "train_G"),
                                                  (dc_info_gan.DCInfoGAN, dc_info_gan.DCInfoGANTrainer, "train_Q")])
def test_began_and_infogan_overrides_are_refused(Model, Trainer, method):
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(torch.rand(8, 3, 64, 64), torch.zeros(8)), batch_size=4)
    tr = _override(Trainer, method)(Model(hidden_dim=16), loader, loader, loader)
    with pytest.raises(GmError, match="not supported"):
        tr.train(num_epochs=1)
    assert tr.Glosses == [] and tr._engine is None
