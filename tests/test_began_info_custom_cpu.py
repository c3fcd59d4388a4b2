"""Which MLP BEGAN / InfoGAN trainers run user-written train_D / train_G / train_Q (README.md:31), without a GPU: the
shipped methods carry the built-in marker, overriding any one of them is detected, and an override under more than one
rank stops train() before any engine is built."""
import pytest
import torch

import be_gan
import info_gan
from gm_b200 import GmError
from gm_b200 import parallel as par


def _loader():
    return torch.utils.data.DataLoader(torch.utils.data.TensorDataset(torch.rand(8, 1, 28, 28), torch.zeros(8)), batch_size=4)


def _began(Trainer=be_gan.BEGANTrainer):
    it = _loader()
    return Trainer(be_gan.BEGAN(784, 32, 8), it, it, it)


def _info(Trainer=info_gan.InfoGANTrainer):
    it = _loader()
    return Trainer(info_gan.InfoGAN(784, 32, 8, 10, 10), it, it, it)


def _override(Trainer, name):
    def step(self, images, *args, **kw):
        return torch.zeros((), requires_grad=True)
    return type("Custom" + name + Trainer.__name__, (Trainer,), {name: step})


def test_shipped_steps_are_marked_builtin():
    for fn in (be_gan.BEGANTrainer.train_D, be_gan.BEGANTrainer.train_G, info_gan.InfoGANTrainer.train_D,
               info_gan.InfoGANTrainer.train_G, info_gan.InfoGANTrainer.train_Q):
        assert getattr(fn, "_gm_builtin", False), fn
    assert _began()._has_custom_step() is False
    assert _info()._has_custom_step() is False


@pytest.mark.parametrize("name", ["train_D", "train_G"])
def test_a_began_override_is_detected(name):
    assert _began(_override(be_gan.BEGANTrainer, name))._has_custom_step() is True


@pytest.mark.parametrize("name", ["train_D", "train_G", "train_Q"])
def test_an_infogan_override_is_detected(name):
    assert _info(_override(info_gan.InfoGANTrainer, name))._has_custom_step() is True


@pytest.mark.parametrize("make,Trainer,name", [(_began, be_gan.BEGANTrainer, "train_D"), (_began, be_gan.BEGANTrainer, "train_G"),
                                               (_info, info_gan.InfoGANTrainer, "train_D"),
                                               (_info, info_gan.InfoGANTrainer, "train_G"),
                                               (_info, info_gan.InfoGANTrainer, "train_Q")])
def test_a_multi_rank_override_is_refused_before_any_engine(make, Trainer, name, monkeypatch):
    tr = make(_override(Trainer, name))
    monkeypatch.setattr(par, "world_size", lambda group=None: 2)
    with pytest.raises(GmError, match="one process"):
        tr.train(num_epochs=1)
    assert tr._engine is None and tr.Dlosses == [] and tr.Glosses == [] and tr.num_epochs == 0
