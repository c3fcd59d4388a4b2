""" (DCLSGAN) Least-squares GAN with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/ls_gan.py's, so its driver code runs on the conv model:

    model = DCLSGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCLSGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1)

L(D) = 0.5 mean((D(x) - b)^2) + 0.5 mean((D(G(z)) - a)^2), L(G) = 0.5 mean((D(G(z)) - c)^2) (src/ls_gan.py:173-215) with D's
sigmoid output and the reference's defaults a = 0, b = 1, c = 1.  train_D(images, a, b) and train_G(images, c) take them
per call; the fused train() takes them from `trainer.loss_consts = dict(ls_a=..., ls_b=..., ls_c=...)`.  The loss kernel
reads them on the device (gm_loss_rows_c).
"""
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import builtin_step
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer  # noqa: F401


class DCLSGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/ls_gan.py:64-75) """


class DCLSGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv LSGAN (surface of src/ls_gan.py:78-290) """
    variant = "ls"
    # the targets of the fused train(): any of ls_a, ls_b, ls_c; the rest keep the reference's defaults
    loss_consts = {}
    _DEFAULTS = dict(ls_a=0.0, ls_b=1.0, ls_c=1.0)

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=1):
        """ Trainer.train (src/ls_gan.py:95-170) on the fused conv step """
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _set_targets(self, eng, **kw):
        unknown = set(self.loss_consts) - set(self._DEFAULTS)
        if unknown:
            raise GmError("loss_consts of the LSGAN are ls_a, ls_b, ls_c (got %s)" % ", ".join(sorted(unknown)))
        want = dict(self._DEFAULTS, **self.loss_consts)
        want.update(kw)
        eng.ls_a, eng.ls_b, eng.ls_c = float(want["ls_a"]), float(want["ls_b"]), float(want["ls_c"])

    def _pre_train(self, eng):
        self._set_targets(eng)

    @builtin_step
    def train_D(self, images, a=0, b=1):
        """ Run 1 step of training for discriminator (src/ls_gan.py:173-195): returns D_loss; .backward() delivers the
        gradients """
        self._set_targets(self._engine_synced(), ls_a=a, ls_b=b)
        return super().train_D(images)

    @builtin_step
    def train_G(self, images, c=1):
        """ Run 1 step of training for generator (src/ls_gan.py:197-215) """
        self._set_targets(self._engine_synced(), ls_c=c)
        return super().train_G(images)


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCLSGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCLSGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1)
