""" (DCfGAN) f-GAN with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/f_gan.py's, so its driver code runs on the conv model:

    model = DCfGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCfGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, method='jensen_shannon', G_lr=1e-4, D_lr=1e-4, D_steps=1)

The six divergences of src/f_gan.py:99-142 are rows of the loss kernel (gm_b200.DcganEngine(variant="f_<method>")) on the
batch-norm DCGAN D's sigmoid output; `Divergence` is f_gan's, plain torch for user code that calls it.  A train() call with
a different method rebuilds the engine for it; the weights and BatchNorm running statistics carry over.
"""
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer, pull_running_stats, push_running_stats  # noqa: F401
from f_gan import Divergence  # noqa: F401


class DCfGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/f_gan.py:71-82) """


class DCfGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv f-GAN (surface of src/f_gan.py:145-360) """
    variant = "f_jensen_shannon"

    def train(self, num_epochs, method, G_lr=1e-4, D_lr=1e-4, D_steps=1):
        """ Trainer.train (src/f_gan.py:162-242) on the fused conv step """
        self._set_method(method)
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _set_method(self, method):
        self.loss_fnc = Divergence(method)                          # src/f_gan.py:175
        variant = "f_" + self.loss_fnc.method
        if self._engine is not None and variant != self.variant:
            if self._dirty:                 # the modules hold the newest weights; the engine the newest running statistics
                pull_running_stats(self._engine, self._nets())
            else:
                self._pull()                # the trained weights and running statistics into the modules
            self._engine = None
            self.variant = variant
            push_running_stats(self._engine_synced(), self._nets())  # the new engine loads the weights, then takes the statistics
        self.variant = variant


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCfGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCfGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, method='jensen_shannon', G_lr=1e-4, D_lr=1e-4, D_steps=1)
