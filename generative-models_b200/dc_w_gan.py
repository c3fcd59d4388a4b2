""" (DCWGAN) Wasserstein GAN with weight clipping, with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/w_gan.py's, so its driver code runs on the conv model:

    model = DCWGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCWGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=5e-5, D_lr=5e-5, D_steps=5, clip=0.01)

L(D) = mean(D(G(z))) - mean(D(x)), L(G) = -mean(D(G(z))) (src/w_gan.py:206-227) with D's sigmoid output, as the reference's
D has (src/w_gan.py:70).  After every D step all D parameters, BatchNorm's weight and bias included, are clamped to
[-clip, clip] (src/w_gan.py:158,241-243): inside the D Adam kernel in train() (so under torchrun the clamp follows the
summed gradient's step and the replicas stay identical), and by FusedAdam(clamp=clip) when train_D / train_G are overridden.
"""
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer  # noqa: F401


class DCWGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/w_gan.py:74-85) """


class DCWGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv WGAN (surface of src/w_gan.py:88-310) """
    variant = "w"
    _clip = 0.01

    def train(self, num_epochs, G_lr=5e-5, D_lr=5e-5, D_steps=5, clip=0.01):
        """ Trainer.train (src/w_gan.py:105-188) on the fused conv step, the clamp fused into D's Adam """
        self._clip = float(clip)
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _d_clamp(self):
        return self._clip

    def clip_D_weights(self, clip):
        """ Clamp every D parameter to [-clip, clip] (src/w_gan.py:241-243); the next engine call loads them """
        if self._engine is not None and not self._dirty:
            self._pull()                                    # the engine holds the newest weights: the modules take them first
        for parameter in self.model.D.parameters():
            parameter.data.clamp_(-clip, clip)
        self._dirty = True


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCWGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCWGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=5e-5, D_lr=5e-5, D_steps=5, clip=0.01)
