""" (DCRaNSGAN) Relativistic non-saturating GAN with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/ra_gan.py's, so its driver code runs on the conv model:

    model = DCRaNSGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCRaNSGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1)

L(D) = -mean(log(sigmoid(D(x) - mean(D(G(z)))) + 1e-8) + log(sigmoid(1 - D(G(z))) + 1e-8)) / 2 (src/ra_gan.py:204-205), with
D's sigmoid output; L(G) is the non-saturating -mean(log(D(G(z)) + 1e-8)).  The discriminator is DCGAN's batch-norm one.
mean(D(G(z))) is a statistic of the batch: gm_b200.DcganEngine(variant="ra") computes it (and the sum its gradient needs)
in separate passes of the loss kernel, and under torchrun the trainer sums those statistics over the ranks (NCCL) between
the passes, so that N ranks x n images train on the statistics of the global batch.
"""
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer  # noqa: F401


class DCRaNSGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/ra_gan.py:75-86) """


class DCRaNSGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv RaNSGAN (surface of src/ra_gan.py:89-300) """
    variant = "ra"

    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1):
        """ Trainer.train (src/ra_gan.py:106-180) on the fused conv step """
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCRaNSGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCRaNSGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1)
