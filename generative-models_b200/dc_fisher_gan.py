""" (DCFisherGAN) Fisher GAN with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/fisher_gan.py's, so its driver code runs on the conv model:

    model = DCFisherGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCFisherGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1, RHO=1e-6)

L(D) = -((mean D(x) - mean D(G(z))) + LAMBDA Omega - RHO/2 Omega^2), Omega = 1 - (mean D(x)^2 + mean D(G(z))^2) / 2
(src/fisher_gan.py:214-223), with D's sigmoid output and DCGAN's batch-norm discriminator; L(G) = -mean(D(G(z))).  The
multiplier LAMBDA is device state of gm_b200.DcganEngine(variant="fisher"): every D step moves it by LAMBDA += RHO dL/dLAMBDA
= -RHO Omega (src/fisher_gan.py:152-159), and train() resets it to 0 with the given RHO (src/fisher_gan.py:117-118).  The
moments are statistics of the batch; under torchrun the trainer sums them over the ranks (NCCL) before the loss pass.
"""
import torch
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import to_cuda, builtin_step
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer  # noqa: F401


class DCFisherGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/fisher_gan.py:70-81) """


class DCFisherGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv Fisher GAN (surface of src/fisher_gan.py:84-300) """
    variant = "fisher"
    _rho = 1e-6

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=1, RHO=1e-6):
        """ Trainer.train (src/fisher_gan.py:101-190): LAMBDA starts at 0, RHO as given """
        self._rho = float(RHO)
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)
        lam, _ = self._engine.fisher_state()
        self.LAMBDA = torch.tensor([lam])
        self.RHO = torch.tensor(RHO)

    def _pre_train(self, eng):
        eng.fisher_state(0.0, self._rho)                                # src/fisher_gan.py:117-118

    @builtin_step
    def train_D(self, images):
        """ Run 1 step of training for D (src/fisher_gan.py:193-229): returns (D_loss, IPM_ratio); .backward() on D_loss
        delivers the gradients.  LAMBDA moves on the device in the same step.  IPM_ratio is the reference's logging
        expression (with its operator precedence), NaN where its square root is of a negative number. """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        noise = self.compute_noise(n, self.model.z_dim)
        loss = eng.d_grad(eng.stage_images(images.reshape(n, -1).float()), n, noise=noise.float().contiguous())
        m1x, m1g, m2x, m2g = (v / n for v in eng.loss_stats_[:4].tolist())
        ipm = m1x - m1g / 0.5 * (m2x - m2g) ** 0.5 if m2x >= m2g else float("nan")
        return self._loss(1, loss.clone()), ipm


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCFisherGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCFisherGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1, RHO=1e-6)
