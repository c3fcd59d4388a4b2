""" (VAE) Variational autoencoder — drop-in for the reference's src/vae.py.

Same classes and signatures (src/vae.py:47-396).  Losses follow the reference CODE:
reconstruction = sum((x - out)^2) (src/vae.py:203; a sum of squared errors although the
comments say cross-entropy), KL = sum(0.5 (mu^2 + exp(lv) - lv - 1)) (src/vae.py:212),
Adam with coupled weight decay (src/vae.py:139-142).  Forward, both losses, the backward
and Adam run in the hand-written sm_90a kernels of libgm_b200.so.
"""
from copy import deepcopy  # noqa: F401

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403

from gm_b200 import VaeEngine
from gm_b200.gan_api import to_cuda, engine_call
from gm_b200.vae_api import engine_of, encoder_call, VaeFamilyModel, VaeFamilyTrainer


class Encoder(nn.Module):
    """ MLP encoder for VAE (src/vae.py:47-61). Input is an image, outputs are mu, log_var """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)
        self.log_var = nn.Linear(hidden_dim, z_dim)

    def forward(self, x):
        x = to_cuda(x).float()
        eng = engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # (mu, log_var) and their backward: gm_vae_encoder_forward / _backward
            return encoder_call(self, eng, x, eng.encoder_forward)
        _, mu, lv, _ = eng.forward(x, want_images=False)
        return mu, lv


class Decoder(nn.Module):
    """ MLP decoder for VAE (src/vae.py:64-77). Input is z, output is the reconstructed image """

    def __init__(self, z_dim, hidden_dim, image_size):
        super().__init__()
        self.linear = nn.Linear(z_dim, hidden_dim)
        self.recon = nn.Linear(hidden_dim, image_size)

    def forward(self, z):
        z = to_cuda(z)
        if z.dim() == 1:                       # the reference decodes single latent vectors too (src/vae.py:289-290)
            z = z.view(1, -1)
        eng = engine_of(self, "Decoder", z.shape[0])
        if torch.is_grad_enabled():                # the images and their backward, with dL/dz when z requires grad
            n = z.shape[0]

            def backward(slot, grads, need_dz):
                return eng.decoder_backward(slot, n, grads[0], need_dz)
            return engine_call(eng, "Decoder", eng.num_slots(), z.float(), self.named_parameters("decoder"),
                               eng.decoder_forward, backward)
        return eng.decode(z)


class VAE(VaeFamilyModel):
    """ VAE super class to reconstruct an image (src/vae.py:80-106) """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.shape = int(image_size ** 0.5)
        self._link()

    def _make_engine(self, max_batch):
        return VaeEngine(self.image_size, self.hidden_dim, self.z_dim, max_batch=max_batch)

    def forward(self, x):
        x = to_cuda(x).float()
        if torch.is_grad_enabled():                                  # src/vae.py:94-98 on the differentiable encoder / decoder
            mu, log_var = self.encoder(x)
            z = self.reparameterize(mu, log_var)
            return self.decoder(z), mu, log_var
        eng = self._engine_for(x.shape[0])
        eps = to_cuda(torch.randn(x.shape[0], self.z_dim))          # src/vae.py:104
        out, mu, lv, _ = eng.forward(x, eps=eps)
        return out, mu, lv

    def reparameterize(self, mu, log_var):
        """ z = mean + std * epsilon (src/vae.py:100-106); plain torch for direct use """
        epsilon = to_cuda(torch.randn(mu.shape))
        return mu + epsilon * torch.exp(log_var / 2)


class VAETrainer(VaeFamilyTrainer):
    def _resident_step(self, eng, hp, row, rows, epoch, k):
        row.copy_(eng.grad(self._resident.bits, fmt="bits", batch=rows, seed=self._seed, step=k))
        eng.apply(hp)

    def kl_divergence(self, mu, log_var):
        """ src/vae.py:210-212 (torch, for direct use) """
        return torch.sum(0.5 * (mu ** 2 + torch.exp(log_var) - log_var - 1))

    def sample_interpolated_images(self):
        """ Viz method 2 (src/vae.py:278-293): decode the interpolation between two random latent vectors; returns the
        list of decoded images instead of displaying them """
        z1 = torch.normal(torch.zeros(self.model.z_dim), 1)
        z2 = torch.normal(torch.zeros(self.model.z_dim), 1)
        out = []
        for alpha in np.linspace(0, 1, self.model.z_dim):
            z = to_cuda(float(alpha) * z1 + (1 - float(alpha)) * z2)
            with torch.no_grad():
                out.append(self.model.decoder(z).view(-1, self.model.shape, self.model.shape))
        return out

    def explore_latent_space(self, num_epochs=3):
        """ Viz method 3 (src/vae.py:295-338): train a VAE with a 2-d latent space, collect the variational means of the
        train split and decode a 10 x 10 grid of latent points; returns the trained (best) model, and keeps the means /
        grid samples in self.latent_means / self.latent_grid instead of plotting them """
        train_iter, val_iter, test_iter = get_data()                                   # noqa: F405
        latent_model = VAE(image_size=784, hidden_dim=400, z_dim=2)
        latent_space = VAETrainer(latent_model, train_iter, val_iter, test_iter)
        latent_space.train(num_epochs)
        latent_model = latent_space.best_model
        data = []
        for images, labels in train_iter:
            mu, _ = latent_model.encoder(to_cuda(images.view(images.shape[0], -1)))
            data.append(torch.cat([labels.view(-1, 1).float(), mu.cpu()], dim=1))
        self.latent_means = torch.cat(data)
        mu = torch.stack([torch.FloatTensor([m1, m2]) for m1 in np.linspace(-2, 2, 10) for m2 in np.linspace(-2, 2, 10)])
        self.latent_grid = latent_model.decoder(to_cuda(mu)).view(mu.shape[0], -1, latent_model.shape, latent_model.shape)
        return latent_model

    def make_all(self):
        """ Execute all latent space viz methods outlined in this class (src/vae.py:340-350) """
        print('Sampled images from latent space:')
        self.sample_images(save=False)
        print('Interpolating between two randomly sampled')
        self.sample_interpolated_images()
        print('Exploring latent representations')
        _ = self.explore_latent_space()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()
    model = VAE(image_size=784, hidden_dim=400, z_dim=20)
    trainer = VAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
