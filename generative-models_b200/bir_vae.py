""" (BIR-VAE) Bounded Information Rate VAE — drop-in for the reference's src/bir_vae.py.

Same classes and signatures (src/bir_vae.py:36-400).  The encoder has a single mu head; z = mu + eps with eps of a
fixed scale; the loss is mse = sum((x - out)^2) plus LAMBDA times the Gaussian-kernel maximum mean discrepancy of z
against a N(0, I) sample (src/bir_vae.py:178-222); Adam with coupled weight decay (src/bir_vae.py:127-129).  Forward,
both losses, the backward and Adam run in the hand-written sm_90a kernels of libgm_b200.so (the VAE engine in its BIR
mode; the MMD is one tiled kernel that never stores the batch x batch kernel matrix).

Decisions on the reference's quirks:
- eps is drawn with np.random.normal(0, scale=set_var) (src/bir_vae.py:91): numpy's scale is a standard deviation, so
  the noise std is set_var = 4^(-I / z_dim) itself, not its square root.  Kept as the reference computes it.
- maximum_mean_discrepancy draws its prior sample with torch.randn on the host (src/bir_vae.py:192), which fails against
  a CUDA z in the reference (device mismatch).  Here the sample is moved to z's device: the one deviation.
- train() calls compute_batch(batch) with its default LAMBDA = 1000 (src/bir_vae.py:148); another LAMBDA is trained by
  overriding compute_batch, which is honoured.
- Data-parallel training is not offered: the MMD couples every pair of the global batch.
"""
from copy import deepcopy  # noqa: F401

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403

import vae as _vae
from gm_b200 import GmError, BirVaeEngine, mmd_gaussian
from gm_b200 import parallel as par
from gm_b200.gan_api import to_cuda, builtin_step, first_order
from gm_b200.vae_api import engine_of, encoder_call, VaeFamilyModel, VaeFamilyTrainer

EPOCH_LINE = "Epoch[%d/%d], Total Loss: %.4f, MSE Loss: %.4f, MMD Loss: %.4f, Val Loss: %.4f"   # src/bir_vae.py:173


class Encoder(nn.Module):
    """ MLP encoder for BIR-VAE (src/bir_vae.py:36-48). Input is an image, output is mu """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)

    def forward(self, x):
        x = to_cuda(x).float()
        eng = engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # mu and its backward: gm_vae_encoder_forward / _backward (BIR mode)
            return encoder_call(self, eng, x, eng.encoder_forward)
        _, mu, _ = eng.forward(x, want_images=False)
        return mu


class Decoder(_vae.Decoder):
    """ MLP decoder for BIR-VAE (src/bir_vae.py:51-65): the VAE's decoder, z -> hidden -> image """


class BIRVAE(VaeFamilyModel):
    """ BIR-VAE (src/bir_vae.py:68-95). I: how many 'bits' are let through; eps has std set_var = 4^(-I / z_dim) """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, I=13.3):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, I=I))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.shape = int(image_size ** 0.5)
        self.set_var = 1 / (4 ** (I / z_dim))
        self._link()

    def _args(self):
        return self.image_size, self.hidden_dim, self.z_dim, self.I

    def _make_engine(self, max_batch):
        return BirVaeEngine(self.image_size, self.hidden_dim, self.z_dim, eps_std=self.set_var, max_batch=max_batch)

    def forward(self, x):
        """ src/bir_vae.py:84-88 on the engine-backed encoder / decoder: returns (out_img, z) """
        mu = self.encoder(to_cuda(x).float())
        z = self.reparameterize(mu)
        return self.decoder(z), z

    def reparameterize(self, mu):
        """ z = mu + eps, eps ~ np.random.normal(0, scale=set_var) (src/bir_vae.py:90-95) """
        eps = to_cuda(torch.from_numpy(np.random.normal(loc=0.0, scale=self.set_var, size=tuple(mu.shape))).float())
        return mu + eps


class _MMD(torch.autograd.Function):
    """mmd(z, p) with k(a, b) = exp(-|a - b|^2 / Z^2) on gm_mmd_gaussian; the backward is its dz times the upstream"""

    @staticmethod
    def forward(ctx, z, p):
        out, dz = mmd_gaussian(z.detach(), p, 1.0, want_grad=ctx.needs_input_grad[0])
        ctx.save_for_backward(dz if dz is not None else out)
        return out.view(())

    @staticmethod
    @first_order
    def backward(ctx, gout):
        (dz,) = ctx.saved_tensors
        return dz * gout, None


class BIRVAETrainer(VaeFamilyTrainer):
    _losses = ("recon_loss", "mmd_loss")
    _legend = ("Reconstruction", "Maximum Mean Discrepancy")
    _line = EPOCH_LINE

    def _one_process(self):
        """the MMD couples every pair of the batch, so there is no data-parallel BIR-VAE"""
        if par.world_size() > 1:
            raise GmError("BIR-VAE trains on one process: the MMD couples every pair of the batch, so there is no "
                          "data-parallel BIR-VAE")

    def _resident_step(self, eng, hp, row, rows, epoch, k):
        row.copy_(eng.grad(self._resident.bits, fmt="bits", batch=rows, seed=self._seed + 104729 * epoch, step=k))
        eng.apply(hp)

    def _draws(self, n):
        """the reference's host draws in its order: eps = np.random.normal(0, set_var) in reparameterize, then the prior
        sample torch.randn(z.shape) in maximum_mean_discrepancy (src/bir_vae.py:91,192), both moved to the GPU"""
        eps = torch.from_numpy(np.random.normal(loc=0.0, scale=self.model.set_var, size=(n, self.model.z_dim))).float()
        prior = torch.randn(n, self.model.z_dim)
        return {"eps": to_cuda(eps), "prior": to_cuda(prior)}

    @builtin_step
    def compute_batch(self, batch, LAMBDA=1000.):
        """ Compute loss for a batch of examples (src/bir_vae.py:178-196): returns (mse_loss, mmd_loss); calling
        (mse_loss + mmd_loss).backward() delivers the gradient of their sum, as in src/bir_vae.py:144-148. """
        return self._fused_batch(batch, lam=LAMBDA)

    def maximum_mean_discrepancy(self, z):
        """ Maximum mean discrepancy of a Gaussian kernel (src/bir_vae.py:190-197) as one autograd node over the tiled
        MMD kernel (no batch x batch tensor); the prior sample is drawn like the reference's, then moved to z's device """
        x = torch.randn(z.shape).to(z.device)
        return _MMD.apply(z.float(), x)

    def compute_kernel(self, x, y):
        """ Compute Gaussian kernel for MMD (src/bir_vae.py:199-211; torch, for direct use) """
        x_size, y_size, dim = x.size(0), y.size(0), x.size(1)
        x, y = x.unsqueeze(1), y.unsqueeze(0)
        tiled_x, tiled_y = x.expand(x_size, y_size, dim), y.expand(x_size, y_size, dim)
        kernel_input = torch.div(torch.mean(torch.pow(tiled_x - tiled_y, 2), dim=2), dim)
        return torch.exp(-kernel_input)

    sample_interpolated_images = _vae.VAETrainer.sample_interpolated_images     # src/bir_vae.py:275-290

    def explore_latent_space(self, num_epochs=3):
        """ Viz method 3 (src/bir_vae.py:292-335): train a z = 2 BIR-VAE, keep the train split's means in
        self.latent_means and a decoded 10 x 10 latent grid in self.latent_grid instead of plotting them """
        train_iter, val_iter, test_iter = get_data()                                   # noqa: F405
        latent_model = BIRVAE(image_size=784, hidden_dim=400, z_dim=2, I=13.3)
        latent_space = BIRVAETrainer(latent_model, train_iter, val_iter, test_iter)
        latent_space.train(num_epochs)
        latent_model = latent_space.best_model
        data = []
        with torch.no_grad():
            for images, labels in train_iter:
                mu = latent_model.encoder(to_cuda(images.view(images.shape[0], -1)))
                data.append(torch.cat([labels.view(-1, 1).float(), mu.cpu()], dim=1))
        self.latent_means = torch.cat(data)
        mu = torch.stack([torch.FloatTensor([m1, m2]) for m1 in np.linspace(-2, 2, 10) for m2 in np.linspace(-2, 2, 10)])
        with torch.no_grad():
            self.latent_grid = latent_model.decoder(to_cuda(mu)).view(mu.shape[0], -1, latent_model.shape, latent_model.shape)
        return latent_model

    def make_all(self):
        """ Execute all viz methods (src/bir_vae.py:337-347) """
        print('Sampling images from latent space...')
        self.sample_images(save=False)
        print('Interpolating between two randomly sampled...')
        self.sample_interpolated_images()
        print('Exploring latent representations...')
        _ = self.explore_latent_space()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()                                       # noqa: F405
    model = BIRVAE(image_size=784, hidden_dim=400, z_dim=20, I=13.3)
    trainer = BIRVAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=10, lr=1e-3, weight_decay=1e-5)
