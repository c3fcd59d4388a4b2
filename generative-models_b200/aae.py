""" (AAE) Adversarial autoencoder (Makhzani et al. 2015, arXiv:1511.05644) on the MLP VAE engine.

The reference's conventions (MLP, binary MNIST, Adam, `from aae import *`): a deterministic encoder
z = mu(relu(linear(x))) with bir_vae.py's parameter names, vae.py's decoder, and a latent discriminator Dz - the reference
GAN Discriminator on z-wide input - that outputs the probability that z came from the prior N(0, I).  One train step
per batch x runs three phases in this order, each on the parameters the previous one updated:

1. reconstruction: recon = sum((x - D(E(x)))^2), stepped by optimizer_R = Adam(encoder + decoder, lr, weight_decay);
2. discriminator: z_p ~ N(0, I), z_f = E(x) detached, D_loss = -mean(log(Dz(z_p) + 1e-8) + log(1 - Dz(z_f) + 1e-8)),
   stepped by optimizer_D = Adam(discriminator, D_lr);
3. regularisation: G_loss = -mean(log(Dz(E(x)) + 1e-8)), stepped by optimizer_G = Adam(encoder, G_lr), which keeps
   moments of its own for the encoder.

All three phases, their backward and the three Adams run in the hand-written sm_90a kernels of libgm_b200.so (the VAE
engine in its AAE mode; Dz on the GAN engine's D-step kernels).  train() keeps the train split resident (1 bit per
pixel) and draws every batch and prior sample on the device.  A subclass's own compute_batch, train_D or train_G is
trained by a plain loop over the differentiable model.encoder / model.decoder / model.discriminator nodes instead.
Data-parallel training is not offered.
"""
from copy import deepcopy  # noqa: F401

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403

import vae as _vae
from gm_b200 import AdamHP, GmError, AaeEngine
from gm_b200 import parallel as par
from gm_b200.gan_api import to_cuda, builtin_step, engine_call, GradHandoff, FusedAdam, compute_batch_evaluate
from gm_b200.vae_api import engine_of, encoder_call, VaeFamilyModel, VaeFamilyTrainer

EPOCH_LINE = "Epoch[%d/%d], Recon Loss: %.4f, D Loss: %.4f, G Loss: %.4f, Val Loss: %.4f"


class Encoder(nn.Module):
    """ MLP encoder for the AAE. Input is an image, output is the deterministic code z = mu(relu(linear(x))) """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)

    def forward(self, x):
        x = to_cuda(x).float()
        x = x.view(x.shape[0], -1)
        eng = engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # z and its backward: gm_vae_encoder_forward / _backward (AAE mode)
            return encoder_call(self, eng, x, eng.encoder_forward)
        _, z, _ = eng.forward(x, want_images=False)
        return z


class Decoder(_vae.Decoder):
    """ MLP decoder for the AAE: the VAE's decoder, z -> hidden -> image """


class Discriminator(nn.Module):
    """ Latent discriminator: the reference GAN Discriminator on z-wide input, z -> hidden (ReLU) -> 1 (sigmoid), the
    probability that z came from the prior """

    def __init__(self, z_dim, hidden_dim, output_dim=1):
        super().__init__()
        if output_dim != 1:
            raise GmError("the latent discriminator has one output (got output_dim=%d)" % output_dim)
        self.linear = nn.Linear(z_dim, hidden_dim)
        self.discriminate = nn.Linear(hidden_dim, output_dim)

    def forward(self, z):
        z = to_cuda(z).float()
        if z.dim() == 1:
            z = z.view(1, -1)
        eng = engine_of(self, "Discriminator", z.shape[0])
        n = z.shape[0]

        def forward(slot, z):                      # gm_aae_d_forward / _backward on one of the engine's D slots
            return eng.d_forward(slot, z).view(n, 1)

        def backward(slot, grads, need_dz):                # g: views of the D gradients, which the next call overwrites
            g, dz = eng.d_backward(slot, grads[0], need_dz)
            return {k: v.clone() for k, v in g.items()}, dz
        return engine_call(eng, "Discriminator", eng.num_d_slots(), z, self.named_parameters("discriminator"), forward,
                           backward)


class AAE(VaeFamilyModel):
    """ Adversarial autoencoder: encoder, decoder and the latent discriminator """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.discriminator = Discriminator(z_dim=z_dim, hidden_dim=hidden_dim, output_dim=1)
        self.shape = int(image_size ** 0.5)
        self._link()

    def _make_engine(self, max_batch):
        return AaeEngine(self.image_size, self.hidden_dim, self.z_dim, max_batch=max_batch)

    def forward(self, x):
        """ -> (out, z) """
        x = to_cuda(x).float()
        x = x.view(x.shape[0], -1)
        if torch.is_grad_enabled():                                  # the differentiable encoder / decoder
            z = self.encoder(x)
            return self.decoder(z), z
        eng = self._engine_for(x.shape[0])
        out, z, _ = eng.forward(x)
        return out, z


def has_custom_step(tr):
    """True when tr's class overrides compute_batch, train_D or train_G with a method not marked @builtin_step"""
    return any(not getattr(getattr(type(tr), m), "_gm_builtin", False) for m in ("compute_batch", "train_D", "train_G"))


def reference_loop(tr, num_epochs, lr, D_lr, G_lr, weight_decay):
    """The AAE step in plain torch over the differentiable nodes, for a trainer whose compute_batch, train_D or train_G
    was overridden: optimizer_R over encoder + decoder, optimizer_D over the discriminator and optimizer_G over the
    encoder, three FusedAdam instances (optimizer_G keeps moments of its own for the encoder)"""
    m = tr.model
    enc, dec, dis = ([p for p in mod.parameters() if p.requires_grad] for mod in (m.encoder, m.decoder, m.discriminator))
    optimizer_R = FusedAdam(enc + dec, lr=lr, weight_decay=weight_decay)
    optimizer_D = FusedAdam(dis, lr=D_lr)
    optimizer_G = FusedAdam(enc, lr=G_lr)
    for epoch in range(1, num_epochs + 1):
        m.train()
        epoch_recon, epoch_D, epoch_G = [], [], []
        for batch in tr.train_iter:
            optimizer_R.zero_grad()
            recon = tr.compute_batch(batch)
            recon.backward()
            optimizer_R.step()
            images = tr._images(batch)
            optimizer_D.zero_grad()
            D_loss = tr.train_D(images)
            D_loss.backward()
            optimizer_D.step()
            optimizer_G.zero_grad()
            G_loss = tr.train_G(images)
            G_loss.backward()
            optimizer_G.step()
            epoch_recon.append(recon.detach())
            epoch_D.append(D_loss.detach())
            epoch_G.append(G_loss.detach())
        tr._end_epoch(epoch, num_epochs, [torch.stack(v).tolist() for v in (epoch_recon, epoch_D, epoch_G)])


class AAETrainer(VaeFamilyTrainer):
    _losses = ("recon_loss", "Dlosses", "Glosses")
    _legend = ("Reconstruction", "Discriminator", "Generator")

    def _ensure_engine(self, batch):
        old = self._engine
        eng = super()._ensure_engine(batch)
        if old is not None and eng is not old:  # optimizer_D's and optimizer_G's state carries over as optimizer_R's does
            for name in ("d_exp_avg", "d_exp_avg_sq", "enc_g_exp_avg", "enc_g_exp_avg_sq"):
                getattr(eng, name).copy_(getattr(old, name))
            eng.d_steps, eng.g_steps = old.d_steps, old.g_steps
        return eng

    def train(self, num_epochs, lr=1e-3, D_lr=2e-4, G_lr=2e-4, weight_decay=1e-5):
        """ Train an AAE: per batch the reconstruction, discriminator and regularisation phases, each followed by its
        optimizer; a true epoch over train_iter, losses read back once per epoch, validation with the forward-only
        kernels, best model kept.  A subclass's own compute_batch, train_D or train_G is trained by the plain loop over
        the differentiable nodes instead.  One process only. """
        if par.world_size() > 1:
            raise GmError("the AAE trains on one process: there is no data-parallel AAE")
        if has_custom_step(self):
            return reference_loop(self, num_epochs, lr, D_lr, G_lr, weight_decay)
        self._train(num_epochs, (AdamHP.make(lr, weight_decay=weight_decay), AdamHP.make(D_lr), AdamHP.make(G_lr)))

    def _resident_step(self, eng, hp, row, rows, epoch, k):
        hpR, hpD, hpG = hp
        row[0:1].copy_(eng.recon_grad(self._resident.bits, fmt="bits", batch=rows, step=k))
        eng.apply(hpR)
        row[1:2].copy_(eng.d_grad(rows, seed=self._seed, step=self._step))
        eng.apply_d(hpD)
        row[2:3].copy_(eng.g_grad(rows))
        eng.apply_g(hpG)

    def _host_step(self, batch, hp):
        hpR, hpD, hpG = hp
        images = self._images(batch)
        n = images.shape[0]
        eng = self._ensure_engine(n)
        r = eng.recon_grad(images).clone()
        eng.apply(hpR)
        d = eng.d_grad(n, prior=to_cuda(torch.randn(n, self.model.z_dim))).clone()
        eng.apply_d(hpD)
        g = eng.g_grad(n).clone()
        eng.apply_g(hpG)
        return torch.cat([r, d, g])

    def _epoch_line(self, epoch, num_epochs, cols, val_loss):
        epoch_recon, epoch_D, epoch_G = cols
        return EPOCH_LINE % (epoch, num_epochs, np.mean(epoch_recon), np.mean(epoch_D), np.mean(epoch_G), val_loss)

    def _images(self, batch):
        """the images of a loader batch (or an image tensor) as [n, image_size] fp32 on the GPU"""
        images = batch[0] if isinstance(batch, (tuple, list)) else batch
        return to_cuda(images.reshape(images.shape[0], -1)).float().contiguous()

    @builtin_step
    def compute_batch(self, batch):
        """ Reconstruction loss of a batch: recon = sum((x - D(E(x)))^2); recon.backward() delivers its gradient to the
        encoder and decoder. """
        images = self._images(batch)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        recon = eng.recon_grad(images).clone()
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters() if not k.startswith("discriminator.")]
        return GradHandoff.apply(recon.detach().requires_grad_(True), recon[0], pairs)

    @builtin_step
    def train_D(self, images):
        """ D_loss = -mean(log(Dz(z_p) + 1e-8) + log(1 - Dz(z_f) + 1e-8)), z_p ~ N(0, I), z_f = E(x) detached """
        x = self._images(images)
        with torch.no_grad():
            z_f = self.model.encoder(x)
        z_p = to_cuda(torch.randn(x.shape[0], self.model.z_dim))
        return -torch.mean(torch.log(self.model.discriminator(z_p) + 1e-8) + torch.log(1 - self.model.discriminator(z_f) + 1e-8))

    @builtin_step
    def train_G(self, images):
        """ G_loss = -mean(log(Dz(E(x)) + 1e-8)) """
        x = self._images(images)
        return -torch.mean(torch.log(self.model.discriminator(self.model.encoder(x)) + 1e-8))

    def evaluate(self, iterator):
        """ Mean per-batch reconstruction loss over a dataset with the forward-only kernels, or with an overriding
        compute_batch """
        if not getattr(type(self).compute_batch, "_gm_builtin", False):
            return compute_batch_evaluate(self, iterator, two_losses=False)
        loss = []
        with torch.no_grad():
            for batch in iterator:
                images = self._images(batch)
                eng = self._ensure_engine(images.shape[0])
                _, _, ls = eng.forward(images, want_images=False, want_latent=False, want_losses=True)
                loss.append(ls[0])
        return float(torch.stack(loss).mean().item())


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()                                       # noqa: F405
    model = AAE(image_size=784, hidden_dim=400, z_dim=20)
    trainer = AAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=10, lr=1e-3, D_lr=2e-4, G_lr=2e-4, weight_decay=1e-5)
