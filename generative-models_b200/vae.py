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

from gm_b200 import AdamHP, GmError, VaeEngine
from gm_b200.gan_api import (to_cuda, builtin_step, has_custom_compute_batch, refuse_multi_rank, compute_batch_loop,
                             compute_batch_evaluate, slot_ring, EngineCall, GradHandoff, grow_engine)


def _engine_of(module, what, batch):
    """The engine behind an Encoder / Decoder: the Trainer's (grown on demand), or - for a detached copy such as
    VAETrainer.best_model - a private inference engine built lazily from the copy's own parameters."""
    parent = module._parent() if getattr(module, "_parent", None) is not None else None
    if parent is None:
        raise GmError(what + " is not part of a VAE: construct it through VAE(...)")
    return parent._engine_for(batch, what)


class Encoder(nn.Module):
    """ MLP encoder for VAE (src/vae.py:47-61). Input is an image, outputs are mu, log_var """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)
        self.log_var = nn.Linear(hidden_dim, z_dim)

    def forward(self, x):
        x = to_cuda(x).float()
        eng = _engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # (mu, log_var) and their backward: gm_vae_encoder_forward / _backward
            ring, n = slot_ring(eng, "Encoder", eng.num_slots()), x.shape[0]
            names, params = zip(*self.named_parameters())

            def forward(x):
                slot, gen = ring.take()
                return eng.encoder_forward(slot, x), (slot, gen)

            def backward(handle, grads, need_dx):
                if need_dx:
                    raise RuntimeError("the gradient with respect to the encoder's input is not computed")
                ring.check(*handle)
                g = eng.encoder_backward(handle[0], n, *grads)
                return None, [g["encoder." + k] for k in names]
            return EngineCall.apply(x, forward, backward, *params)
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
        eng = _engine_of(self, "Decoder", z.shape[0])
        if torch.is_grad_enabled():                # the images and their backward, with dL/dz when z requires grad
            ring, n = slot_ring(eng, "Decoder", eng.num_slots()), z.shape[0]
            names, params = zip(*self.named_parameters())

            def forward(z):
                slot, gen = ring.take()
                return eng.decoder_forward(slot, z), (slot, gen)

            def backward(handle, grads, need_dz):
                ring.check(*handle)
                g, dz = eng.decoder_backward(handle[0], n, grads[0], need_dz)
                return dz, [g["decoder." + k] for k in names]
            return EngineCall.apply(z.float(), forward, backward, *params)
        return eng.decode(z)


class VAE(nn.Module):
    """ VAE super class to reconstruct an image (src/vae.py:80-106) """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.shape = int(image_size ** 0.5)
        import weakref
        for mod in (self.encoder, self.decoder):
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the VAETrainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _engine_for(self, batch, what="VAE"):
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            eng = owner._ensure_engine(batch)
            eng.sync_all()
            return eng
        if not torch.cuda.is_available():
            raise GmError(what + " is not attached to a CUDA engine yet: construct the VAETrainer first "
                          "(there is no eager/CPU path)")
        eng = self._own_engine
        if eng is None or batch > eng.max_batch:
            eng = VaeEngine(self.image_size, self.hidden_dim, self.z_dim, max_batch=max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (the reference keeps `best_model = deepcopy(model)`, src/vae.py:178-180): same class, cloned
        parameter values, no link to the Trainer's engine - its encoder / decoder run on a private engine built on use."""
        new = VAE(self.image_size, self.hidden_dim, self.z_dim)
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        new.train(self.training)
        return new

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


class VAETrainer:
    device_noise = True        # in-kernel Philox eps + resident dataset in train(); False: the reference's host draws

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model (src/vae.py:109-125) """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, _ = next(iter(test_iter))
        self.viz = viz
        self.kl_loss, self.recon_loss = [], []
        self.num_epochs = 0
        self._engine, self._max_batch, self._step = None, 0, 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        import weakref
        object.__setattr__(model, "_owner", weakref.ref(self))

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        m = self.model
        return grow_engine(self, batch, lambda rows: VaeEngine(m.image_size, m.hidden_dim, m.z_dim, max_batch=rows))

    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train a Variational Autoencoder (src/vae.py:127-191): a true epoch over train_iter,
        losses read back once per epoch, validation with the forward-only kernels, best model kept.  A subclass's own
        compute_batch (README.md:31) is trained by the reference loop over the differentiable encoder / decoder instead
        (gan_api.compute_batch_loop; train_iter is read on the host, device_noise does not apply). """
        if has_custom_compute_batch(self):
            refuse_multi_rank()
            return compute_batch_loop(self, num_epochs, lr, weight_decay, two_losses=True)
        hp = AdamHP.make(lr, weight_decay=weight_decay)
        if self._engine is not None:
            self._engine.reset_optimizer()
            self._engine.sync_all()
        # fast path (default): the train split packed to 1 bit/pixel in HBM once, batches drawn by the in-kernel epoch
        # sampler, eps by in-kernel Philox, gradient gather fused into Adam - no host work per step.  `device_noise =
        # False` (or a non-binary / non-TensorDataset loader) keeps the reference's host draws (torch.manual_seed replay).
        from gm_b200.gan_api import DeviceDataset
        resident = DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None)) if self.device_noise else None
        self._resident = resident
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            per_step = []
            if resident is not None:
                bs = min(resident.batch_size, resident.n)
                nb = len(resident)
                eng = self._ensure_engine(bs)
                eng.set_lazy_grads(True)
                eng.set_sampler(resident.n, nb, self._seed + 7919 * epoch, batch_size=bs)
                ring = torch.zeros(nb, 2, device="cuda")
                try:
                    for k in range(nb):
                        rows = min(bs, resident.n - k * bs)                        # the last batch of an epoch may be short
                        ring[k].copy_(eng.grad(resident.bits, fmt="bits", batch=rows, seed=self._seed, step=k))
                        eng.apply(hp)
                        self._step += 1
                finally:
                    eng.set_lazy_grads(False)
                    eng.set_sampler(0, 0, 0)
                vals = ring.tolist()
            else:
                for batch in self.train_iter:
                    images = self._images(batch)
                    eng = self._ensure_engine(images.shape[0])
                    eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))      # src/vae.py:104
                    per_step.append(eng.grad(images, eps=eps, seed=self._seed, step=self._step).clone())
                    eng.apply(hp)
                    self._step += 1
                vals = torch.stack(per_step).tolist()
            epoch_recon, epoch_kl = [v[0] for v in vals], [v[1] for v in vals]
            epoch_loss = [a + b for a, b in zip(epoch_recon, epoch_kl)]
            self.kl_loss.extend(epoch_kl)
            self.recon_loss.extend(epoch_recon)
            self.model.eval()
            val_loss = self.evaluate(self.val_iter)
            if val_loss < self.best_val_loss:
                self.best_model = deepcopy(self.model)                  # a detached module copy, like src/vae.py:178-180
                self.best_val_loss = val_loss
            print("Epoch[%d/%d], Total Loss: %.4f, Reconst Loss: %.4f, KL Div: %.7f, Val Loss: %.4f"
                  % (epoch, num_epochs, np.mean(epoch_loss), np.mean(epoch_recon), np.mean(epoch_kl), val_loss))
            self.num_epochs += 1
            if self.viz:
                self.sample_images(epoch)

    def _images(self, batch):
        images, _ = batch
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of examples (src/vae.py:193-208): returns (recon, kl); calling
        (recon + kl).backward() delivers the gradient of their sum, as in src/vae.py:158-161. """
        images = self._images(batch)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))
        losses = eng.grad(images, eps=eps, seed=self._seed, step=self._step).clone()
        self._step += 1
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters()]
        anchor = losses.detach().requires_grad_(True)
        # the fused kernels produced d(recon + kl)/dtheta once: the recon term delivers it, the kl term nothing (the
        # reference always back-propagates their sum)
        return GradHandoff.apply(anchor, losses[0], pairs), GradHandoff.apply(anchor, losses[1], [])

    def kl_divergence(self, mu, log_var):
        """ src/vae.py:210-212 (torch, for direct use) """
        return torch.sum(0.5 * (mu ** 2 + torch.exp(log_var) - log_var - 1))

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/vae.py:214-223) with the forward-only kernels, or with an overriding
        compute_batch as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, two_losses=True)
        loss = []
        with torch.no_grad():
            for batch in iterator:
                images = self._images(batch)
                eng = self._ensure_engine(images.shape[0])
                eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))
                _, _, _, ls = eng.forward(images, eps=eps, want_images=False, want_latent=False, want_losses=True)
                loss.append(ls.sum())
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ src/vae.py:225-252 without the plotting """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images, _, _ = self.model(batch)
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True):
        """ Viz method 1 (src/vae.py:254-276): z ~ p(z), x ~ p(x|z) """
        z = to_cuda(torch.randn(num_images, self.model.z_dim))
        with torch.no_grad():
            sample = self.model.decoder(z)
        return sample.view(num_images, self.model.shape, self.model.shape)

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

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.recon_loss)), self.recon_loss, "r")
        plt.plot(np.linspace(1, self.num_epochs, len(self.kl_loss)), self.kl_loss, "g")
        plt.legend(["Reconstruction", "Kullback-Leibler"])
        plt.title(self.name)
        plt.show()

    def save_model(self, savepath):
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        self.model.load_state_dict(torch.load(loadpath))
        if self._engine is not None:
            self._engine.sync_all()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()
    model = VAE(image_size=784, hidden_dim=400, z_dim=20)
    trainer = VAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
