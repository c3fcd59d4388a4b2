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
from gm_b200 import AdamHP, GmError, BirVaeEngine, mmd_gaussian
from gm_b200.gan_api import (to_cuda, builtin_step, has_custom_compute_batch, compute_batch_loop,
                             compute_batch_evaluate, slot_ring, EngineCall, GradHandoff, grow_engine, first_order)

EPOCH_LINE = "Epoch[%d/%d], Total Loss: %.4f, MSE Loss: %.4f, MMD Loss: %.4f, Val Loss: %.4f"   # src/bir_vae.py:173


class Encoder(nn.Module):
    """ MLP encoder for BIR-VAE (src/bir_vae.py:36-48). Input is an image, output is mu """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)

    def forward(self, x):
        x = to_cuda(x).float()
        eng = _vae._engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # mu and its backward: gm_vae_encoder_forward / _backward (BIR mode)
            ring, n = slot_ring(eng, "Encoder", eng.num_slots()), x.shape[0]
            names, params = zip(*self.named_parameters())

            def forward(x):
                slot, gen = ring.take()
                return eng.encoder_forward(slot, x), (slot, gen)

            def backward(handle, grads, need_dx):
                if need_dx:
                    raise RuntimeError("the gradient with respect to the encoder's input is not computed")
                ring.check(*handle)
                g = eng.encoder_backward(handle[0], n, grads[0])
                return None, [g["encoder." + k] for k in names]
            return EngineCall.apply(x, forward, backward, *params)
        _, mu, _ = eng.forward(x, want_images=False)
        return mu


class Decoder(_vae.Decoder):
    """ MLP decoder for BIR-VAE (src/bir_vae.py:51-65): the VAE's decoder, z -> hidden -> image """


class BIRVAE(nn.Module):
    """ BIR-VAE (src/bir_vae.py:68-95). I: how many 'bits' are let through; eps has std set_var = 4^(-I / z_dim) """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, I=13.3):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, I=I))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.shape = int(image_size ** 0.5)
        self.set_var = 1 / (4 ** (I / z_dim))
        import weakref
        for mod in (self.encoder, self.decoder):
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the BIRVAETrainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _engine_for(self, batch, what="BIRVAE"):
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            eng = owner._ensure_engine(batch)
            eng.sync_all()
            return eng
        if not torch.cuda.is_available():
            raise GmError(what + " is not attached to a CUDA engine yet: construct the BIRVAETrainer first "
                          "(there is no eager/CPU path)")
        eng = self._own_engine
        if eng is None or batch > eng.max_batch:
            eng = BirVaeEngine(self.image_size, self.hidden_dim, self.z_dim, eps_std=self.set_var, max_batch=max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (best_model = deepcopy(model), src/bir_vae.py:161-163) with a private engine built on use"""
        new = BIRVAE(self.image_size, self.hidden_dim, self.z_dim, self.I)
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        new.train(self.training)
        return new

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


class BIRVAETrainer:
    device_noise = True        # in-kernel Philox eps / prior + resident dataset in train(); False: the reference's host draws

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model (src/bir_vae.py:98-114) """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, _ = next(iter(test_iter))
        self.viz = viz
        self.mmd_loss, self.recon_loss = [], []
        self.num_epochs = 0
        self._engine, self._max_batch, self._step = None, 0, 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        import weakref
        object.__setattr__(model, "_owner", weakref.ref(self))

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        m = self.model
        return grow_engine(self, batch, lambda rows: BirVaeEngine(m.image_size, m.hidden_dim, m.z_dim, eps_std=m.set_var,
                                                                  max_batch=rows))

    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train a BIR-VAE (src/bir_vae.py:116-176): a true epoch over train_iter, losses read back once per epoch,
        validation with the forward-only kernels, best model kept.  A subclass's own compute_batch is trained by the
        reference loop over the differentiable encoder / decoder instead.  One process only: the MMD couples every pair
        of the batch, so there is no data-parallel BIR-VAE. """
        from gm_b200 import parallel as par
        if par.world_size() > 1:
            raise GmError("BIR-VAE trains on one process: the MMD couples every pair of the batch, so there is no "
                          "data-parallel BIR-VAE")
        if has_custom_compute_batch(self):
            return compute_batch_loop(self, num_epochs, lr, weight_decay, two_losses=True, second="mmd_loss",
                                      epoch_line=EPOCH_LINE)
        hp = AdamHP.make(lr, weight_decay=weight_decay)
        if self._engine is not None:
            self._engine.reset_optimizer()
            self._engine.sync_all()
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
                        rows = min(bs, resident.n - k * bs)
                        ring[k].copy_(eng.grad(resident.bits, fmt="bits", batch=rows, seed=self._seed + 104729 * epoch, step=k))
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
                    eps, prior = self._draws(images.shape[0])
                    per_step.append(eng.grad(images, eps=eps, prior=prior, seed=self._seed, step=self._step).clone())
                    eng.apply(hp)
                    self._step += 1
                vals = torch.stack(per_step).tolist()
            epoch_recon, epoch_mmd = [v[0] for v in vals], [v[1] for v in vals]
            epoch_loss = [a + b for a, b in zip(epoch_recon, epoch_mmd)]
            self.mmd_loss.extend(epoch_mmd)
            self.recon_loss.extend(epoch_recon)
            self.model.eval()
            val_loss = self.evaluate(self.val_iter)
            if val_loss < self.best_val_loss:
                self.best_model = deepcopy(self.model)
                self.best_val_loss = val_loss
            print(EPOCH_LINE % (epoch, num_epochs, np.mean(epoch_loss), np.mean(epoch_recon), np.mean(epoch_mmd), val_loss))
            self.num_epochs += 1
            if self.viz:
                self.sample_images(epoch)

    def _images(self, batch):
        images, _ = batch
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    def _draws(self, n):
        """the reference's host draws in its order: eps = np.random.normal(0, set_var) in reparameterize, then the prior
        sample torch.randn(z.shape) in maximum_mean_discrepancy (src/bir_vae.py:91,192), both moved to the GPU"""
        eps = torch.from_numpy(np.random.normal(loc=0.0, scale=self.model.set_var, size=(n, self.model.z_dim))).float()
        prior = torch.randn(n, self.model.z_dim)
        return to_cuda(eps), to_cuda(prior)

    @builtin_step
    def compute_batch(self, batch, LAMBDA=1000.):
        """ Compute loss for a batch of examples (src/bir_vae.py:178-196): returns (mse_loss, mmd_loss); calling
        (mse_loss + mmd_loss).backward() delivers the gradient of their sum, as in src/bir_vae.py:144-148. """
        images = self._images(batch)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        eps, prior = self._draws(images.shape[0])
        losses = eng.grad(images, eps=eps, prior=prior, lam=LAMBDA, seed=self._seed, step=self._step).clone()
        self._step += 1
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters()]
        anchor = losses.detach().requires_grad_(True)
        return GradHandoff.apply(anchor, losses[0], pairs), GradHandoff.apply(anchor, losses[1], [])

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

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/bir_vae.py:213-221) with the forward-only kernels, or with an overriding
        compute_batch as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, two_losses=True)
        loss = []
        with torch.no_grad():
            for batch in iterator:
                images = self._images(batch)
                eng = self._ensure_engine(images.shape[0])
                eps, prior = self._draws(images.shape[0])
                _, _, ls = eng.forward(images, eps=eps, prior=prior, want_images=False, want_latent=False, want_losses=True)
                loss.append(ls.sum())
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ src/bir_vae.py:223-250 without the plotting """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images, _ = self.model(batch)
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True):
        """ Viz method 1 (src/bir_vae.py:252-273): z ~ p(z), x ~ p(x|z) """
        z = to_cuda(torch.randn(num_images, self.model.z_dim))
        with torch.no_grad():
            sample = self.model.decoder(z)
        return sample.view(num_images, self.model.shape, self.model.shape)

    def sample_interpolated_images(self):
        """ Viz method 2 (src/bir_vae.py:275-290): the decoded interpolation between two random latent vectors, returned
        instead of displayed """
        z1 = torch.normal(torch.zeros(self.model.z_dim), 1)
        z2 = torch.normal(torch.zeros(self.model.z_dim), 1)
        out = []
        for alpha in np.linspace(0, 1, self.model.z_dim):
            z = to_cuda(float(alpha) * z1 + (1 - float(alpha)) * z2)
            with torch.no_grad():
                out.append(self.model.decoder(z).view(-1, self.model.shape, self.model.shape))
        return out

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

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.recon_loss)), self.recon_loss, "r")
        plt.plot(np.linspace(1, self.num_epochs, len(self.mmd_loss)), self.mmd_loss, "g")
        plt.legend(["Reconstruction", "Maximum Mean Discrepancy"])
        plt.title(self.name)
        plt.show()

    def save_model(self, savepath):
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        self.model.load_state_dict(torch.load(loadpath))
        if self._engine is not None:
            self._engine.sync_all()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()                                       # noqa: F405
    model = BIRVAE(image_size=784, hidden_dim=400, z_dim=20, I=13.3)
    trainer = BIRVAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=10, lr=1e-3, weight_decay=1e-5)
