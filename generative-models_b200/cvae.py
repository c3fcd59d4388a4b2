""" (CVAE) Conditional variational autoencoder on the MLP VAE engine.

The standard conditional VAE (Sohn et al. 2015; the conditional decoder of Kingma et al. 2014's M2 model) built on
vae.py's model and loss: the encoder q(z | x, y) reads [x | onehot(y)], the decoder p(x | z, y) reads [z | onehot(y)],
z = mu + eps * exp(log_var / 2), recon = sum((x - out)^2), kl = sum(0.5 (mu^2 + exp(lv) - lv - 1)), Adam with coupled
weight decay.  The one-hot columns follow the x (z) columns, so only encoder.linear.weight [h, x + C] and
decoder.linear.weight [h, z + C] are wider than vae.py's; the state_dict keys are vae.py's.

Labels are integer class ids, as the loaders yield them; the one-hot is formed on the device by the staging and latent
kernels, and labels outside [0, C) raise GmError on the host before anything is uploaded.  Forward, both losses, the
backward and Adam run in the hand-written sm_90a kernels of libgm_b200.so (the VAE engine in its CVAE mode).  train()
keeps the train split resident (1 bit per pixel) with its labels beside it as int32, and draws every batch of
(image, label) pairs on the device.  A subclass's own compute_batch is trained by the reference loop over the
differentiable encoder / decoder.  Data-parallel training is not offered.
"""
from copy import deepcopy  # noqa: F401

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403

import vae as _vae
from gm_b200 import AdamHP, GmError, CvaeEngine
from gm_b200.engine import class_ids
from gm_b200.gan_api import (to_cuda, builtin_step, has_custom_compute_batch, compute_batch_loop, compute_batch_evaluate,
                             slot_ring, EngineCall, GradHandoff, grow_engine, VAE_EPOCH_LINE)

MAX_LATENT_ROW = 63          # z_dim + num_classes: the decoder's operand row [z | onehot(y) | 1] is one 64-wide row


def _labels(y, n):
    """y as a tensor of class ids for n rows: one class id is given to every row"""
    y = y if torch.is_tensor(y) else torch.as_tensor(np.asarray(y))
    return y.expand(n) if y.dim() == 0 else y


class Encoder(nn.Module):
    """ MLP encoder q(z | x, y). Input is an image and its class, outputs are mu, log_var """

    def __init__(self, image_size, hidden_dim, z_dim, num_classes):
        super().__init__()
        self.linear = nn.Linear(image_size + num_classes, hidden_dim)
        self.mu = nn.Linear(hidden_dim, z_dim)
        self.log_var = nn.Linear(hidden_dim, z_dim)

    def forward(self, x, y):
        x = to_cuda(x).float()
        x = x.view(x.shape[0], -1)
        eng = _vae._engine_of(self, "Encoder", x.shape[0])
        y = eng.class_ids(_labels(y, x.shape[0]), x.shape[0])
        if torch.is_grad_enabled():                # (mu, log_var) and their backward: gm_cvae_encoder_forward / gm_vae_encoder_backward
            ring, n = slot_ring(eng, "Encoder", eng.num_slots()), x.shape[0]
            names, params = zip(*self.named_parameters())

            def forward(x):
                slot, gen = ring.take()
                return eng.encoder_forward(slot, x, y), (slot, gen)

            def backward(handle, grads, need_dx):
                if need_dx:
                    raise RuntimeError("the gradient with respect to the encoder's input is not computed")
                ring.check(*handle)
                g = eng.encoder_backward(handle[0], n, *grads)
                return None, [g["encoder." + k] for k in names]
            return EngineCall.apply(x, forward, backward, *params)
        _, mu, lv, _ = eng.forward(x, y, want_images=False)
        return mu, lv


class Decoder(nn.Module):
    """ MLP decoder p(x | z, y). Input is z and a class, output is the reconstructed image """

    def __init__(self, z_dim, hidden_dim, image_size, num_classes):
        super().__init__()
        self.linear = nn.Linear(z_dim + num_classes, hidden_dim)
        self.recon = nn.Linear(hidden_dim, image_size)

    def forward(self, z, y):
        z = to_cuda(z)
        if z.dim() == 1:                       # a single latent vector
            z = z.view(1, -1)
        eng = _vae._engine_of(self, "Decoder", z.shape[0])
        y = eng.class_ids(_labels(y, z.shape[0]), z.shape[0])
        if torch.is_grad_enabled():                # the images and their backward, with dL/dz when z requires grad
            ring, n = slot_ring(eng, "Decoder", eng.num_slots()), z.shape[0]
            names, params = zip(*self.named_parameters())

            def forward(z):
                slot, gen = ring.take()
                return eng.decoder_forward(slot, z, y), (slot, gen)

            def backward(handle, grads, need_dz):
                ring.check(*handle)
                g, dz = eng.decoder_backward(handle[0], n, grads[0], need_dz)
                return dz, [g["decoder." + k] for k in names]
            return EngineCall.apply(z.float(), forward, backward, *params)
        return eng.decode(z, y)


class CVAE(nn.Module):
    """ Conditional VAE: reconstructs an image given its class, and samples images of a chosen class """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, num_classes=10):
        super().__init__()
        if int(num_classes) < 1:
            raise GmError("num_classes must be >= 1 (got %d)" % num_classes)
        if z_dim + num_classes > MAX_LATENT_ROW:
            raise GmError("z_dim + num_classes must be <= %d (got %d + %d)" % (MAX_LATENT_ROW, z_dim, num_classes))
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, num_classes=int(num_classes)))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, num_classes=num_classes)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size, num_classes=num_classes)
        self.shape = int(image_size ** 0.5)
        import weakref
        for mod in (self.encoder, self.decoder):
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the CVAETrainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _engine_for(self, batch, what="CVAE"):
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            eng = owner._ensure_engine(batch)
            eng.sync_all()
            return eng
        if not torch.cuda.is_available():
            raise GmError(what + " is not attached to a CUDA engine yet: construct the CVAETrainer first "
                          "(there is no eager/CPU path)")
        eng = self._own_engine
        if eng is None or batch > eng.max_batch:
            eng = CvaeEngine(self.image_size, self.hidden_dim, self.z_dim, self.num_classes, max_batch=max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (best_model): same class, cloned parameter values, its own inference engine built on use"""
        new = CVAE(self.image_size, self.hidden_dim, self.z_dim, self.num_classes)
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        new.train(self.training)
        return new

    def forward(self, x, y):
        """ -> (out, mu, log_var) of x given its classes y """
        x = to_cuda(x).float()
        x = x.view(x.shape[0], -1)
        if torch.is_grad_enabled():                                  # the differentiable encoder / decoder
            mu, log_var = self.encoder(x, y)
            z = self.reparameterize(mu, log_var)
            return self.decoder(z, y), mu, log_var
        eng = self._engine_for(x.shape[0])
        eps = to_cuda(torch.randn(x.shape[0], self.z_dim))
        out, mu, lv, _ = eng.forward(x, y, eps=eps)
        return out, mu, lv

    def reparameterize(self, mu, log_var):
        """ z = mean + std * epsilon (plain torch, for direct use) """
        epsilon = to_cuda(torch.randn(mu.shape))
        return mu + epsilon * torch.exp(log_var / 2)


class CVAETrainer:
    device_noise = True        # in-kernel Philox eps + resident dataset and labels in train(); False: host draws

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, self.debugging_labels = next(iter(test_iter))
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
        return grow_engine(self, batch, lambda rows: CvaeEngine(m.image_size, m.hidden_dim, m.z_dim, m.num_classes, max_batch=rows))

    def _resident_labels(self, resident):
        """the train split's labels, checked on the host and uploaded once as int32 beside resident.bits (None when the
        loader's dataset holds no label tensor: the host path runs)"""
        tensors = getattr(getattr(self.train_iter, "dataset", None), "tensors", None)
        if resident is None or tensors is None or len(tensors) < 2:
            return None
        cached = getattr(self, "_resident_y", None)
        if cached is not None and cached[0] is tensors[1]:
            return cached[1]
        y = class_ids(tensors[1], self.model.num_classes, torch.device("cuda", torch.cuda.current_device()), resident.n)
        self._resident_y = (tensors[1], y)
        return y

    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train a conditional VAE: a true epoch over train_iter, losses read back once per epoch, validation with the
        forward-only kernels, best model kept.  A subclass's own compute_batch is trained by the reference loop over the
        differentiable encoder / decoder instead.  One process only. """
        from gm_b200 import parallel as par
        if par.world_size() > 1:
            raise GmError("the CVAE trains on one process: there is no data-parallel CVAE")
        if has_custom_compute_batch(self):
            return compute_batch_loop(self, num_epochs, lr, weight_decay, two_losses=True)
        hp = AdamHP.make(lr, weight_decay=weight_decay)
        if self._engine is not None:
            self._engine.reset_optimizer()
            self._engine.sync_all()
        # fast path (default): the train split packed to 1 bit/pixel in HBM once and its labels as int32 beside it,
        # (image, label) pairs drawn by the in-kernel epoch sampler, eps by in-kernel Philox - no host work per step
        from gm_b200.gan_api import DeviceDataset
        resident = DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None)) if self.device_noise else None
        labels = self._resident_labels(resident)
        if labels is None:
            resident = None
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
                        ring[k].copy_(eng.grad(resident.bits, labels, fmt="bits", batch=rows, seed=self._seed, step=k))
                        eng.apply(hp)
                        self._step += 1
                finally:
                    eng.set_lazy_grads(False)
                    eng.set_sampler(0, 0, 0)
                vals = ring.tolist()
            else:
                for batch in self.train_iter:
                    images, y = self._batch(batch)
                    eng = self._ensure_engine(images.shape[0])
                    eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))
                    per_step.append(eng.grad(images, y, eps=eps, seed=self._seed, step=self._step).clone())
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
                self.best_model = deepcopy(self.model)                  # a detached module copy
                self.best_val_loss = val_loss
            print(VAE_EPOCH_LINE % (epoch, num_epochs, np.mean(epoch_loss), np.mean(epoch_recon), np.mean(epoch_kl), val_loss))
            self.num_epochs += 1
            if self.viz:
                self.sample_images(epoch)

    def _batch(self, batch):
        """(images [n, image_size] fp32 on the GPU, labels checked for the model's classes) of one loader batch"""
        images, labels = batch
        y = class_ids(labels, self.model.num_classes, torch.device("cuda", torch.cuda.current_device()), images.shape[0])
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous(), y

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of (images, labels): returns (recon, kl); calling (recon + kl).backward() delivers
        the gradient of their sum. """
        images, y = self._batch(batch)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))
        losses = eng.grad(images, y, eps=eps, seed=self._seed, step=self._step).clone()
        self._step += 1
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters()]
        anchor = losses.detach().requires_grad_(True)
        # the fused kernels produced d(recon + kl)/dtheta once: the recon term delivers it, the kl term nothing
        return GradHandoff.apply(anchor, losses[0], pairs), GradHandoff.apply(anchor, losses[1], [])

    def kl_divergence(self, mu, log_var):
        """ torch, for direct use """
        return torch.sum(0.5 * (mu ** 2 + torch.exp(log_var) - log_var - 1))

    def evaluate(self, iterator):
        """ Mean per-batch loss over a dataset with the forward-only kernels, or with an overriding compute_batch """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, two_losses=True)
        loss = []
        with torch.no_grad():
            for batch in iterator:
                images, y = self._batch(batch)
                eng = self._ensure_engine(images.shape[0])
                eps = to_cuda(torch.randn(images.shape[0], self.model.z_dim))
                _, _, _, ls = eng.forward(images, y, eps=eps, want_images=False, want_latent=False, want_losses=True)
                loss.append(ls.sum())
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, labels, epoch, save=True):
        """ the reconstructions of images given their labels, shaped like images (no plotting) """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images, _, _ = self.model(batch, labels)
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True, labels=None):
        """ z ~ p(z), x ~ p(x | z, y): labels (default arange(num_images) % num_classes) pick each image's class """
        if labels is None:
            labels = torch.arange(num_images) % self.model.num_classes
        z = to_cuda(torch.randn(num_images, self.model.z_dim))
        with torch.no_grad():
            sample = self.model.decoder(z, labels)
        return sample.view(num_images, self.model.shape, self.model.shape)

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
    train_iter, val_iter, test_iter = get_data()                                       # noqa: F405
    model = CVAE(image_size=784, hidden_dim=400, z_dim=20, num_classes=10)
    trainer = CVAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
