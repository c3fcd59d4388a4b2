"""Host-side plumbing shared by the drop-ins on the MLP VAE engine (vae.py, cvae.py, bir_vae.py, aae.py): how a model's
modules find the engine, the detached copy a trainer keeps as best_model, and the trainer's engine growth, train()
epochs, validation and persistence.  A drop-in supplies its engine (the model's _make_engine), its train steps, its host
draws and its epoch line; gan_api.engine_call runs the grad-mode calls of its modules.
"""
import weakref
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from ._lib import AdamHP, GmError
from .gan_api import (to_cuda, builtin_step, has_custom_compute_batch, refuse_multi_rank, compute_batch_loop,
                      compute_batch_evaluate, engine_call, GradHandoff, grow_engine, DeviceDataset, VAE_EPOCH_LINE)


def engine_of(module, what, batch):
    """The engine behind an Encoder / Decoder / Discriminator: the Trainer's (grown on demand), or - for a detached copy
    such as VAETrainer.best_model - a private inference engine built lazily from the copy's own parameters."""
    parent = module._parent() if getattr(module, "_parent", None) is not None else None
    if parent is None:
        raise GmError(what + " is not part of a VAE: construct it through VAE(...)")
    return parent._engine_for(batch, what)


def encoder_call(module, eng, x, forward):
    """module, an Encoder, on x under grad mode: forward(slot, x) runs eng's per-call encoder kernels, the backward
    gm_vae_encoder_backward; the gradient with respect to x is not computed"""
    n = x.shape[0]

    def backward(slot, grads, need_dx):
        if need_dx:
            raise RuntimeError("the gradient with respect to the encoder's input is not computed")
        return eng.encoder_backward(slot, n, *grads), None
    return engine_call(eng, "Encoder", eng.num_slots(), x, module.named_parameters("encoder"), forward, backward)


class VaeFamilyModel(nn.Module):
    """A model on the MLP VAE engine.  The class that derives from this one directly (VAE, CVAE, BIRVAE, AAE) names the
    model: a detached copy is of that class, and an engine error names its Trainer.  A subclass builds its modules, then
    calls _link(), and implements _make_engine(max_batch)."""

    def __init_subclass__(cls, **kwargs):
        super().__init_subclass__(**kwargs)
        if VaeFamilyModel in cls.__bases__:
            cls._family = cls

    def _link(self):
        for mod in self.children():
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the Trainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _args(self):
        """the constructor arguments of a copy"""
        return self.image_size, self.hidden_dim, self.z_dim

    def _engine_for(self, batch, what=None):
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            eng = owner._ensure_engine(batch)
            eng.sync_all()
            return eng
        name = self._family.__name__
        if not torch.cuda.is_available():
            raise GmError("%s is not attached to a CUDA engine yet: construct the %sTrainer first (there is no eager/CPU "
                          "path)" % (what or name, name))
        eng = self._own_engine
        if eng is None or batch > eng.max_batch:
            eng = self._make_engine(max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (the reference keeps `best_model = deepcopy(model)`, src/vae.py:178-180): the model's class,
        cloned parameter values, no link to the Trainer's engine - its modules run on a private engine built on use."""
        new = self._family(*self._args())
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        new.train(self.training)
        return new


class VaeFamilyTrainer:
    """The Trainer of a VaeFamilyModel.  A subclass implements _resident_step(eng, hp, row, rows, epoch, k): the built-in
    step on batch k (rows images) of the resident train split, its losses written into row.  Where its engine's calls
    differ from the VAE's it overrides the hooks that make them (_inputs, _draws, _host_step, _epoch_line, ...)."""
    device_noise = True        # in-kernel noise + resident dataset in train(); False: the reference's host draws
    _losses = ("recon_loss", "kl_loss")                 # the per-step loss lists, in the engine's loss order
    _legend = ("Reconstruction", "Kullback-Leibler")
    _line = VAE_EPOCH_LINE     # formats (epoch, epochs, total, first loss, second loss, validation loss)

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model (src/vae.py:109-125) """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self._keep_debugging_batch(next(iter(test_iter)))
        self.viz = viz
        for name in self._losses:
            setattr(self, name, [])
        self.num_epochs = 0
        self._engine, self._max_batch, self._step = None, 0, 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        object.__setattr__(model, "_owner", weakref.ref(self))

    def _keep_debugging_batch(self, batch):
        self.debugging_image, _ = batch

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        return grow_engine(self, batch, self.model._make_engine)

    def _one_process(self):
        """raises when the model trains on one process only and a process group of more ranks runs; the default lets
        the built-in step run on every rank"""

    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train the model (src/vae.py:127-191): a true epoch over train_iter, losses read back once per epoch,
        validation with the forward-only kernels, best model kept.  A subclass's own compute_batch (README.md:31) is
        trained by the reference loop over the differentiable encoder / decoder instead (gan_api.compute_batch_loop;
        train_iter is read on the host, device_noise does not apply). """
        self._one_process()
        if has_custom_compute_batch(self):
            refuse_multi_rank()
            return compute_batch_loop(self, num_epochs, lr, weight_decay, two_losses=True, second=self._losses[1],
                                      epoch_line=self._line)
        self._train(num_epochs, AdamHP.make(lr, weight_decay=weight_decay))

    def _train(self, num_epochs, hp):
        """num_epochs of the built-in step; hp: what the step hooks pass to the engine's optimizer steps"""
        if self._engine is not None:
            self._engine.reset_optimizer()
            self._engine.sync_all()
        # fast path (default): the train split packed to 1 bit/pixel in HBM once, batches drawn by the in-kernel epoch
        # sampler, noise by in-kernel Philox, gradient gather fused into Adam - no host work per step.  `device_noise =
        # False` (or a non-binary / non-TensorDataset loader) keeps the reference's host draws (torch.manual_seed replay).
        resident = self._resident = self._device_dataset()
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            if resident is not None:
                bs = min(resident.batch_size, resident.n)
                nb = len(resident)
                eng = self._ensure_engine(bs)
                eng.set_lazy_grads(True)
                eng.set_sampler(resident.n, nb, self._seed + 7919 * epoch, batch_size=bs)
                ring = torch.zeros(nb, len(self._losses), device="cuda")
                try:
                    for k in range(nb):
                        rows = min(bs, resident.n - k * bs)                        # the last batch of an epoch may be short
                        self._resident_step(eng, hp, ring[k], rows, epoch, k)
                        self._step += 1
                finally:
                    eng.set_lazy_grads(False)
                    eng.set_sampler(0, 0, 0)
                cols = ring.t().tolist()
            else:
                per_step = []
                for batch in self.train_iter:
                    per_step.append(self._host_step(batch, hp))
                    self._step += 1
                cols = torch.stack(per_step).t().tolist()
            self._end_epoch(epoch, num_epochs, cols)

    def _device_dataset(self):
        """the train split resident on the device for the fast path, or None: train_iter is read on the host"""
        return DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None)) if self.device_noise else None

    def _host_step(self, batch, hp):
        """the built-in step on a loader batch with the host draws -> its losses"""
        inputs = self._inputs(batch)
        n = inputs[0].shape[0]
        eng = self._ensure_engine(n)
        losses = eng.grad(*inputs, **self._draws(n), seed=self._seed, step=self._step).clone()
        eng.apply(hp)
        return losses

    def _end_epoch(self, epoch, num_epochs, cols):
        """the loss lists (cols: each loss's per-step values), validation, best model and the epoch line"""
        for name, vals in zip(self._losses, cols):
            getattr(self, name).extend(vals)
        self.model.eval()
        val_loss = self.evaluate(self.val_iter)
        if val_loss < self.best_val_loss:
            self.best_model = deepcopy(self.model)                  # a detached module copy, like src/vae.py:178-180
            self.best_val_loss = val_loss
        print(self._epoch_line(epoch, num_epochs, cols, val_loss))
        self.num_epochs += 1
        if self.viz:
            self.sample_images(epoch)

    def _epoch_line(self, epoch, num_epochs, cols, val_loss):
        first, second = cols
        total = [a + b for a, b in zip(first, second)]
        return self._line % (epoch, num_epochs, np.mean(total), np.mean(first), np.mean(second), val_loss)

    def _images(self, batch):
        images, _ = batch
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    def _inputs(self, batch):
        """the engine's positional inputs for a loader batch"""
        return (self._images(batch),)

    def _draws(self, n):
        """the host draws of n rows, as keywords of the engine's grad / forward"""
        return {"eps": to_cuda(torch.randn(n, self.model.z_dim))}      # src/vae.py:104

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of examples (src/vae.py:193-208): returns (recon, kl); calling
        (recon + kl).backward() delivers the gradient of their sum, as in src/vae.py:158-161. """
        return self._fused_batch(batch)

    def _fused_batch(self, batch, **kw):
        """the built-in compute_batch: the fused step's two losses, whose backward() hands its gradients over"""
        inputs = self._inputs(batch)
        n = inputs[0].shape[0]
        eng = self._ensure_engine(n)
        eng.sync_all()
        losses = eng.grad(*inputs, **self._draws(n), **kw, seed=self._seed, step=self._step).clone()
        self._step += 1
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters()]
        anchor = losses.detach().requires_grad_(True)
        # the fused kernels produced d(first + second)/dtheta once: the first term delivers it, the second nothing (the
        # reference always back-propagates their sum)
        return GradHandoff.apply(anchor, losses[0], pairs), GradHandoff.apply(anchor, losses[1], [])

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/vae.py:214-223) with the forward-only kernels, or with an overriding
        compute_batch as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, two_losses=True)
        loss = []
        with torch.no_grad():
            for batch in iterator:
                inputs = self._inputs(batch)
                n = inputs[0].shape[0]
                eng = self._ensure_engine(n)
                ls = eng.forward(*inputs, **self._draws(n), want_images=False, want_latent=False, want_losses=True)[-1]
                loss.append(ls.sum())
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ src/vae.py:225-252 without the plotting: the reconstructions of images, shaped like images """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images = self.model(batch)[0]
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True):
        """ Viz method 1 (src/vae.py:254-276): z ~ p(z), x ~ p(x|z) """
        z = to_cuda(torch.randn(num_images, self.model.z_dim))
        with torch.no_grad():
            sample = self.model.decoder(z)
        return sample.view(num_images, self.model.shape, self.model.shape)

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        for name, color in zip(self._losses, "rgb"):
            vals = getattr(self, name)
            plt.plot(np.linspace(1, self.num_epochs, len(vals)), vals, color)
        plt.legend(list(self._legend))
        plt.title(self.name)
        plt.show()

    def save_model(self, savepath):
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        self.model.load_state_dict(torch.load(loadpath))
        if self._engine is not None:
            self._engine.sync_all()
