""" (AE) Standard autoencoder — drop-in for the reference's src/ae.py.

Same classes and signatures (src/ae.py:28-240): Encoder (784 -> hidden, ReLU), Decoder (hidden -> 784, sigmoid),
Autoencoder, AutoencoderTrainer with train / compute_batch / evaluate / reconstruct_images / viz_loss / save_model /
load_model and the attributes recon_loss, best_val_loss, num_epochs.  The loss follows the reference code: the sum of
squared errors (src/ae.py:158).  Forward, loss, backward and Adam run in the sm_90a kernels behind gm_b200.AeEngine.
"""
import weakref
from copy import deepcopy  # noqa: F401

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from torch.autograd.function import once_differentiable

from gm_b200 import AdamHP, AeEngine, GmError
from gm_b200.gan_api import (to_cuda, builtin_step, first_order, has_custom_compute_batch, refuse_multi_rank, compute_batch_loop,
                             compute_batch_evaluate, SlotRing)


def _ring(eng, what):
    """the engine's SlotRing of per-call Encoder / Decoder slots"""
    rings = eng.__dict__.setdefault("rings", {})
    if what not in rings:
        rings[what] = SlotRing(eng.SLOTS, what)
    return rings[what]


class _EncoderCall(torch.autograd.Function):
    """Encoder.forward under grad mode: the code relu(linear(x)) and its backward on the CUDA kernels
    (AeEngine.encoder_forward / encoder_backward); autograd routes dL/dcode in and the parameter gradients out"""

    @staticmethod
    def forward(ctx, x, eng, *params):
        ctx.slot, ctx.gen = _ring(eng, "Encoder").take()
        ctx.eng, ctx.n = eng, x.shape[0]
        return eng.encoder_forward(ctx.slot, x)

    @staticmethod
    @first_order
    @once_differentiable
    def backward(ctx, dcode):
        if ctx.needs_input_grad[0]:
            raise RuntimeError("the gradient with respect to the encoder's input is not computed")
        _ring(ctx.eng, "Encoder").check(ctx.slot, ctx.gen)
        g = ctx.eng.encoder_backward(ctx.slot, ctx.n, dcode)
        return None, None, g["encoder.linear.weight"], g["encoder.linear.bias"]


class _DecoderCall(torch.autograd.Function):
    """Decoder.forward under grad mode: sigmoid(linear(code)) and its backward, with dL/dcode when the code requires grad"""

    @staticmethod
    def forward(ctx, code, eng, *params):
        ctx.slot, ctx.gen = _ring(eng, "Decoder").take()
        ctx.eng, ctx.n = eng, code.shape[0]
        return eng.decoder_forward(ctx.slot, code)

    @staticmethod
    @first_order
    @once_differentiable
    def backward(ctx, dimages):
        _ring(ctx.eng, "Decoder").check(ctx.slot, ctx.gen)
        g, dcode = ctx.eng.decoder_backward(ctx.slot, ctx.n, dimages)
        return (dcode if ctx.needs_input_grad[0] else None), None, g["decoder.linear.weight"], g["decoder.linear.bias"]


class Encoder(nn.Module):
    """ Feedforward network encoder (src/ae.py:28-38) """

    def __init__(self, image_size, hidden_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)

    def forward(self, x):
        eng, attached = _engine_of(self, "Encoder", x.shape[0])
        if attached and torch.is_grad_enabled():
            return _EncoderCall.apply(to_cuda(x).float(), eng, self.linear.weight, self.linear.bias)
        return eng.encode(to_cuda(x).float())


class Decoder(nn.Module):
    """ Feedforward network decoder (src/ae.py:40-50) """

    def __init__(self, hidden_dim, image_size):
        super().__init__()
        self.linear = nn.Linear(hidden_dim, image_size)

    def forward(self, encoder_output):
        eng, attached = _engine_of(self, "Decoder", encoder_output.shape[0])
        if attached and torch.is_grad_enabled():
            return _DecoderCall.apply(to_cuda(encoder_output).float(), eng, self.linear.weight, self.linear.bias)
        return eng.decode(to_cuda(encoder_output).float())


def _engine_of(module, what, batch):
    """(the engine behind an Encoder / Decoder, whether it is a trainer's): the AutoencoderTrainer's (grown on demand), or -
    for a detached copy such as the best_model of an overridden compute_batch - the copy's private inference engine"""
    tr = getattr(module, "_owner", None)
    if tr is not None:
        return tr._ensure_engine(batch), True
    copy = module._copy_of() if getattr(module, "_copy_of", None) is not None else None
    if copy is None:
        raise GmError(what + " is not attached to a CUDA engine yet: construct the AutoencoderTrainer first (there is no eager/CPU path)")
    return copy._private_engine(batch), False


class Autoencoder(nn.Module):
    """ Autoencoder super class to encode then decode an image (src/ae.py:53-64) """

    def __init__(self, image_size=784, hidden_dim=32):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim)
        self.decoder = Decoder(hidden_dim=hidden_dim, image_size=image_size)

    def forward(self, x):
        eng, attached = _engine_of(self.encoder, "Autoencoder", x.shape[0])
        if attached and torch.is_grad_enabled():                # src/ae.py:63-64 on the differentiable encoder / decoder
            return self.decoder(self.encoder(x))
        out, _ = eng.forward(to_cuda(x).float())
        return out

    def _private_engine(self, batch):
        """the inference engine of a detached copy, loaded from the copy's own parameters on every call"""
        eng = getattr(self, "_own_engine", None)
        if eng is None or batch > eng.max_batch:
            eng = AeEngine(self.image_size, self.hidden_dim, max_batch=max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (the reference keeps best_model = deepcopy(model), src/ae.py:134): same class, cloned parameter
        values, no link to the trainer's engine; its encoder / decoder / forward run the inference calls on a private engine"""
        new = Autoencoder(self.image_size, self.hidden_dim)
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        for mod in (new.encoder, new.decoder):
            object.__setattr__(mod, "_copy_of", weakref.ref(new))
        new.train(self.training)
        return new


class _AeLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, anchor, val, holder):
        ctx.holder = holder
        return val.clone()

    @staticmethod
    def backward(ctx, gout):
        for p, g in ctx.holder():
            p.grad = g * gout if p.grad is None else p.grad + g * gout
        return None, None, None


class AutoencoderTrainer:
    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model (src/ae.py:67-82) """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, _ = next(iter(test_iter))
        self.viz = viz
        self.recon_loss = []
        self.num_epochs = 0
        self._engine, self._max_batch = None, 0
        for mod in (model.encoder, model.decoder):
            object.__setattr__(mod, "_owner", self)

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            self._engine.sync_all()
            return self._engine
        m, old = self.model, self._engine
        batch = max(batch, self._max_batch, 64)
        eng = AeEngine(m.image_size, m.hidden_dim, max_batch=batch)
        named = dict(m.named_parameters())
        eng.load({k: v.data for k, v in named.items()})
        views = eng.views()
        for k, p in named.items():
            p.data = views[k]                      # nn.Parameter storage == the engine's fp32 master weights
        if old is not None:
            eng.exp_avg.copy_(old.exp_avg)
            eng.exp_avg_sq.copy_(old.exp_avg_sq)
            eng.steps = old.steps
            for ring in getattr(old, "rings", {}).values():
                ring.retire()
        self._engine, self._max_batch = eng, batch
        return eng

    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train the autoencoder (src/ae.py:84-145): a true epoch over train_iter, losses read back once per epoch.  A
        subclass's own compute_batch (README.md:31) is trained by the reference loop over the differentiable encoder /
        decoder instead (gan_api.compute_batch_loop). """
        if has_custom_compute_batch(self):
            refuse_multi_rank()
            return compute_batch_loop(self, num_epochs, lr, weight_decay, two_losses=False)
        hp = AdamHP.make(lr, weight_decay=weight_decay)
        if self._engine is not None:
            self._engine.reset_optimizer()
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            per_step = []
            for batch in self.train_iter:
                images = self._images(batch)
                eng = self._ensure_engine(images.shape[0])
                per_step.append(eng.grad(images).clone())
                eng.apply(hp)
            epoch_loss = torch.stack(per_step).tolist()
            self.recon_loss.extend(epoch_loss)
            self.model.eval()
            val_loss = self.evaluate(self.val_iter)
            if val_loss < self.best_val_loss:
                self.best_model = deepcopy(self.model.state_dict())
                self.best_val_loss = val_loss
            print("Epoch[%d/%d], Train Loss: %.4f, Val Loss: %.4f" % (epoch, num_epochs, np.mean(epoch_loss), val_loss))
            self.num_epochs += 1

    def _images(self, batch):
        images, _ = batch
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of examples (src/ae.py:147-160): .backward() delivers the gradients """
        images = self._images(batch)
        eng = self._ensure_engine(images.shape[0])
        loss = eng.grad(images).clone()
        named = dict(self.model.named_parameters())
        gviews = eng.views(eng.grads)
        return _AeLoss.apply(loss.detach().requires_grad_(True), loss, lambda: [(named[k], gviews[k]) for k in named])

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/ae.py:162-164), with an overriding compute_batch as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, two_losses=False)
        vals = []
        with torch.no_grad():
            for batch in iterator:
                images = self._images(batch)
                _, loss = self._ensure_engine(images.shape[0]).forward(images, want_loss=True)
                vals.append(loss)
        return float(torch.stack(vals).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ Reconstruct a fixed input (src/ae.py:166-195 without the plotting) """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            return self.model(batch).view(images.shape).squeeze()

    def viz_loss(self):
        print("viz_loss: matplotlib is not installed")

    def save_model(self, savepath):
        """ Save model state dictionary (src/ae.py:213-215) """
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        """ Load state dictionary into model (src/ae.py:217-220) """
        self.model.load_state_dict(torch.load(loadpath))
        if self._engine is not None:
            self._engine.sync_all()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()  # noqa: F405
    model = Autoencoder(image_size=784, hidden_dim=32)
    trainer = AutoencoderTrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
