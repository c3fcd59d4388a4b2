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

from gm_b200 import AdamHP, AeEngine, GmError
from gm_b200.gan_api import (to_cuda, builtin_step, has_custom_compute_batch, refuse_multi_rank, compute_batch_loop,
                             compute_batch_evaluate, engine_call, GradHandoff, grow_engine)


class Encoder(nn.Module):
    """ Feedforward network encoder (src/ae.py:28-38) """

    def __init__(self, image_size, hidden_dim):
        super().__init__()
        self.linear = nn.Linear(image_size, hidden_dim)

    def forward(self, x):
        eng, attached = _engine_of(self, "Encoder", x.shape[0])
        if attached and torch.is_grad_enabled():   # the code relu(linear(x)) and its backward on the CUDA kernels
            n = x.shape[0]

            def backward(slot, grads, need_dx):
                if need_dx:
                    raise RuntimeError("the gradient with respect to the encoder's input is not computed")
                return eng.encoder_backward(slot, n, grads[0]), None
            return engine_call(eng, "Encoder", eng.SLOTS, to_cuda(x).float(), self.named_parameters("encoder"),
                               eng.encoder_forward, backward)
        return eng.encode(to_cuda(x).float())


class Decoder(nn.Module):
    """ Feedforward network decoder (src/ae.py:40-50) """

    def __init__(self, hidden_dim, image_size):
        super().__init__()
        self.linear = nn.Linear(hidden_dim, image_size)

    def forward(self, encoder_output):
        eng, attached = _engine_of(self, "Decoder", encoder_output.shape[0])
        if attached and torch.is_grad_enabled():   # sigmoid(linear(code)) and its backward, with dL/dcode when the code requires grad
            n = encoder_output.shape[0]

            def backward(slot, grads, need_dcode):
                g, dcode = eng.decoder_backward(slot, n, grads[0])
                return g, (dcode if need_dcode else None)
            return engine_call(eng, "Decoder", eng.SLOTS, to_cuda(encoder_output).float(), self.named_parameters("decoder"),
                               eng.decoder_forward, backward)
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
        m = self.model
        return grow_engine(self, batch, lambda rows: AeEngine(m.image_size, m.hidden_dim, max_batch=rows))

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
        gviews = eng.views(eng.grads)
        pairs = [(p, gviews[k]) for k, p in self.model.named_parameters()]
        return GradHandoff.apply(loss.detach().requires_grad_(True), loss, pairs)

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
