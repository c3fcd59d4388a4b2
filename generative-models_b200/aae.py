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
from gm_b200.gan_api import (to_cuda, builtin_step, slot_ring, EngineCall, GradHandoff, grow_engine, FusedAdam,
                             compute_batch_evaluate)

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
        eng = _vae._engine_of(self, "Encoder", x.shape[0])
        if torch.is_grad_enabled():                # z and its backward: gm_vae_encoder_forward / _backward (AAE mode)
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
        eng = _vae._engine_of(self, "Discriminator", z.shape[0])
        ring, n = slot_ring(eng, "Discriminator", eng.num_d_slots()), z.shape[0]
        names, params = zip(*self.named_parameters())

        def forward(z):                            # gm_aae_d_forward / _backward on one of the engine's D slots
            slot, gen = ring.take()
            return eng.d_forward(slot, z).view(n, 1), (slot, gen)

        def backward(handle, grads, need_dz):
            ring.check(*handle)
            g, dz = eng.d_backward(handle[0], grads[0], need_dz)
            return dz, [g["discriminator." + k].clone() for k in names]
        return EngineCall.apply(z, forward, backward, *params)


class AAE(nn.Module):
    """ Adversarial autoencoder: encoder, decoder and the latent discriminator """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim))
        self.encoder = Encoder(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim)
        self.decoder = Decoder(z_dim=z_dim, hidden_dim=hidden_dim, image_size=image_size)
        self.discriminator = Discriminator(z_dim=z_dim, hidden_dim=hidden_dim, output_dim=1)
        self.shape = int(image_size ** 0.5)
        import weakref
        for mod in (self.encoder, self.decoder, self.discriminator):
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the AAETrainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _engine_for(self, batch, what="AAE"):
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            eng = owner._ensure_engine(batch)
            eng.sync_all()
            return eng
        if not torch.cuda.is_available():
            raise GmError(what + " is not attached to a CUDA engine yet: construct the AAETrainer first "
                          "(there is no eager/CPU path)")
        eng = self._own_engine
        if eng is None or batch > eng.max_batch:
            eng = AaeEngine(self.image_size, self.hidden_dim, self.z_dim, max_batch=max(batch, 64))
            object.__setattr__(self, "_own_engine", eng)
        eng.load({k: v.data for k, v in self.named_parameters()})
        return eng

    def __deepcopy__(self, memo):
        """A detached copy (best_model): same class, cloned parameter values, its own inference engine built on use"""
        new = AAE(self.image_size, self.hidden_dim, self.z_dim)
        with torch.no_grad():
            for (_, a), (_, b) in zip(new.named_parameters(), self.named_parameters()):
                a.copy_(b.detach().cpu())
        new.train(self.training)
        return new

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


class AAETrainer:
    device_noise = True        # resident dataset and in-kernel prior draws in train(); False: host batches and prior

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        """ Object to hold data iterators, train the model """
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, _ = next(iter(test_iter))
        self.viz = viz
        self.recon_loss, self.Dlosses, self.Glosses = [], [], []
        self.num_epochs = 0
        self._engine, self._max_batch, self._step = None, 0, 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        import weakref
        object.__setattr__(model, "_owner", weakref.ref(self))

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        m, old = self.model, self._engine
        eng = grow_engine(self, batch, lambda rows: AaeEngine(m.image_size, m.hidden_dim, m.z_dim, max_batch=rows))
        if old is not None:                    # optimizer_D's and optimizer_G's state carries over as optimizer_R's does
            for name in ("d_exp_avg", "d_exp_avg_sq", "enc_g_exp_avg", "enc_g_exp_avg_sq"):
                getattr(eng, name).copy_(getattr(old, name))
            eng.d_steps, eng.g_steps = old.d_steps, old.g_steps
        return eng

    def train(self, num_epochs, lr=1e-3, D_lr=2e-4, G_lr=2e-4, weight_decay=1e-5):
        """ Train an AAE: per batch the reconstruction, discriminator and regularisation phases, each followed by its
        optimizer; a true epoch over train_iter, losses read back once per epoch, validation with the forward-only
        kernels, best model kept.  A subclass's own compute_batch, train_D or train_G is trained by the plain loop over
        the differentiable nodes instead.  One process only. """
        from gm_b200 import parallel as par
        if par.world_size() > 1:
            raise GmError("the AAE trains on one process: there is no data-parallel AAE")
        if has_custom_step(self):
            return reference_loop(self, num_epochs, lr, D_lr, G_lr, weight_decay)
        hpR, hpD, hpG = AdamHP.make(lr, weight_decay=weight_decay), AdamHP.make(D_lr), AdamHP.make(G_lr)
        if self._engine is not None:
            self._engine.reset_optimizer()
            self._engine.sync_all()
        from gm_b200.gan_api import DeviceDataset
        resident = DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None)) if self.device_noise else None
        self._resident = resident
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            if resident is not None:
                bs = min(resident.batch_size, resident.n)
                nb = len(resident)
                eng = self._ensure_engine(bs)
                eng.set_lazy_grads(True)
                eng.set_sampler(resident.n, nb, self._seed + 7919 * epoch, batch_size=bs)
                ring = torch.zeros(nb, 3, device="cuda")
                try:
                    for k in range(nb):
                        rows = min(bs, resident.n - k * bs)                        # the last batch of an epoch may be short
                        ring[k, 0:1].copy_(eng.recon_grad(resident.bits, fmt="bits", batch=rows, step=k))
                        eng.apply(hpR)
                        ring[k, 1:2].copy_(eng.d_grad(rows, seed=self._seed, step=self._step))
                        eng.apply_d(hpD)
                        ring[k, 2:3].copy_(eng.g_grad(rows))
                        eng.apply_g(hpG)
                        self._step += 1
                finally:
                    eng.set_lazy_grads(False)
                    eng.set_sampler(0, 0, 0)
                vals = ring.t().tolist()
            else:
                per_step = []
                for batch in self.train_iter:
                    images = self._images(batch)
                    n = images.shape[0]
                    eng = self._ensure_engine(n)
                    r = eng.recon_grad(images).clone()
                    eng.apply(hpR)
                    d = eng.d_grad(n, prior=to_cuda(torch.randn(n, self.model.z_dim))).clone()
                    eng.apply_d(hpD)
                    g = eng.g_grad(n).clone()
                    eng.apply_g(hpG)
                    per_step.append(torch.cat([r, d, g]))
                    self._step += 1
                vals = torch.stack(per_step).t().tolist()
            self._end_epoch(epoch, num_epochs, vals)

    def _end_epoch(self, epoch, num_epochs, vals):
        """the three loss lists, validation, best model and the epoch line"""
        epoch_recon, epoch_D, epoch_G = vals
        self.recon_loss.extend(epoch_recon)
        self.Dlosses.extend(epoch_D)
        self.Glosses.extend(epoch_G)
        self.model.eval()
        val_loss = self.evaluate(self.val_iter)
        if val_loss < self.best_val_loss:
            self.best_model = deepcopy(self.model)                  # a detached module copy
            self.best_val_loss = val_loss
        print(EPOCH_LINE % (epoch, num_epochs, np.mean(epoch_recon), np.mean(epoch_D), np.mean(epoch_G), val_loss))
        self.num_epochs += 1
        if self.viz:
            self.sample_images(epoch)

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

    def reconstruct_images(self, images, epoch, save=True):
        """ the reconstructions of images, shaped like images (no plotting) """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images, _ = self.model(batch)
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True):
        """ z ~ p(z), x = D(z): the decoded prior samples [num_images, side, side] """
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
        for vals, color in ((self.recon_loss, "r"), (self.Dlosses, "g"), (self.Glosses, "b")):
            plt.plot(np.linspace(1, self.num_epochs, len(vals)), vals, color)
        plt.legend(["Reconstruction", "Discriminator", "Generator"])
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
    model = AAE(image_size=784, hidden_dim=400, z_dim=20)
    trainer = AAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=10, lr=1e-3, D_lr=2e-4, G_lr=2e-4, weight_decay=1e-5)
