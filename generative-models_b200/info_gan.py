""" (InfoGAN) Information-maximising GAN — drop-in for the reference's src/info_gan.py.

G's input is noise z plus a one-hot categorical code and a Gaussian continuous code
(src/info_gan.py:306-325); D is the NS discriminator (src/info_gan.py:223-267); the
auxiliary network Q (src/info_gan.py:78-94) recovers the codes from G's output and the
mutual-information step trains G and Q with a third Adam (src/info_gan.py:146-148,196-205).
"""
import weakref

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import parallel as par
from gm_b200 import AdamHP, GmError, InfoGanEngine
from gm_b200.gan_api import (builtin_step, Generator as _Generator, Discriminator as _Discriminator, GANTrainerBase, GradHandoff,
                             EngineCall, _EngineBacked, info_reference_loop, refuse_multi_rank, slot_ring, _split_like, flat_pairs,
                             to_cuda, G_NET, D_NET)


class Generator(_Generator):
    """ Generator. Input is noise and latent variables, output is a generated image (src/info_gan.py:45-57) """

    def __init__(self, image_size, hidden_dim, z_dim, disc_dim, cont_dim):
        super().__init__(image_size, hidden_dim, z_dim + disc_dim + cont_dim)


class Discriminator(_Discriminator):
    """ Discriminator (src/info_gan.py:60-75); note the second layer is named `discriminator` """

    def __init__(self, image_size, hidden_dim, output_dim):
        nn.Module.__init__(self)
        if output_dim != 1:
            raise GmError("only output_dim=1 discriminators are built")
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, output_dim=output_dim))
        self.linear = nn.Linear(image_size, hidden_dim)
        self.discriminator = nn.Linear(hidden_dim, output_dim)


class Q(_EngineBacked):
    """ Auxiliary network Q(c|x) (src/info_gan.py:78-94); parameters live in the engine """

    def __init__(self, image_size, hidden_dim, disc_dim, cont_dim):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, disc_dim=disc_dim, cont_dim=cont_dim))
        self.linear = nn.Linear(image_size, hidden_dim)
        self.inference = nn.Linear(hidden_dim, disc_dim + cont_dim)

    def forward(self, x):
        if not torch.is_grad_enabled():
            # inference: plain torch on the engine's master weights
            inferred = self.inference(torch.relu(self.linear(to_cuda(x))))
            return inferred[:, :self.disc_dim], inferred[:, self.disc_dim:]
        # a user-written train_Q (README.md:31): one autograd node over gm_gan_q_forward / _backward with buffers of its
        # own per live call, so Q(G(z)) can await its backward while G's does
        x = to_cuda(x).float().contiguous()
        eng = self._engine_for(x.shape[0], "Q")
        ring = slot_ring(eng, "Q", eng.num_q_slots())
        params = tuple(self.parameters())

        def fwd(x):
            slot, gen = ring.take()
            return eng.q_forward(slot, x), (slot, gen)

        def bwd(handle, grads, need_dx):
            ring.check(*handle)
            flat, dx = eng.q_backward(handle[0], grads[0].float().contiguous(), need_dx)
            return dx, _split_like(flat, params)
        inferred = EngineCall.apply(x, fwd, bwd, *params)
        return inferred[:, :self.disc_dim], inferred[:, self.disc_dim:]


class InfoGAN(nn.Module):
    """ Super class to contain D, G and Q (src/info_gan.py:97-109) """

    def __init__(self, image_size, hidden_dim, z_dim, disc_dim, cont_dim, output_dim=1):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, disc_dim=disc_dim,
                                  cont_dim=cont_dim, output_dim=output_dim))
        self.G = Generator(image_size, hidden_dim, z_dim, disc_dim, cont_dim)
        self.D = Discriminator(image_size, hidden_dim, output_dim)
        self.Q = Q(image_size, hidden_dim, disc_dim, cont_dim)
        self.shape = int(image_size ** 0.5)


class InfoGANTrainer(GANTrainerBase):
    """ Object to hold data iterators, train an InfoGAN (src/info_gan.py:112-390) """
    variant = "info"

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        super().__init__(model, train_iter, val_iter, test_iter, viz)
        self.MIlosses = []
        if isinstance(getattr(model, "Q", None), _EngineBacked):
            object.__setattr__(model.Q, "_owner", weakref.ref(self))

    def _has_custom_step(self):
        return super()._has_custom_step() or not getattr(type(self).train_Q, "_gm_builtin", False)

    def _ensure_engine(self, batch):
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        m, old = self.model, self._engine
        batch = max(batch, self._max_batch or 0, 64)
        eng = InfoGanEngine(m.image_size, m.hidden_dim, m.z_dim, m.disc_dim, m.cont_dim, max_batch=batch)
        for net, mod in ((G_NET, m.G), (D_NET, m.D)):
            params = list(mod.parameters())
            eng.load(net, [p.data for p in params])
            for p, v in zip(params, eng.views(net)):
                p.data = v
            mod._attach(eng, net)
        qp = list(m.Q.parameters())
        eng.load_q([p.data for p in qp])
        for p, v in zip(qp, eng.q_views()):
            p.data = v
        m.Q._attach(eng, None)
        if old is not None:
            for a, b in ((eng.exp_avg, old.exp_avg), (eng.exp_avg_sq, old.exp_avg_sq)):
                for net in (G_NET, D_NET):
                    a[net].copy_(b[net])
            for name in ("q_exp_avg", "q_exp_avg_sq", "g_mi_exp_avg", "g_mi_exp_avg_sq"):
                getattr(eng, name).copy_(getattr(old, name))
            eng.steps, eng.mi_steps = list(old.steps), old.mi_steps
        self._engine, self._max_batch = eng, batch
        self._needs_sync = False
        return eng

    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1):
        """ src/info_gan.py:130-221: per outer step D update(s), G update, then the Q / MI update """
        if self._has_custom_step():
            # an overridden train_D / train_G / train_Q: the reference's loop verbatim over the autograd nodes of model.G /
            # model.D / model.Q
            refuse_multi_rank("train_D / train_G / train_Q")
            self._ensure_engine(getattr(self.train_iter, "batch_size", None) or next(iter(self.train_iter))[0].shape[0])
            return info_reference_loop(self, num_epochs, G_lr, D_lr, D_steps)
        par.require_single_process(self.name + "Trainer")
        hpG, hpD = AdamHP.make(G_lr), AdamHP.make(D_lr)
        epoch_steps = int(np.ceil(len(self.train_iter) / D_steps))
        self._pre_train(num_epochs, hpG, hpD, D_steps, {})
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            dl, gl, ml = [], [], []
            for _ in range(epoch_steps):
                dstep = []
                for _ in range(D_steps):
                    images = self.process_batch(self.train_iter)
                    dstep.append(self._fused_D(images, hpD))
                dl.append(torch.stack(dstep).mean())
                gl.append(self._fused_G(images.shape[0], hpG))
                eng = self._engine
                noise = self.compute_noise(images.shape[0], self.model.z_dim, self.model.disc_dim, self.model.cont_dim)
                ml.append(eng.q_grad(images.shape[0], noise.float().contiguous()).clone())
                eng.apply_mi(hpG)
            G_losses, D_losses, MI_losses = torch.stack(gl).tolist(), torch.stack(dl).tolist(), torch.stack(ml).tolist()
            self.Glosses.extend(G_losses)
            self.Dlosses.extend(D_losses)
            self.MIlosses.extend(MI_losses)
            print("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f, MI Loss: %.4f"
                  % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses), np.mean(MI_losses)))
            self.num_epochs += 1

    def _fused_D(self, images, hp):
        eng = self._ensure_engine(images.shape[0])
        self._sync_once(eng)
        m = self.model
        noise = self.compute_noise(images.shape[0], m.z_dim, m.disc_dim, m.cont_dim)
        loss = eng.d_grad(images, noise=noise.float().contiguous()).clone()
        eng.apply(D_NET, hp)
        return loss

    def _fused_G(self, batch, hp):
        eng = self._ensure_engine(batch)
        self._sync_once(eng)
        m = self.model
        noise = self.compute_noise(batch, m.z_dim, m.disc_dim, m.cont_dim)
        loss = eng.g_grad(batch, noise=noise.float().contiguous()).clone()
        eng.apply(G_NET, hp)
        return loss

    @builtin_step
    def train_D(self, images):
        images = to_cuda(images)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        m = self.model
        noise = self.compute_noise(images.shape[0], m.z_dim, m.disc_dim, m.cont_dim)
        loss = eng.d_grad(images.float().contiguous(), noise=noise.float().contiguous())
        return self._loss_tensor(D_NET, loss)

    @builtin_step
    def train_G(self, images):
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        m = self.model
        noise = self.compute_noise(images.shape[0], m.z_dim, m.disc_dim, m.cont_dim)
        loss = eng.g_grad(images.shape[0], noise=noise.float().contiguous())
        return self._loss_tensor(G_NET, loss)

    @builtin_step
    def train_Q(self, images, LAMBDA=1):
        """ src/info_gan.py:269-304: returns MI_loss; .backward() delivers the G and Q gradients """
        if LAMBDA != 1:
            raise ValueError("the fused MI loss is built for the reference default LAMBDA=1")
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        m = self.model
        noise = self.compute_noise(images.shape[0], m.z_dim, m.disc_dim, m.cont_dim)
        loss = eng.q_grad(images.shape[0], noise.float().contiguous())
        params = list(m.G.parameters()) + list(m.Q.parameters())
        flat = torch.cat([eng.grads[G_NET], eng.q_grads])
        return GradHandoff.apply(flat.detach().requires_grad_(True), loss, flat_pairs(params, flat))

    def compute_noise(self, batch_size, z_dim, disc_dim=None, cont_dim=None, c=None):
        """ src/info_gan.py:306-325: z, a uniformly drawn one-hot code, a Gaussian code """
        disc_dim = self.model.disc_dim if disc_dim is None else disc_dim
        cont_dim = self.model.cont_dim if cont_dim is None else cont_dim
        z = torch.randn(batch_size, z_dim)
        disc_c = torch.zeros((batch_size, disc_dim))
        if c is not None:
            categorical = int(c) * torch.ones((batch_size,), dtype=torch.long)
        else:
            categorical = torch.randint(0, disc_dim, (batch_size,), dtype=torch.long)
        disc_c[range(batch_size), categorical] = 1
        cont_c = torch.randn(batch_size, cont_dim)
        return to_cuda(torch.cat((z, disc_c, cont_c), dim=1))

    def generate_images(self, epoch, num_outputs=36, save=True):
        self.model.eval()
        m = self.model
        noise = self.compute_noise(num_outputs, m.z_dim, m.disc_dim, m.cont_dim)
        images = m.G(noise)
        return images.view(images.shape[0], m.shape, m.shape, -1).squeeze()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()
    model = InfoGAN(image_size=784, hidden_dim=400, z_dim=20, disc_dim=10, cont_dim=10)
    trainer = InfoGANTrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1)
