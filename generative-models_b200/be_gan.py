""" (BEGAN) Boundary equilibrium GAN — drop-in for the reference's src/be_gan.py.

The discriminator is an autoencoder x -> hidden -> x (src/be_gan.py:63-76); losses are L1
reconstruction errors, D_loss = DX - K*DG, G_loss = DG (src/be_gan.py:225-256); K follows
the proportional control K <- clip(K + LAMBDA (GAMMA DX - DG), 0, 1) and two
ReduceLROnPlateau schedulers halve the learning rates on a plateau of the convergence
measure (src/be_gan.py:133-136,186-195).  K, the convergence measure and the schedulers
live on the device, so the fused train() never synchronises inside an epoch.
"""
import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import parallel as par
from gm_b200 import AdamHP, GmError
from gm_b200.gan_api import (builtin_step, Generator, GANTrainerBase, _EngineBacked, EngineCall, began_reference_loop,
                             refuse_multi_rank, slot_ring, _split_like, to_cuda, G_NET, D_NET)


class Discriminator(_EngineBacked):
    """ Autoencoder. Input is an image (real, generated), output is the reconstructed image (src/be_gan.py:63-76) """

    def __init__(self, image_size, hidden_dim):
        super().__init__()
        self.encoder = nn.Linear(image_size, hidden_dim)
        self.decoder = nn.Linear(hidden_dim, image_size)

    def forward(self, x):
        if not torch.is_grad_enabled():
            # inference: plain torch on the engine's fp32 master weights
            return self.decoder(torch.relu(self.encoder(to_cuda(x))))
        # a user-written train_D / train_G (README.md:31): one autograd node over gm_gan_ae_forward / _backward, whose
        # call keeps its activations in one of the engine's D row regions until its backward ran
        x = to_cuda(x).float().contiguous()
        eng = self._engine_for(x.shape[0], "Discriminator")
        ring = slot_ring(eng, "Discriminator", eng.num_slots())
        params = tuple(self.parameters())

        def fwd(x):
            slot, gen = ring.take()
            return eng.ae_forward(slot, x), (slot, gen)

        def bwd(handle, grads, need_dx):
            ring.check(*handle)
            flat, dx = eng.ae_backward(handle[0], grads[0].float().contiguous(), need_dx)
            return dx, _split_like(flat, params)
        return EngineCall.apply(x, fwd, bwd, *params)


class BEGAN(nn.Module):
    """ Super class to contain both Discriminator (D) and Generator (G) (src/be_gan.py:79-90) """

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim))
        self.G = Generator(image_size, hidden_dim, z_dim)
        self.D = Discriminator(image_size, hidden_dim)
        self.shape = int(image_size ** 0.5)


class BEGANTrainer(GANTrainerBase):
    variant = "began"

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00):
        if self._has_custom_step():
            # an overridden train_D / train_G: the reference's loop verbatim over the autograd nodes of model.G / model.D
            refuse_multi_rank("train_D / train_G")
            self._ensure_engine(getattr(self.train_iter, "batch_size", None) or next(iter(self.train_iter))[0].shape[0])
            return began_reference_loop(self, num_epochs, G_lr, D_lr, D_steps, GAMMA, LAMBDA, K)
        par.require_single_process(self.name + "Trainer")
        hpG, hpD = AdamHP.make(G_lr), AdamHP.make(D_lr)
        epoch_steps = int(np.ceil(len(self.train_iter) / D_steps))
        patience = 5 * len(self.train_iter)                      # src/be_gan.py:133-136
        self._pre_train(num_epochs, hpG, hpD, D_steps, {})
        self._began_pending = K
        if self._engine is not None:
            self._engine.began_init(K, self._last_batch)
            self._began_pending = None
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            dl, gl = [], []
            for _ in range(epoch_steps):
                dstep = []
                for _ in range(D_steps):
                    images = self.process_batch(self.train_iter)
                    dstep.append(self._fused_D(images, hpD))
                dl.append(torch.stack(dstep).mean())
                gl.append(self._fused_G(images.shape[0], hpG))
                self._engine.began_control(GAMMA, LAMBDA, patience)     # src/be_gan.py:186-195
            G_losses, D_losses = torch.stack(gl).tolist(), torch.stack(dl).tolist()
            self.Glosses.extend(G_losses)
            self.Dlosses.extend(D_losses)
            st = self._engine.began_state()
            print("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f, K: %.4f, Convergence Measure: %.4f"
                  % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses), st[0], st[10]))
            self.num_epochs += 1

    def _ensure_engine(self, batch):
        fresh = self._engine is None or batch > (self._max_batch or 0)
        eng = super()._ensure_engine(batch)
        self._last_batch = batch
        if fresh:
            K = getattr(self, "_began_pending", None)
            eng.began_init(0.0 if K is None else K, batch)
            self._began_pending = None
        return eng

    @builtin_step
    def train_D(self, images, K):
        """ returns (D_loss, DX_loss, DG_loss) like src/be_gan.py:212-238 """
        images = to_cuda(images)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_all()
        eng.began_init(float(K), images.shape[0])
        noise = self.compute_noise(images.shape[0], self.model.z_dim)
        loss = eng.d_grad(images.float().contiguous(), noise=noise.float().contiguous())
        st = eng.began_state()
        return self._loss_tensor(D_NET, loss), torch.tensor(st[3]), torch.tensor(st[4])

    def generate_images(self, epoch, num_outputs=36, save=True):
        self.model.eval()
        noise = self.compute_noise(num_outputs, self.model.z_dim)
        images = self.model.G(noise)
        return images.view(images.shape[0], self.model.shape, self.model.shape, -1).squeeze()


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()
    model = BEGAN(image_size=784, hidden_dim=400, z_dim=20)
    trainer = BEGANTrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)
