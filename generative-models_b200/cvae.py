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

from gm_b200 import GmError, CvaeEngine
from gm_b200 import parallel as par
from gm_b200.engine import class_ids
from gm_b200.gan_api import to_cuda, engine_call, VAE_EPOCH_LINE  # noqa: F401
from gm_b200.vae_api import engine_of, encoder_call, VaeFamilyModel, VaeFamilyTrainer

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
        eng = engine_of(self, "Encoder", x.shape[0])
        y = eng.class_ids(_labels(y, x.shape[0]), x.shape[0])
        if torch.is_grad_enabled():                # (mu, log_var) and their backward: gm_cvae_encoder_forward / gm_vae_encoder_backward
            return encoder_call(self, eng, x, lambda slot, x: eng.encoder_forward(slot, x, y))
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
        eng = engine_of(self, "Decoder", z.shape[0])
        y = eng.class_ids(_labels(y, z.shape[0]), z.shape[0])
        if torch.is_grad_enabled():                # the images and their backward, with dL/dz when z requires grad
            n = z.shape[0]

            def forward(slot, z):
                return eng.decoder_forward(slot, z, y)

            def backward(slot, grads, need_dz):
                return eng.decoder_backward(slot, n, grads[0], need_dz)
            return engine_call(eng, "Decoder", eng.num_slots(), z.float(), self.named_parameters("decoder"), forward,
                               backward)
        return eng.decode(z, y)


class CVAE(VaeFamilyModel):
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
        self._link()

    def _args(self):
        return self.image_size, self.hidden_dim, self.z_dim, self.num_classes

    def _make_engine(self, max_batch):
        return CvaeEngine(self.image_size, self.hidden_dim, self.z_dim, self.num_classes, max_batch=max_batch)

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


class CVAETrainer(VaeFamilyTrainer):
    def _keep_debugging_batch(self, batch):
        self.debugging_image, self.debugging_labels = batch

    def _one_process(self):
        if par.world_size() > 1:
            raise GmError("the CVAE trains on one process: there is no data-parallel CVAE")

    def _device_dataset(self):
        """the train split packed to 1 bit/pixel in HBM once, with its labels checked on the host and uploaded once as
        int32 beside it (self._resident_y); None when the loader's dataset holds no label tensor: the host path runs"""
        resident = super()._device_dataset()
        tensors = getattr(getattr(self.train_iter, "dataset", None), "tensors", None)
        if resident is None or tensors is None or len(tensors) < 2:
            return None
        cached = getattr(self, "_resident_y", None)
        if cached is None or cached[0] is not tensors[1]:
            y = class_ids(tensors[1], self.model.num_classes, torch.device("cuda", torch.cuda.current_device()), resident.n)
            self._resident_y = (tensors[1], y)
        return resident

    def _resident_step(self, eng, hp, row, rows, epoch, k):
        row.copy_(eng.grad(self._resident.bits, self._resident_y[1], fmt="bits", batch=rows, seed=self._seed, step=k))
        eng.apply(hp)

    def _inputs(self, batch):
        """(images [n, image_size] fp32 on the GPU, labels checked for the model's classes) of one loader batch"""
        images, labels = batch
        y = class_ids(labels, self.model.num_classes, torch.device("cuda", torch.cuda.current_device()), images.shape[0])
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous(), y

    def kl_divergence(self, mu, log_var):
        """ torch, for direct use """
        return torch.sum(0.5 * (mu ** 2 + torch.exp(log_var) - log_var - 1))

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


if __name__ == "__main__":
    train_iter, val_iter, test_iter = get_data()                                       # noqa: F405
    model = CVAE(image_size=784, hidden_dim=400, z_dim=20, num_classes=10)
    trainer = CVAETrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
