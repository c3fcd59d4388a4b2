""" (DCDRAGAN) DRAGAN with the DCGAN convolutional generator and a batch-norm-free convolutional discriminator, on 64x64
images.

The class surface is src/dra_gan.py's, so its driver code runs on the conv model:

    model = DCDRAGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCDRAGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1)

L(D) = -mean(log(D(x) + 1e-8) + log(1 - D(G(z)) + 1e-8)) + LAMBDA mean((||grad D(x_hat)||_2 - K)^2) with
x_hat = delta x + (1 - delta)(x + C std(x) u), one delta per image and u per element, std over the whole real batch
(src/dra_gan.py:174-225); L(G) = -mean(log(D(G(z)) + 1e-8)).  D keeps its sigmoid (src/dra_gan.py:59) and has no BatchNorm,
so one image's gradient does not depend on the batch.  The penalty's double backward runs in closed form in the sm_90a
kernels behind gm_b200.DcganEngine(variant="dra") (DESIGN.md §6b).  Under torchrun the trainer is data-parallel like
DCGANTrainer, with std(x) taken over the global batch.
"""
import torch
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import to_cuda, builtin_step
from dc_gan import Generator, DCGAN, DCGANTrainer  # noqa: F401
from dc_w_gp_gan import Discriminator as _Critic


class Discriminator(_Critic):
    """ 64x64 -> 32x32 -> 16x16 -> 8x8 -> 4x4 -> 1 (convolutions + LeakyReLU(0.2), no BatchNorm, sigmoid output): the
    WGAN-GP critic's layers with src/dra_gan.py:59's sigmoid """
    out_acts = ("sigmoid",)

    def __init__(self, image_size, hidden_dim, output_dim=1, channels=3):
        super().__init__(image_size, hidden_dim, output_dim, channels, out_act="sigmoid")


class DCDRAGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/dra_gan.py:63-74) """
    _D = Discriminator


class DCDRAGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv DRAGAN (surface of src/dra_gan.py:77-300) """
    variant = "dra"

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=5):
        """ Trainer.train (src/dra_gan.py:94-172) with LAMBDA = 10, K = 1, C = 1 and delta, u drawn on the device per rank """
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    @builtin_step
    def train_D(self, images, LAMBDA=10, K=1, C=1):
        """ Run 1 step of training for D (src/dra_gan.py:174-225): returns D_loss; .backward() delivers the gradients """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        flat = images.reshape(n, -1).float()
        noise = self.compute_noise(n, self.model.z_dim)
        delta = torch.rand(n, 1)                                    # src/dra_gan.py:200
        u = torch.rand(flat.shape)                                  # src/dra_gan.py:205, NCHW-flattened like the images
        loss = eng.d_grad(eng.stage_images(flat), n, noise=noise.float().contiguous(), gp_lambda=float(LAMBDA), gp_k=float(K),
                          dra_c=float(C), delta=to_cuda(delta), u=to_cuda(u))
        return self._loss(1, loss.clone())


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCDRAGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCDRAGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1)
