""" (DCWGPGAN) WGAN-GP with the DCGAN convolutional generator and a batch-norm-free convolutional critic — how the
WGAN-GP paper trains (Gulrajani et al. 2017, https://arxiv.org/abs/1704.00028), on 64x64 images.

The class surface is src/w_gp_gan.py's, so its driver code runs on the conv model:

    model = DCWGPGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCWGPGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1)

L(D) = mean(D(G(z))) - mean(D(x)) + LAMBDA mean((||grad D(x_hat)||_2 - 1)^2), x_hat = eps x + (1 - eps) G(z) with one eps
per image (src/w_gp_gan.py:186-218); L(G) = -mean(D(G(z))).  The critic has no BatchNorm (with it one image's input
gradient would depend on the whole batch, WGAN-GP paper §4) and ends in ReLU like src/w_gp_gan.py:61, or with
out_act="none" in the identity.  Its gradient penalty runs as a closed-form double backward in the sm_90a kernels behind
gm_b200.DcganEngine(variant="wgp") (DESIGN.md §6b).  Under torchrun the trainer is data-parallel like DCGANTrainer.
"""
import torch

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import to_cuda, builtin_step
import dc_gan
from dc_gan import Generator, DCGAN, DCGANTrainer  # noqa: F401


class Discriminator(dc_gan.Discriminator):
    """ Critic: 64x64 -> 32x32 -> 16x16 -> 8x8 -> 4x4 -> 1 (convolutions + LeakyReLU(0.2), no BatchNorm, relu / linear output) """
    out_acts = ("relu", "none")

    def __init__(self, image_size, hidden_dim, output_dim=1, channels=3, out_act="relu"):
        super().__init__(image_size, hidden_dim, output_dim, channels, batch_norm=False, out_act=out_act)


class DCWGPGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/w_gp_gan.py:65-76) """
    _D = Discriminator

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, output_dim=1, channels=3, out_act="relu"):
        super().__init__(image_size, hidden_dim, z_dim, output_dim, channels, out_act=out_act)


class DCWGPGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv WGAN-GP (surface of src/w_gp_gan.py:79-315) """
    variant = "wgp"

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=5):
        """ Trainer.train (src/w_gp_gan.py:96-175) with LAMBDA = 10 and eps drawn on the device per rank """
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    @builtin_step
    def train_D(self, images, LAMBDA=10):
        """ Run 1 step of training for the critic (src/w_gp_gan.py:177-220): returns D_loss; .backward() delivers the gradients """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        noise = self.compute_noise(n, self.model.z_dim)
        eps = to_cuda(torch.rand(n, 1)).reshape(-1)                   # one eps per image (src/w_gp_gan.py:197)
        loss = eng.d_grad(eng.stage_images(images.reshape(n, -1).float()), n, noise=noise.float().contiguous(),
                          gp_lambda=float(LAMBDA), eps=eps.float())
        return self._loss(1, loss.clone())


# the name src/w_gp_gan.py's notebook uses, on the conv model
DCWGANGP, DCWGANGPTrainer = DCWGPGAN, DCWGPGANTrainer

if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCWGPGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCWGPGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1)
