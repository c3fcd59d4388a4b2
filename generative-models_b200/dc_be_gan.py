""" (DCBEGAN) Boundary equilibrium GAN with the DCGAN convolutional G and a convolutional autoencoder D, on 64x64 images.

The class surface is src/be_gan.py's, so its driver code runs on the conv model:

    model = DCBEGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCBEGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)

D is an autoencoder (src/be_gan.py:63-76) built from the two DCGAN stacks: the encoder is the DCGAN D trunk (BatchNorm on
conv 2-4) ending in a linear Conv2d(8h, embed_dim, 4, 1, 0); the decoder is the DCGAN generator stack with embed_dim in
place of z and a linear output, as the reference's decoder has no activation.  embed_dim defaults to z_dim (the BEGAN
paper's N_h = N_z).  The BatchNorm layers follow the DCGAN paper the conv path is built on; the BEGAN paper's own
autoencoder has none.  L(v) = sum |D(v) - v| per image; D_loss = mean L(x) - K mean L(G(z)), G_loss = mean L(G(z)) with the
gradient reaching G(z) through D and through the target (src/be_gan.py:225-256).  K's proportional control, the convergence
measure and the two ReduceLROnPlateau schedulers (src/be_gan.py:133-136,186-195) run on the device
(gm_b200.DcganEngine(variant="be")), so train() does not synchronise inside an epoch.  Under torchrun DX and DG are sums
over the ranks (NCCL), so K and the learning-rate scale stay identical on every rank.
"""
import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import to_cuda, builtin_step
from dc_gan import Generator, DCGAN, DCGANTrainer


class Encoder(nn.Module):
    """ 64x64 -> 32x32 -> 16x16 -> 8x8 -> 4x4 (convolutions + LeakyReLU(0.2), BatchNorm on layers 2-4) -> embedding [n, embed_dim]
    (linear conv 5) """

    def __init__(self, hidden_dim, embed_dim, channels=3):
        super().__init__()
        c = [hidden_dim, 2 * hidden_dim, 4 * hidden_dim, 8 * hidden_dim]
        self.l1 = nn.Conv2d(channels, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], embed_dim, 4, 1, 0, bias=False)
        self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])


class Decoder(Generator):
    """ The generator stack on the embedding (embed_dim in place of z) with a linear output (src/be_gan.py:73-76); it runs
    inside D(x) """

    def forward(self, x):
        raise GmError("the decoder runs inside D(x) (model.D), which returns the reconstruction")


class Discriminator(nn.Module):
    """ Autoencoder. Input is an image (real, generated), output is the reconstructed image (src/be_gan.py:63-76) """
    out_act = "none"

    def __init__(self, image_size, hidden_dim, output_dim=1, channels=3, embed_dim=100):
        super().__init__()
        self.embed_dim = embed_dim
        self.encoder = Encoder(hidden_dim, embed_dim, channels)
        self.decoder = Decoder(image_size, hidden_dim, embed_dim, channels)
        self._owner = None

    def forward(self, x):
        tr = self._owner
        if tr is None:
            raise GmError("Discriminator is not attached to a CUDA engine yet: construct its trainer first")
        return tr._engine_synced().reconstruct(to_cuda(x).float().reshape(x.shape[0], -1))


class DCBEGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/be_gan.py:79-90) """
    _D = Discriminator

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, channels=3, embed_dim=None):
        super().__init__(image_size, hidden_dim, z_dim, 1, channels, embed_dim=z_dim if embed_dim is None else embed_dim)


class DCBEGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv BEGAN (surface of src/be_gan.py:93-337) """
    variant = "be"
    _custom_step_limit = "BEGAN's discriminator is an autoencoder, and custom losses are built for one score per image"

    def train(self, num_epochs, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00):
        """ Trainer.train (src/be_gan.py:109-205): DCGANTrainer's loop; after each G update K, the convergence measure and
        the plateau schedulers (patience 5 len(train_iter)) move on the device """
        self._control = (float(GAMMA), float(LAMBDA), 5 * len(self.train_iter), float(K))
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _pre_train(self, eng):
        eng.began_init(self._control[3], getattr(self.train_iter, "batch_size", None) or 1)   # fresh schedulers per train()

    def _after_g_step(self, eng, n, inv, seed):
        eng.began_control(*self._control[:3])                                                # src/be_gan.py:186-195

    def _epoch_line(self, eng, epoch, num_epochs, G_losses, D_losses):
        st = eng.began_state()
        return ("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f, K: %.4f, Convergence Measure: %.4f"
                % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses), st[0], st[10]))

    def _pull(self):
        super()._pull()
        if self._engine is None:
            return
        eng = self._engine
        with torch.no_grad():
            for mod, runs, first in ((self.model.D.encoder, eng.run_D, 2), (self.model.D.decoder, eng.run_dec, 1)):
                for i in range(first, 5):
                    bn = getattr(mod, "bn%d" % i)
                    bn.running_mean.copy_(runs[i - 1][0].cpu())
                    bn.running_var.copy_(runs[i - 1][1].cpu())

    @builtin_step
    def train_D(self, images, K):
        """ Run 1 step of training for D (src/be_gan.py:212-238): returns (D_loss, DX_loss, DG_loss); .backward() on D_loss
        delivers the gradients """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        eng.be_state[0] = float(K)
        noise = self.compute_noise(n, self.model.z_dim)
        loss = eng.d_grad(eng.stage_images(images.reshape(n, -1).float()), n, noise=noise.float().contiguous())
        return self._loss(1, loss.clone()), eng.be_state[3].clone(), eng.be_state[4].clone()


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCBEGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCBEGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=1e-4, D_lr=1e-4, D_steps=1, GAMMA=0.50, LAMBDA=1e-3, K=0.00)
