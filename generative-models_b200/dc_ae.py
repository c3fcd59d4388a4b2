""" (DCAutoencoder) Autoencoder with a deep-convolutional encoder and decoder, on 64x64 images - the conv model the
reference's README recommends for more complex datasets (README.md:68), with src/ae.py's class surface, so its driver
code runs on the conv model:

    model = DCAutoencoder(image_size=64 * 64 * 3, hidden_dim=64, z_dim=32)
    trainer = DCAutoencoderTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)

  Encoder: the DCGAN discriminator trunk, Conv(ch, h, 4, 2, 1) LReLU(0.2) -> Conv(h, 2h) BN LReLU -> Conv(2h, 4h) BN LReLU
           -> Conv(4h, 8h) BN LReLU, then the code relu(Conv2d(8h, z, 4, 1, 0)) (src/ae.py:38-39's relu(linear(x))).
  Decoder: the DCGAN generator, ConvT(z, 8h, 4, 1, 0) BN ReLU -> ... -> ConvT(h, ch, 4, 2, 1) -> sigmoid (src/ae.py:51-52).

z_dim is the code width, src/ae.py's hidden_dim (32 by default, src/ae.py:58); hidden_dim is the conv trunk's base channel
width.  The loss is the reference's sum (x - out)^2 (src/ae.py:158) and one Adam with coupled weight decay runs over all
parameters (src/ae.py:98-101).  BatchNorm follows model.training, as in dc_vae.  All arithmetic runs in the sm_90a kernels
behind gm_b200.DcganEngine(variant="ae"); the modules only hold the parameters, so state_dict() has encoder.* / decoder.*
keys in torch's layouts.  Training, batching (host loader or device_dataset) and data parallelism are DCVAETrainer's.
"""
import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200.gan_api import to_cuda, builtin_step, has_custom_compute_batch, compute_batch_evaluate
from dc_gan import pull_running_stats
from dc_vae import DCVAE, DCVAETrainer, Decoder, _encoder_forward  # noqa: F401  (Decoder: src/ae.py's surface)


class Encoder(nn.Module):
    """ Conv encoder of the autoencoder: 64x64 image -> the code relu(l5(trunk(x))) [n, z_dim] """

    def __init__(self, image_size, hidden_dim, z_dim, channels=3):
        super().__init__()
        c = [hidden_dim, 2 * hidden_dim, 4 * hidden_dim, 8 * hidden_dim]
        self.l1 = nn.Conv2d(channels, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], z_dim, 4, 1, 0, bias=False)
        self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])

    def forward(self, x):
        return _encoder_forward(self, x)


class DCAutoencoder(DCVAE):
    """ Autoencoder super class to encode then decode an image (as src/ae.py:55-67), with conv encoder and decoder """
    variant = "ae"
    _Encoder = Encoder

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=32, channels=3):
        super().__init__(image_size, hidden_dim, z_dim, channels)

    def _engine_names(self, named):
        return dict(named)                     # encoder.l5 is the engine's D.l5: the names agree

    def _module_names(self, tensors):
        return dict(tensors)

    def forward(self, x):
        x = to_cuda(x).float()
        n = x.shape[0]
        if torch.is_grad_enabled() and self.training:               # src/ae.py:63-64 on the differentiable encoder / decoder
            return self.decoder(self.encoder(x))
        eng = self._engine()
        out, _, _ = eng.ae_forward(eng.stage_images(x.reshape(n, -1)), n, train=self.training)
        self._after_forward(eng, self.training)
        return out


class DCAutoencoderTrainer(DCVAETrainer):
    """ Object to hold data iterators, train the conv autoencoder (surface of src/ae.py:70-218) """
    _two_losses = False                 # compute_batch returns one loss

    def _grad_step(self, eng, rows, n, seed):
        return eng.ae_grad(rows, n)

    def _log_epoch(self, epoch, num_epochs, vals, val_loss):
        epoch_loss = [v[0] for v in vals]
        self.recon_loss.extend(epoch_loss)
        return "Epoch[%d/%d], Train Loss: %.4f, Val Loss: %.4f" % (epoch, num_epochs, np.mean(epoch_loss), val_loss)

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of examples (src/ae.py:147-160): returns recon = sum (x - out)^2; .backward() delivers
        the engine's gradient to the module parameters """
        images = self._images(batch)
        eng = self._engine_synced()
        loss = eng.ae_grad(eng.stage_images(images), images.shape[0]).clone()
        pull_running_stats(eng, self._nets())                     # the training-mode forward's update, as torch makes it
        return self._fused_loss(self._nets(), loss[0])

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/ae.py:162-164): the mean per-batch loss of the forward-only kernels, BatchNorm
        in the model's mode; with an overriding compute_batch, its loss as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, self._two_losses)
        eng = self._engine_synced()
        loss = []
        for batch in iterator:
            images = self._images(batch)
            n = images.shape[0]
            _, _, ls = eng.ae_forward(eng.stage_images(images), n, train=self.model.training)
            loss.append(ls[0])
        self.model._after_forward(eng, self.model.training)
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ src/ae.py:166-193 without the plotting: the reconstructions in the images' shape """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            return self.model(batch).view(images.shape).squeeze()

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.recon_loss)), self.recon_loss, "r")
        plt.legend(["Reconstruction loss"])
        plt.title(self.name)
        plt.show()


if __name__ == "__main__":
    imgs = (torch.rand(8192, 3, 64, 64) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCAutoencoder(image_size=64 * 64 * 3, hidden_dim=64, z_dim=32)
    trainer = DCAutoencoderTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
