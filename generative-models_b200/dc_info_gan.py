""" (DCInfoGAN) Information GAN with the DCGAN convolutional G / D and a convolutional auxiliary network Q, on 64x64 images.

The class surface is src/info_gan.py's, so its driver code runs on the conv model:

    model = DCInfoGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, disc_dim=10, cont_dim=10)
    trainer = DCInfoGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1)

G's input is [z | one-hot categorical code (disc_dim) | Gaussian continuous code (cont_dim)] (src/info_gan.py:306-325), so
G.l1 is a ConvTranspose2d(z + disc_dim + cont_dim, 8h, 4, 1, 0).  D is the batch-norm DCGAN discriminator with a sigmoid
output; the D and G steps are NSGAN's (src/info_gan.py:223-267).  Q (src/info_gan.py:78-94) is its own network: the DCGAN D
trunk (BatchNorm on conv 2-4) ending in a linear Conv2d(8h, disc_dim + cont_dim, 4, 1, 0), whose first disc_dim outputs are
the categorical logits and the rest the continuous code.  MI_loss = LAMBDA (CE + MSE) on Q(G(noise)) trains Q and G through
MI_optimizer = Adam(G + Q, lr=G_lr), which keeps its own moments for G (src/info_gan.py:142-148,269-304).  In train() the
codes are drawn on the device (gm_b200.DcganEngine(variant="info")) and the MI step follows every G update without
synchronising; under torchrun the G and Q gradients of the MI step are summed (NCCL) before MI_optimizer's step.
"""
import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError
from gm_b200 import parallel as par
from gm_b200.gan_api import to_cuda, builtin_step
from dc_gan import DCGAN, DCGANTrainer, dcgan_init


class Q(nn.Module):
    """ Auxiliary network Q(c|x) that approximates P(c|x), the true posterior (src/info_gan.py:78-94): 64x64 -> 4x4
    (convolutions + LeakyReLU(0.2), BatchNorm on layers 2-4) -> [discrete logits (disc_dim) | continuous (cont_dim)] """

    def __init__(self, image_size, hidden_dim, disc_dim, cont_dim, channels=3):
        super().__init__()
        c = [hidden_dim, 2 * hidden_dim, 4 * hidden_dim, 8 * hidden_dim]
        self.disc_dim, self.cont_dim = disc_dim, cont_dim
        self.l1 = nn.Conv2d(channels, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], disc_dim + cont_dim, 4, 1, 0, bias=False)
        self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])
        self._owner = None

    def forward(self, x):
        tr = self._owner
        if tr is None:
            raise GmError("Q is not attached to a CUDA engine yet: construct the DCInfoGANTrainer first")
        return tr._engine_synced().infer_codes(to_cuda(x).float().reshape(x.shape[0], -1))


class DCInfoGAN(DCGAN):
    """ Super class to contain the Discriminator (D), the Generator (G) and Q (as src/info_gan.py:97-109) """

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, disc_dim=10, cont_dim=10, output_dim=1, channels=3):
        if disc_dim < 1 or cont_dim < 1:
            raise GmError("InfoGAN needs disc_dim >= 1 and cont_dim >= 1")
        super().__init__(image_size, hidden_dim, z_dim + disc_dim + cont_dim, output_dim, channels)   # G reads [z | codes]
        self.__dict__.update(dict(z_dim=z_dim, disc_dim=disc_dim, cont_dim=cont_dim))
        self.Q = Q(image_size, hidden_dim, disc_dim, cont_dim, channels)
        dcgan_init(self.Q)


class DCInfoGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv InfoGAN (surface of src/info_gan.py:112-395) """
    variant = "info"
    _custom_step_limit = "InfoGAN's coded generator input and Q network have no per-call autograd nodes"

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        super().__init__(model, train_iter, val_iter, test_iter, viz)
        self.MIlosses = []
        self._mi_epoch = []
        object.__setattr__(model.Q, "_owner", self)

    def _nets(self):
        return super()._nets() + [("Q", self.model.Q)]

    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1):
        """ Train InfoGAN (src/info_gan.py:130-221): DCGANTrainer's loop; after each G update the MI step and
        MI_optimizer = Adam(G + Q, lr=G_lr) with its own moments """
        self._hp_mi = AdamHP.make(G_lr)
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _pre_train(self, eng):
        import torch.distributed as dist
        for t in (eng.Q.exp_avg, eng.Q.exp_avg_sq, eng.g_mi_avg, eng.g_mi_avg_sq):         # a fresh MI_optimizer per train()
            t.zero_()
        eng.Q.step = 0
        if par.world_size() > 1:                                                            # Q starts from rank 0's weights
            dist.broadcast(eng.Q.params, src=0)
            eng.Q.refresh()
        self._mi_epoch = []

    def _after_g_step(self, eng, n, inv, seed):
        # src/info_gan.py:196-205: fresh codes, MI_loss.backward() into G and Q, MI_optimizer.step()
        self._mi_epoch.append(eng.q_grad(n, inv_global_batch=inv, seed=seed, step=self._step).clone())
        par.sum_gradients(eng.G.grads)
        par.sum_gradients(eng.Q.grads)
        eng.apply_mi(self._hp_mi)

    def _epoch_line(self, eng, epoch, num_epochs, G_losses, D_losses):
        MI_losses = torch.stack(self._mi_epoch).tolist()          # the epoch's one synchronisation, with the G / D losses'
        self._mi_epoch = []
        self.MIlosses.extend(MI_losses)
        return ("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f, MI Loss: %.4f"
                % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses), np.mean(MI_losses)))

    def _noise(self, n):
        m = self.model
        return self.compute_noise(n, m.z_dim, m.disc_dim, m.cont_dim).float().contiguous()

    @builtin_step
    def train_D(self, images):
        """ Run 1 step of training for discriminator (src/info_gan.py:223-246): returns D_loss; .backward() delivers the
        gradients """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        loss = eng.d_grad(eng.stage_images(images.reshape(n, -1).float()), n, noise=self._noise(n))
        return self._loss(1, loss.clone())

    @builtin_step
    def train_G(self, images):
        """ Run 1 step of training for generator (src/info_gan.py:248-267) """
        eng = self._engine_synced()
        n = images.shape[0]
        loss = eng.g_grad(n, noise=self._noise(n))
        return self._loss(0, loss.clone())

    @builtin_step
    def train_Q(self, images, LAMBDA=1):
        """ Run 1 step of training for the auxiliary network (src/info_gan.py:269-304): returns MI_loss; .backward()
        delivers the gradients to G's and Q's parameters """
        eng = self._engine_synced()
        n = images.shape[0]
        loss = eng.q_grad(n, noise=self._noise(n), lam=float(LAMBDA))
        return self._fused_loss([("G", self.model.G), ("Q", self.model.Q)], loss.clone())

    def compute_noise(self, batch_size, z_dim, disc_dim, cont_dim, c=None):
        """ Compute random noise for the generator to learn to make images (src/info_gan.py:306-325)
        OPTIONAL: set c to explore latent dimension space. """
        z = torch.randn(batch_size, z_dim)
        disc_c = torch.zeros((batch_size, disc_dim))
        if c is not None:
            categorical = int(c) * torch.ones((batch_size,), dtype=torch.long)
        else:
            categorical = torch.randint(0, disc_dim, (batch_size,), dtype=torch.long)
        disc_c[range(batch_size), categorical] = 1
        cont_c = torch.randn(batch_size, cont_dim)
        return to_cuda(torch.cat((z, disc_c, cont_c), dim=1))

    def generate_images(self, epoch, num_outputs=36, save=True, c=None):
        """ Sample a grid from G (src/info_gan.py:333-365 without the plotting); c fixes the categorical code """
        self.model.eval()
        m = self.model
        noise = self.compute_noise(num_outputs, m.z_dim, m.disc_dim, m.cont_dim, c=c)
        images = m.G(noise)
        return images.view(num_outputs, m.channels, 64, 64)


if __name__ == "__main__":
    imgs = (torch.rand(8192, 3, 64, 64) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCInfoGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, disc_dim=10, cont_dim=10)
    trainer = DCInfoGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1)
