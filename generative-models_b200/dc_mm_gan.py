""" (DCMMGAN) Minimax GAN with the DCGAN convolutional G / D, on 64x64 images.

The class surface is src/mm_gan.py's, so its driver code runs on the conv model:

    model = DCMMGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCMMGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1, G_init=5)

L(D) is NSGAN's -mean(log(D(x) + 1e-8) + log(1 - D(G(z)) + 1e-8)); L(G) is the minimax mean(log(1 - D(G(z)) + 1e-8))
(src/mm_gan.py:214-235), both rows of the loss kernel (gm_b200.DcganEngine(variant="mm")) on the batch-norm DCGAN D's
logits.  train() first pre-trains G for G_init steps with the same optimizer (src/mm_gan.py:119-138).
"""
import torch  # noqa: F401
import torch.nn as nn  # noqa: F401

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError  # noqa: F401
from gm_b200 import parallel as par
from dc_gan import Generator, Discriminator, DCGAN, DCGANTrainer  # noqa: F401


class DCMMGAN(DCGAN):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/mm_gan.py:66-77) """


class DCMMGANTrainer(DCGANTrainer):
    """ Object to hold data iterators, train the conv MMGAN (surface of src/mm_gan.py:80-310) """
    variant = "mm"
    _G_init, _G_lr = 0, 2e-4

    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1, G_init=5):
        """ Trainer.train (src/mm_gan.py:97-186) on the fused conv step """
        self._G_init, self._G_lr = int(G_init), G_lr
        super().train(num_epochs, G_lr=G_lr, D_lr=D_lr, D_steps=D_steps)

    def _pre_train(self, eng):
        """G_init G steps before the joint loop (src/mm_gan.py:119-138), on G's freshly reset optimizer"""
        if self._G_init <= 0:
            print("G not pre-trained -- GAN unlikely to converge.")
            return
        hp, world = AdamHP.make(self._G_lr), par.world_size()
        seed = par.rank_seed(self._seed, par.rank_of())
        for _ in range(self._G_init):
            n = self.process_batch(self.train_iter).shape[0]      # the batch size train_G would see (src/mm_gan.py:124-128)
            eng.g_grad(n, inv_global_batch=par.inv_global_batch(n, world), seed=seed, step=self._step)
            par.sum_gradients(eng.G.grads)
            eng.apply(0, hp)
            self._step += 1
        print("G pre-trained for {0} training steps.".format(self._G_init))


if __name__ == "__main__":
    imgs = torch.rand(8192, 3, 64, 64)
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCMMGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCMMGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1, G_init=5)
