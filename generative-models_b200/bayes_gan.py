""" (BayesGAN) https://arxiv.org/abs/1705.09558
Bayesian GAN (Saatchi & Wilson 2017) on the MLP GAN engine.

The reference ships this model as a docstring only (src/bayes_gan.py); this module follows its description and the
conventions of the other MLP GANs (src/ns_gan.py: Generator, Discriminator, binary MNIST, `from bayes_gan import *`).
Instead of one point estimate of the generator, the model keeps J = num_g_samples generators G_1..G_J, samples from the
posterior over the generator weights, and trains one discriminator against all of them.  With the NS energies

    U_D = -mean_i log(D(x_i) + 1e-8) - mean_{j,i} log(1 - D(G_j(z_ji)) + 1e-8)     (the second mean over all J B fake rows)
    U_j = -mean_i log(D(G_j(z_ji)) + 1e-8)                                         (one energy per generator sample)

every net moves by stochastic-gradient Hamiltonian Monte Carlo (SGHMC, the paper's Algorithm 1 with beta = 0): with
momentum v, step size lr, friction alpha, a N(0, prior_std^2) prior and N = data_size training images,

    v <- (1 - alpha) v - lr (dU/dtheta + theta / (prior_std^2 N)) + sqrt(2 alpha lr / N) xi,   xi ~ N(0, 1)
    theta <- theta + v

v starts at rest at every train() call.  The energies, their gradients and the SGHMC updates run in the hand-written
sm_90a kernels of libgm_b200.so (the GAN engine in its Bayes mode); train() keeps the train split resident (1 bit per
pixel) and draws batches, noise and xi on the device.  With J = 1 the gradients are NSGAN's.  This trainer has no
user-written train_D / train_G path, and trains on one process.
"""
import os

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403

from gm_b200 import GmError, SghmcHP, BayesGanEngine
from gm_b200 import gan_api
from gm_b200.gan_api import to_cuda, builtin_step, DeviceDataset, G_NET, D_NET


class Generator(gan_api.Generator):
    """ One generator sample: noise -> hidden (ReLU) -> image (sigmoid), src/ns_gan.py:35-46 """
    _sample = 0

    def forward(self, x):
        x = to_cuda(x).float().contiguous()
        eng = self._engine_for(x.shape[0], "Generator")
        return eng.generate(self._sample, x)


class Discriminator(gan_api.Discriminator):
    """ Discriminator: image -> hidden (ReLU) -> probability that the image is real, src/ns_gan.py:49-60 """

    def forward(self, x):
        x = to_cuda(x).float().contiguous()
        return self._engine_for(x.shape[0], "Discriminator").discriminate(x)


class BayesGAN(nn.Module):
    """ J generator samples (model.G, an nn.ModuleList, each initialised on its own so the chains start apart) and one
    discriminator (model.D) """

    def __init__(self, image_size, hidden_dim, z_dim, num_g_samples=10, output_dim=1):
        super().__init__()
        if not 1 <= int(num_g_samples) <= 16:
            raise GmError("num_g_samples must be in [1, 16] (got %r)" % (num_g_samples,))
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim,
                                  num_g_samples=int(num_g_samples), output_dim=output_dim))
        self.G = nn.ModuleList([Generator(image_size, hidden_dim, z_dim) for _ in range(self.num_g_samples)])
        for j, g in enumerate(self.G):
            object.__setattr__(g, "_sample", j)
        self.D = Discriminator(image_size, hidden_dim, output_dim)
        self.shape = int(image_size ** 0.5)


def _overrides(tr):
    """the train_D / train_G of tr's class that are not this module's own"""
    return [m for m in ("train_D", "train_G") if not getattr(getattr(type(tr), m), "_gm_builtin", False)]


class BayesGANTrainer:
    """ Object to hold data iterators and train a Bayesian GAN """
    device_noise = True       # in-kernel Philox noise; False (or a compute_noise override): host noise through noise_dev

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.Glosses, self.Dlosses = [], []
        self.viz = viz
        self.num_epochs = 0
        self._engine, self._max_batch = None, None
        self._step, self._dcount = 0, 0      # G updates / D updates so far: the Philox keys of the noise and of xi
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        import weakref
        for mod in list(model.G) + [model.D]:
            object.__setattr__(mod, "_owner", weakref.ref(self))

    # ------------------------------------------------------------------ engine plumbing
    def _ensure_engine(self, batch):
        """Create (or grow) the engine; the model's parameters become views of its flat fp32 buffers."""
        if self._engine is not None and batch <= self._max_batch:
            return self._engine
        m, old = self.model, self._engine
        batch = max(batch, self._max_batch or 0, 64)
        eng = BayesGanEngine(m.image_size, m.hidden_dim, m.z_dim, num_g=m.num_g_samples, max_batch=batch)
        for j, g in enumerate(m.G):
            params = list(g.parameters())
            eng.load(G_NET, [p.data for p in params], sample=j)
            for p, v in zip(params, eng.views(G_NET, sample=j)):
                p.data = v
            g._attach(eng, G_NET)
        params = list(m.D.parameters())
        eng.load(D_NET, [p.data for p in params])
        for p, v in zip(params, eng.views(D_NET)):
            p.data = v
        m.D._attach(eng, D_NET)
        if old is not None:
            for net in (G_NET, D_NET):
                eng.momentum[net].copy_(old.momentum[net])
        self._engine, self._max_batch = eng, batch
        return eng

    def _use_device_noise(self):
        return self.device_noise and getattr(self.compute_noise, "__func__", None) is BayesGANTrainer.compute_noise

    def _refuse(self):
        bad = _overrides(self)
        if bad:
            raise GmError("the Bayesian GAN trains through its fused SGHMC step only: %s cannot be overridden" % " / ".join(bad))
        from gm_b200 import parallel as par
        if par.world_size() > 1:
            raise GmError("the Bayesian GAN trains on one process: there is no data-parallel Bayesian GAN")

    # ------------------------------------------------------------------ training
    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1, alpha=0.1, prior_std=1.0, data_size=None):
        """ Train the J generator samples and D with SGHMC: per outer step D_steps discriminator updates and one update
        of every generator sample; losses are logged per step and read back once per epoch """
        self._refuse()
        N = float(len(self.train_iter.dataset) if data_size is None else data_size)
        hpG, hpD = SghmcHP(G_lr, alpha, prior_std, N), SghmcHP(D_lr, alpha, prior_std, N)
        if self._engine is not None:
            self._engine.reset_optimizer()                  # v starts at rest at every train() call
            self._engine.sync_all()
        resident = DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None))
        self._resident = resident
        epoch_steps = int(np.ceil(len(self.train_iter) / D_steps))
        dev = self._use_device_noise()
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            ring = torch.zeros(D_steps + 1, epoch_steps, device="cuda")
            for i in range(epoch_steps):
                for k in range(D_steps):
                    if resident is not None:
                        batch = min(resident.batch_size, resident.n)
                        eng = self._ensure_engine(batch)
                        eng.set_sampler(resident.n, self._seed ^ 0x5DEECE66D)
                        noise = None if dev else self._noise(batch)
                        eng.d_grad(resident.bits, noise=noise, fmt="bits", batch=batch, seed=self._seed, step=self._dcount,
                                   loss_out=ring[k, i])
                    else:
                        images = self.process_batch(self.train_iter)
                        batch = images.shape[0]
                        eng = self._ensure_engine(batch)
                        eng.set_sampler(0)
                        noise = None if dev else self._noise(batch)
                        eng.d_grad(images, noise=noise, seed=self._seed, step=self._dcount, loss_out=ring[k, i])
                    eng.apply(D_NET, hpD, seed=self._seed, step=self._dcount)
                    self._dcount += 1
                noise = None if dev else self._noise(batch)
                eng.g_grad(batch, noise=noise, seed=self._seed, step=self._step, loss_out=ring[D_steps, i])
                eng.apply(G_NET, hpG, seed=self._seed, step=self._step)
                self._step += 1
            G_losses = ring[D_steps].tolist()
            D_losses = ring[:D_steps].mean(dim=0).tolist()
            self.Glosses.extend(G_losses)
            self.Dlosses.extend(D_losses)
            print("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f" % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses)))
            self.num_epochs += 1
            if self.viz:
                self.generate_images(epoch)

    def _noise(self, batch):
        """compute_noise for every generator sample's rows: [num_g * batch, z], sample-major"""
        return self.compute_noise(self.model.num_g_samples * batch, self.model.z_dim).float().contiguous()

    @builtin_step
    def train_D(self, images):
        """ U_D of a batch and D's gradient (in the engine's gradient buffer); train() applies SGHMC after it """
        images = to_cuda(images.reshape(images.shape[0], -1)).float().contiguous()
        self._refuse()
        eng = self._ensure_engine(images.shape[0])
        eng.set_sampler(0)
        return eng.d_grad(images, noise=self._noise(images.shape[0])).clone()

    @builtin_step
    def train_G(self, images):
        """ mean_j U_j of a batch and every generator sample's gradient; train() applies SGHMC after it """
        self._refuse()
        eng = self._ensure_engine(images.shape[0])
        return eng.g_grad(images.shape[0], noise=self._noise(images.shape[0])).clone()

    def compute_noise(self, batch_size, z_dim):
        """ Random noise for the generators (src/ns_gan.py:218-220) """
        return to_cuda(torch.randn(batch_size, z_dim))

    def process_batch(self, iterator):
        """ A processed batch for D (src/ns_gan.py:222-226) """
        images, _ = next(iter(iterator))
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    def generate_images(self, epoch=-100, num_outputs=36, save=True):
        """ Samples from the posterior predictive: num_outputs images spread over the J generator samples """
        self.model.eval()
        noise = self.compute_noise(num_outputs, self.model.z_dim)
        chunks = [c for c in torch.tensor_split(noise, self.model.num_g_samples) if c.shape[0] > 0]
        with torch.no_grad():
            images = torch.cat([self.model.G[j](c) for j, c in enumerate(chunks)])
        images = images.view(images.shape[0], self.model.shape, self.model.shape, -1).squeeze()
        if save:
            try:
                import torchvision
                outname = "../viz/" + self.name + "/"
                os.makedirs(outname, exist_ok=True)
                torchvision.utils.save_image(images.unsqueeze(1).data.cpu(), outname + "reconst_%d.png" % epoch,
                                             nrow=int(num_outputs ** 0.5))
            except Exception as e:  # pragma: no cover
                print("generate_images: not saved (%s)" % e)
        return images

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.Dlosses)), self.Dlosses, "r")
        plt.plot(np.linspace(1, self.num_epochs, len(self.Glosses)), self.Glosses, "g")
        plt.legend(["Discriminator", "Generator"])
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
    model = BayesGAN(image_size=784, hidden_dim=400, z_dim=20, num_g_samples=10)
    trainer = BayesGANTrainer(model=model, train_iter=train_iter, val_iter=val_iter, test_iter=test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1)
