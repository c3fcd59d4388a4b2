""" (DCVAE) Variational autoencoder with a deep-convolutional encoder and decoder, on 64x64 images - the conv VAE the
reference's README recommends ("use deep convolutional architectures (i.e. DCGANs) ... by editing ... the Encoder and
Decoder classes for VAEs", README.md:68).

The class surface is src/vae.py's, so its driver code runs on the conv model:

    model = DCVAE(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCVAETrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)

  Encoder: the DCGAN discriminator trunk, Conv(ch, h, 4, 2, 1) LReLU(0.2) -> Conv(h, 2h) BN LReLU -> Conv(2h, 4h) BN LReLU
           -> Conv(4h, 8h) BN LReLU, with two linear heads mu = Conv2d(8h, z, 4, 1, 0) and log_var = Conv2d(8h, z, 4, 1, 0)
           (the roles of src/vae.py:47-61's Encoder.mu / Encoder.log_var).
  Decoder: the DCGAN generator, ConvT(z, 8h, 4, 1, 0) BN ReLU -> ... -> ConvT(h, ch, 4, 2, 1) -> sigmoid.

Every conv is bias-free, as everywhere on the conv path (the reference's MLP heads are nn.Linear with biases; here the
heads follow the DCGAN convention and BatchNorm's shift provides the offsets).  The losses are the reference's code
(src/vae.py:193-212): recon = sum (x - out)^2 over all pixels of the batch, KL = sum 0.5 (mu^2 + e^lv - lv - 1), with
z = mu + eps e^(lv/2), and one Adam with coupled weight decay over all parameters (src/vae.py:139-142).  BatchNorm follows
model.training: train() uses batch statistics and updates the running ones, eval() (validation, best_model) normalises with
the running statistics.  All arithmetic runs in the sm_90a kernels behind gm_b200.DcganEngine(variant="vae"); the modules
only hold the parameters, so state_dict() has encoder.* / decoder.* keys in torch's layouts.  Under torchrun the trainer is
data-parallel: replicas start from rank 0's parameters, eps is drawn per rank, and the gradients (of sums, so they need no
rescaling) are summed before each Adam step; BatchNorm statistics stay per rank.
"""
import weakref
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError, DcganEngine
from gm_b200 import parallel as par
from gm_b200.dcgan import DevicePool
from gm_b200.gan_api import (to_cuda, builtin_step, first_order, has_custom_compute_batch, refuse_multi_rank, compute_batch_loop,
                             compute_batch_evaluate)
from torch.autograd.function import once_differentiable
from dc_gan import EngineSync, dcgan_init, module_params, pull_running_stats, push_running_stats, _grads_for, _node_args


def _parent_of(module, what):
    parent = module._parent() if getattr(module, "_parent", None) is not None else None
    if parent is None:
        raise GmError(what + " is not part of a DCVAE: construct it through DCVAE(...)")
    return parent


class _EncoderCall(torch.autograd.Function):
    """Encoder.forward in training mode under grad mode: the VAE's (mu, log_var) or the autoencoder's code and their
    backward on the conv kernels (DcganEngine.custom_d_forward / custom_d_backward); autograd routes the upstream in and
    the encoder's parameter gradients out"""

    @staticmethod
    def forward(ctx, x, parent, eng, mod, names, *params):
        out, ctx.handle = eng.custom_d_forward(x)
        ctx.parent, ctx.eng, ctx.mod, ctx.names = parent, eng, mod, names
        return out

    @staticmethod
    @first_order
    @once_differentiable
    def backward(ctx, *dout):
        grads, _ = ctx.eng.custom_d_backward(ctx.handle, dout if len(dout) == 2 else dout[0], ctx.needs_input_grad[0])
        return (None, None, None, None, None, *_grads_for(ctx.parent._module_names(grads), "D", ctx.mod, ctx.names))


class _DecoderCall(torch.autograd.Function):
    """Decoder.forward in training mode under grad mode: the images and their backward, with dL/dz when z requires grad"""

    @staticmethod
    def forward(ctx, z, eng, mod, names, *params):
        out, ctx.handle = eng.custom_g_forward(z)
        ctx.eng, ctx.mod, ctx.names = eng, mod, names
        return out

    @staticmethod
    @first_order
    @once_differentiable
    def backward(ctx, dimages):
        grads, dz = ctx.eng.custom_g_backward(ctx.handle, dimages.float().contiguous(), need_dz=True)
        return ((dz if ctx.needs_input_grad[0] else None), None, None, None, *_grads_for(grads, "G", ctx.mod, ctx.names))


def _encoder_forward(mod, x):
    """Encoder.forward of the VAE and the autoencoder: per-call kernels with a backward in training mode under grad mode,
    the inference calls otherwise"""
    x = to_cuda(x).float()
    parent = _parent_of(mod, "Encoder")
    eng = parent._engine()
    if torch.is_grad_enabled() and mod.training:
        out = _EncoderCall.apply(x.reshape(x.shape[0], -1), parent, eng, *_node_args(mod))
    else:
        out = eng.encode(x.reshape(x.shape[0], -1), train=mod.training)
    parent._after_forward(eng, mod.training)
    return out


class Encoder(nn.Module):
    """ Conv encoder for the VAE: 64x64 image -> (mu, log_var) of the latent variable z pre-reparametrization """

    def __init__(self, image_size, hidden_dim, z_dim, channels=3):
        super().__init__()
        c = [hidden_dim, 2 * hidden_dim, 4 * hidden_dim, 8 * hidden_dim]
        self.l1 = nn.Conv2d(channels, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])
        self.mu = nn.Conv2d(c[3], z_dim, 4, 1, 0, bias=False)
        self.log_var = nn.Conv2d(c[3], z_dim, 4, 1, 0, bias=False)

    def forward(self, x):
        return _encoder_forward(self, x)


class Decoder(nn.Module):
    """ Conv decoder for the VAE (the DCGAN generator): z -> 4x4 -> ... -> 64x64 image, sigmoid output """

    def __init__(self, z_dim, hidden_dim, image_size, channels=3):
        super().__init__()
        c = [8 * hidden_dim, 4 * hidden_dim, 2 * hidden_dim, hidden_dim, channels]
        self.l1 = nn.ConvTranspose2d(z_dim, c[0], 4, 1, 0, bias=False)
        self.l2 = nn.ConvTranspose2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.ConvTranspose2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.ConvTranspose2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.ConvTranspose2d(c[3], c[4], 4, 2, 1, bias=False)
        self.bn1, self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[:4])

    def forward(self, z):
        z = to_cuda(z).float()
        if z.dim() == 1:                       # the reference decodes single latent vectors too (src/vae.py:289-290)
            z = z.view(1, -1)
        parent = _parent_of(self, "Decoder")
        eng = parent._engine()
        if torch.is_grad_enabled() and self.training:
            out = _DecoderCall.apply(z, eng, *_node_args(self))
        else:
            out = eng.decode(z, train=self.training)
        parent._after_forward(eng, self.training)
        return out


def _engine_names(named):
    """{"G." / "D." + module parameter name: tensor} -> the engine's names: D.mu and D.log_var stacked into D.l5"""
    out = dict(named)
    out["D.l5.weight"] = torch.cat([out.pop("D.mu.weight"), out.pop("D.log_var.weight")])
    return out


def _module_names(tensors, z):
    """the inverse of _engine_names"""
    out = dict(tensors)
    l5 = out.pop("D.l5.weight")
    out["D.mu.weight"], out["D.log_var.weight"] = l5[:z], l5[z:2 * z]
    return out


class DCVAE(nn.Module):
    """ VAE super class to reconstruct an image (as src/vae.py:80-106), with conv encoder and decoder """
    variant = "vae"                                    # the DcganEngine variant that trains this model
    _Encoder = Encoder

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, channels=3):
        super().__init__()
        if image_size != 64 * 64 * channels:
            raise GmError("the conv path is built for 64x64 images (image_size = 64*64*channels)")
        if hidden_dim % 16 or hidden_dim <= 0 or z_dim <= 0:
            raise GmError("hidden_dim must be a positive multiple of 16 and z_dim positive")
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, channels=channels))
        self.encoder = self._Encoder(image_size, hidden_dim, z_dim, channels)
        self.decoder = Decoder(z_dim, hidden_dim, image_size, channels)
        dcgan_init(self)
        self.shape = 64
        for mod in (self.encoder, self.decoder):
            object.__setattr__(mod, "_parent", weakref.ref(self))
        object.__setattr__(self, "_owner", None)        # weakref to the DCVAETrainer that trains this model
        object.__setattr__(self, "_own_engine", None)   # private inference engine of a detached copy

    def _nets(self):
        """(state_dict prefix, module) of the engine's two nets: G is the decoder, D the encoder"""
        return [("G", self.decoder), ("D", self.encoder)]

    def _engine_names(self, named):
        """{"G." / "D." + module parameter name: tensor} -> the engine's names (_engine_names)"""
        return _engine_names(named)

    def _module_names(self, tensors):
        """the inverse of the method _engine_names"""
        return _module_names(tensors, self.z_dim)

    def _engine(self):
        """the trainer's engine, or - for a model without one, such as DCVAETrainer.best_model - a private engine loaded
        from this module's parameters and running statistics"""
        owner = self._owner() if self._owner is not None else None
        if owner is not None:
            return owner._engine_synced()
        if not torch.cuda.is_available():
            raise GmError("DCVAE is not attached to a CUDA engine: there is no eager / CPU path")
        if self._own_engine is None:
            object.__setattr__(self, "_own_engine", DcganEngine(self.hidden_dim, self.z_dim, self.channels, variant=self.variant))
        self._own_engine.load_torch_weights(self._engine_names(module_params(self._nets())))
        push_running_stats(self._own_engine, self._nets())
        return self._own_engine

    def _after_forward(self, eng, train):
        """a training-mode forward updated the engine's running statistics: the BatchNorm modules take them, as torch's
        would"""
        if train:
            pull_running_stats(eng, self._nets())

    def __deepcopy__(self, memo):
        """A detached copy (the reference keeps best_model = deepcopy(model), src/vae.py:178-180): same class, cloned
        parameters and statistics, no link to the trainer's engine.  The new module's initialisation draws are taken on a
        forked RNG, so that copying leaves torch's random stream (the eps of later forwards) where it was."""
        with torch.random.fork_rng(devices=[]):
            new = type(self)(self.image_size, self.hidden_dim, self.z_dim, self.channels)
        new.load_state_dict({k: v.detach().clone() for k, v in self.state_dict().items()})
        new.train(self.training)
        return new

    def forward(self, x):
        x = to_cuda(x).float()
        n = x.shape[0]
        if torch.is_grad_enabled() and self.training:               # src/vae.py:94-98 on the differentiable encoder / decoder
            mu, log_var = self.encoder(x)
            z = self.reparameterize(mu, log_var)
            return self.decoder(z), mu, log_var
        eng = self._engine()
        eps = torch.randn(n, self.z_dim, device=eng.device)                                # src/vae.py:104
        out, mu, lv, _ = eng.vae_forward(eng.stage_images(x.reshape(n, -1)), n, eps=eps, train=self.training)
        self._after_forward(eng, self.training)
        return out, mu, lv

    def reparameterize(self, mu, log_var):
        """ z = mean + std * epsilon (src/vae.py:100-106); plain torch for direct use """
        epsilon = torch.randn(mu.shape, device=mu.device)
        return mu + epsilon * torch.exp(log_var / 2)


class DCVAETrainer(EngineSync):
    """ Object to hold data iterators, train the conv VAE (surface of src/vae.py:109-374) """
    _two_losses = True                  # compute_batch returns (recon, kl)

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.best_val_loss = 1e10
        self.debugging_image, _ = next(iter(test_iter))
        self.viz = viz
        self.kl_loss, self.recon_loss = [], []
        self.num_epochs = 0
        # _dirty: the module parameters are newer than the engine's (construction, load_model, an optimizer step after
        # compute_batch); _stats_dirty: the modules' BatchNorm running statistics are (construction, load_model).  Otherwise
        # the engine's statistics are the current ones: every training-mode forward updates them there.
        self._engine, self._dirty, self._stats_dirty, self._step = None, True, True, 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        object.__setattr__(model, "_owner", weakref.ref(self))

    # ------------------------------------------------------------------ engine <-> module parameters (dc_gan.EngineSync)
    def _nets(self):
        return self.model._nets()

    def _sd(self):
        return self.model._engine_names(super()._sd())

    def _torch_tensors(self, grads=False):
        return self.model._module_names(super()._torch_tensors(grads))

    def _engine_synced(self):
        m = self.model
        if self._engine is None:
            self._engine = DcganEngine(m.hidden_dim, m.z_dim, m.channels, variant=m.variant)
            self._dirty = self._stats_dirty = True
        if self._dirty:
            self._engine.load_torch_weights(self._sd())
            self._dirty = False
        if self._stats_dirty:
            push_running_stats(self._engine, self._nets())
            self._stats_dirty = False
        return self._engine

    # ------------------------------------------------------------------ reference surface
    def train(self, num_epochs, lr=1e-3, weight_decay=1e-5):
        """ Train a Variational Autoencoder (src/vae.py:127-191): a true epoch over train_iter with eps drawn on the device,
        losses read back once per epoch, model.eval() validation, best model kept as a detached copy.  A subclass's own
        compute_batch (README.md:31) is trained by the reference loop over the differentiable encoder / decoder instead
        (gan_api.compute_batch_loop; train_iter is read on the host, device_dataset does not apply). """
        import torch.distributed as dist
        if has_custom_compute_batch(self):
            return self._train_custom(num_epochs, lr, weight_decay)
        eng = self._engine_synced()
        hp = AdamHP.make(lr, weight_decay=weight_decay)
        for net in eng.nets():                                      # a fresh optimizer per train() call (src/vae.py:139-142)
            net.exp_avg.zero_(); net.exp_avg_sq.zero_(); net.step = 0
        world, rank = par.world_size(), par.rank_of()
        if world > 1:                                               # replicas start from rank 0's parameters
            for net in eng.nets():
                dist.broadcast(net.params, src=0)
                net.refresh()
        seed = par.rank_seed(self._seed, rank)
        pool = self._device_pool()
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            per_step = []
            for rows, n in (self._pool_batches(eng, pool, seed) if pool is not None else self._host_batches(eng)):
                per_step.append(self._grad_step(eng, rows, n, seed).clone())
                par.sum_gradients(eng.G.grads)                      # NCCL SUM (no-op on one GPU): the losses are sums
                par.sum_gradients(eng.D.grads)
                eng.apply(hp)
                self._step += 1
            vals = torch.stack(per_step).tolist()
            self.model.eval()
            val_loss = self.evaluate(self.val_iter)
            if val_loss < self.best_val_loss:
                self._pull()
                self.best_model = deepcopy(self.model)
                self.best_val_loss = val_loss
            print(self._log_epoch(epoch, num_epochs, vals, val_loss))
            self.num_epochs += 1
            if self.viz:
                self.sample_images(epoch)
        self._pull()

    def _train_custom(self, num_epochs, lr, weight_decay):
        refuse_multi_rank()
        eng = self._engine_synced()
        self.model.to(eng.device)                   # the reference's to_cuda(model): Adam runs on the device

        def after_step():
            self._dirty = True                      # the module parameters are newer than the engine's
        compute_batch_loop(self, num_epochs, lr, weight_decay, self._two_losses, after_step)

    def _grad_step(self, eng, rows, n, seed):
        """one train step's gradients into eng.G.grads / eng.D.grads; returns its losses (this process's sums)"""
        return eng.vae_grad(rows, n, seed=seed, step=self._step)

    def _log_epoch(self, epoch, num_epochs, vals, val_loss):
        """keeps an epoch's per-step losses vals and returns its progress line (src/vae.py:172-187)"""
        epoch_recon, epoch_kl = [v[0] for v in vals], [v[1] for v in vals]
        epoch_loss = [a + b for a, b in zip(epoch_recon, epoch_kl)]
        self.kl_loss.extend(epoch_kl)
        self.recon_loss.extend(epoch_recon)
        return ("Epoch[%d/%d], Total Loss: %.4f, Reconst Loss: %.4f, KL Div: %.7f, Val Loss: %.4f"
                % (epoch, num_epochs, np.mean(epoch_loss), np.mean(epoch_recon), np.mean(epoch_kl), val_loss))

    def _host_batches(self, eng):
        """one epoch of train_iter: (NHWC bf16 rows, n) per batch"""
        for batch in self.train_iter:
            images = self._images(batch)
            yield eng.stage_images(images), images.shape[0]

    def _pool_batches(self, eng, pool, seed):
        """one epoch drawn on the device from the DevicePool: batch k stages rows [kB, min((k+1)B, N)) of this epoch's
        permutation (round = the epochs trained so far), so every image is used once per epoch, as by a shuffling loader"""
        B = pool.batch_size
        for k in range(len(self.train_iter)):
            n = min(B, pool.n - k * B)
            yield eng.stage_pool(pool, n, seed ^ DevicePool.SEED_MIX, self.num_epochs, offset=k * B), n

    def _images(self, batch):
        images, _ = batch
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    @builtin_step
    def compute_batch(self, batch):
        """ Compute loss for a batch of examples (src/vae.py:193-208): returns (recon, kl); (recon + kl).backward() delivers
        the engine's gradient of their sum to the module parameters (it rides on recon; kl carries none) """
        images = self._images(batch)
        eng = self._engine_synced()
        n = images.shape[0]
        eps = torch.randn(n, self.model.z_dim, device=eng.device)                           # src/vae.py:104
        losses = eng.vae_grad(eng.stage_images(images), n, eps=eps).clone()
        pull_running_stats(eng, self._nets())                     # the training-mode forward's update, as torch makes it
        recon = self._fused_loss(self._nets(), losses[0])
        return recon, losses[1]

    def kl_divergence(self, mu, log_var):
        """ Compute Kullback-Leibler divergence (src/vae.py:210-212; torch, for direct use) """
        return torch.sum(0.5 * (mu ** 2 + torch.exp(log_var) - log_var - 1))

    def evaluate(self, iterator):
        """ Evaluate on a given dataset (src/vae.py:214-223): recon + kl per batch with the forward-only kernels, BatchNorm
        in the model's mode; with an overriding compute_batch, its losses as the reference does """
        if has_custom_compute_batch(self):
            return compute_batch_evaluate(self, iterator, self._two_losses)
        eng = self._engine_synced()
        loss = []
        for batch in iterator:
            images = self._images(batch)
            n = images.shape[0]
            eps = torch.randn(n, self.model.z_dim, device=eng.device)
            _, _, _, ls = eng.vae_forward(eng.stage_images(images), n, eps=eps, train=self.model.training)
            loss.append(ls.sum())
        self.model._after_forward(eng, self.model.training)
        return float(torch.stack(loss).mean().item())

    def reconstruct_images(self, images, epoch, save=True):
        """ src/vae.py:225-252 without the plotting: the reconstructions in the images' shape """
        batch = to_cuda(images.view(images.shape[0], -1))
        with torch.no_grad():
            reconst_images, _, _ = self.model(batch)
        return reconst_images.view(images.shape).squeeze()

    def sample_images(self, epoch=-100, num_images=36, save=True):
        """ Viz method 1 (src/vae.py:254-276): z ~ p(z), x ~ p(x|z) """
        z = to_cuda(torch.randn(num_images, self.model.z_dim))
        with torch.no_grad():
            sample = self.model.decoder(z)
        return sample.view(num_images, self.model.channels, self.model.shape, self.model.shape)

    def sample_interpolated_images(self):
        """ Viz method 2 (src/vae.py:278-293): decode the interpolation between two random latent vectors; returns the
        list of decoded images instead of displaying them """
        z1 = torch.normal(torch.zeros(self.model.z_dim), 1)
        z2 = torch.normal(torch.zeros(self.model.z_dim), 1)
        out = []
        for alpha in np.linspace(0, 1, self.model.z_dim):
            z = to_cuda(float(alpha) * z1 + (1 - float(alpha)) * z2)
            with torch.no_grad():
                out.append(self.model.decoder(z).view(-1, self.model.channels, self.model.shape, self.model.shape))
        return out

    def explore_latent_space(self, num_epochs=3):
        """ Viz method 3 (src/vae.py:295-334) trains a VAE with z = 2 on MNIST at 28x28, which this 64x64 conv model
        cannot take """
        raise GmError("explore_latent_space trains the reference's 784-400-2 MNIST VAE: use vae.VAETrainer.explore_latent_space")

    def make_all(self):
        """ src/vae.py:336-346: its last step is explore_latent_space (MNIST at 28x28, z = 2) """
        raise GmError("make_all ends in explore_latent_space on 28x28 MNIST with z = 2: use vae.VAETrainer.make_all")

    def viz_loss(self):
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.recon_loss)), self.recon_loss, "r")
        plt.plot(np.linspace(1, self.num_epochs, len(self.kl_loss)), self.kl_loss, "g")
        plt.legend(["Reconstruction", "Kullback-Leibler"])
        plt.title(self.name)
        plt.show()

    def save_model(self, savepath):
        """ Save model state dictionary (src/vae.py:367-369) """
        if not self._dirty:
            self._pull()
        elif self._engine is not None:                           # module weights are newer; the statistics are the engine's
            pull_running_stats(self._engine, self._nets())
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        """ Load state dictionary into model (src/vae.py:371-374) """
        self.model.load_state_dict(torch.load(loadpath))
        self._dirty = self._stats_dirty = True


if __name__ == "__main__":
    imgs = (torch.rand(8192, 3, 64, 64) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCVAE(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCVAETrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=5, lr=1e-3, weight_decay=1e-5)
