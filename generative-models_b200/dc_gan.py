""" (DCGAN) NSGAN with deep-convolutional G / D — the model the reference's README recommends ("for more complex
datasets ... DCGAN", README.md:68) and lists under To-Do (README.md:96); BASELINE configs[4]: 64x64x3 images.

There is no src/dc_gan.py in the reference.  This module gives the conv model the SAME class surface as src/ns_gan.py
so the reference's driver code runs on it unchanged:

    model = DCGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCGANTrainer(model, train_iter, val_iter, test_iter, viz=False)
    trainer.train(num_epochs=25, G_lr=2e-4, D_lr=2e-4, D_steps=1)

Losses, loop and optimizers are NSGAN's (src/ns_gan.py:94-216); images cross the class boundary flattened to
[B, image_size] exactly as process_batch produces them (src/ns_gan.py:222-226) and D un-flattens.  All arithmetic runs
in the sm_90a kernels behind gm_b200.DcganEngine (im2col / col2im + wgmma GEMMs, BatchNorm, loss, Adam); the
nn.Conv2d / nn.ConvTranspose2d / nn.BatchNorm2d members only hold the parameters in torch's layouts, so state_dict()
has the usual DCGAN keys and shapes.  Under torchrun the trainer is data-parallel: per-rank batches and noise, NCCL
all-reduce (SUM) of the flat G and D gradients before each Adam step.

A subclass may override train_D / train_G with its own torch loss, as the reference's README invites (README.md:31):
under grad mode model.G / model.D are autograd nodes whose forward and backward are the same kernels, and train() then
runs the reference's loop (src/ns_gan.py:107-156) on one process with Adam over the module parameters (FusedAdam).
"""
import numpy as np
import torch
import torch.nn as nn

from utils import *  # noqa: F401,F403
from gm_b200 import AdamHP, GmError, DcganEngine
from gm_b200 import parallel as par
from gm_b200.dcgan import DevicePool
from gm_b200.gan_api import to_cuda, EngineCall, GradHandoff, flat_pairs, FusedAdam, builtin_step, reference_loop


class Generator(nn.Module):
    """ z -> 4x4 -> 8x8 -> 16x16 -> 32x32 -> 64x64 (transposed convolutions, BatchNorm + ReLU, sigmoid output) """

    def __init__(self, image_size, hidden_dim, z_dim, channels=3):
        super().__init__()
        c = [8 * hidden_dim, 4 * hidden_dim, 2 * hidden_dim, hidden_dim, channels]
        self.l1 = nn.ConvTranspose2d(z_dim, c[0], 4, 1, 0, bias=False)
        self.l2 = nn.ConvTranspose2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.ConvTranspose2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.ConvTranspose2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.ConvTranspose2d(c[3], c[4], 4, 2, 1, bias=False)
        self.bn1, self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[:4])
        self._owner = None

    def forward(self, x):
        tr = self._owner
        if tr is None:
            raise GmError("Generator is not attached to a CUDA engine yet: construct the DCGANTrainer first")
        eng = tr._engine_synced()
        if torch.is_grad_enabled() and eng.supports_custom_loss:   # G(z) and its backward on the conv kernels
            named = list(self.named_parameters())

            def backward(handle, grads, need_dx):
                g = eng.custom_g_backward(handle, grads[0].float().contiguous())
                return None, [g["G." + k].contiguous().to(p.device) for k, p in named]
            return EngineCall.apply(to_cuda(x).float(), eng.custom_g_forward, backward, *(p for _, p in named))
        return eng.generate(to_cuda(x).float())


class Discriminator(nn.Module):
    """ 64x64 -> 32x32 -> 16x16 -> 8x8 -> 4x4 -> 1 (convolutions + LeakyReLU(0.2), BatchNorm on layers 2-4 unless
    batch_norm=False, output activation out_act: one of the class's out_acts) """
    out_acts = ("sigmoid",)

    def __init__(self, image_size, hidden_dim, output_dim=1, channels=3, batch_norm=True, out_act="sigmoid"):
        super().__init__()
        if output_dim != 1:
            raise GmError("only output_dim=1 discriminators are built")
        if out_act not in self.out_acts:
            raise GmError("the output activation of %s is one of %s" % (type(self).__name__, ", ".join(self.out_acts)))
        c = [hidden_dim, 2 * hidden_dim, 4 * hidden_dim, 8 * hidden_dim]
        self.l1 = nn.Conv2d(channels, c[0], 4, 2, 1, bias=False)
        self.l2 = nn.Conv2d(c[0], c[1], 4, 2, 1, bias=False)
        self.l3 = nn.Conv2d(c[1], c[2], 4, 2, 1, bias=False)
        self.l4 = nn.Conv2d(c[2], c[3], 4, 2, 1, bias=False)
        self.l5 = nn.Conv2d(c[3], 1, 4, 1, 0, bias=False)
        if batch_norm:
            self.bn2, self.bn3, self.bn4 = (nn.BatchNorm2d(k) for k in c[1:])
        self.out_act = out_act
        self._owner = None

    def forward(self, x):
        tr = self._owner
        if tr is None:
            raise GmError("Discriminator is not attached to a CUDA engine yet: construct its trainer first")
        eng = tr._engine_synced()
        if torch.is_grad_enabled() and eng.supports_custom_loss:   # D(x) and its backward, with dL/dx when x requires grad
            named = list(self.named_parameters())

            def backward(handle, grads, need_dx):
                g, dx = eng.custom_d_backward(handle, grads[0].float(), need_dx)
                return dx, [g["D." + k].contiguous().to(p.device) for k, p in named]
            return EngineCall.apply(to_cuda(x).float().reshape(x.shape[0], -1), eng.custom_d_forward, backward,
                                    *(p for _, p in named))
        return eng.discriminate(to_cuda(x).float().reshape(x.shape[0], -1))


class DCGAN(nn.Module):
    """ Super class to contain both Discriminator (D) and Generator (G) (as src/ns_gan.py:63-74).  A subclass names its
    discriminator class in _D; d_options are that class's keyword options (e.g. the WGAN-GP critic's out_act). """
    _D = Discriminator

    def __init__(self, image_size=64 * 64 * 3, hidden_dim=64, z_dim=100, output_dim=1, channels=3, **d_options):
        super().__init__()
        if image_size != 64 * 64 * channels:
            raise GmError("the conv path is built for 64x64 images (image_size = 64*64*channels)")
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, output_dim=output_dim,
                                  channels=channels))
        self.G = Generator(image_size, hidden_dim, z_dim, channels)
        self.D = self._D(image_size, hidden_dim, output_dim, channels, **d_options)
        dcgan_init(self)
        self.shape = 64


def dcgan_init(module):
    """DCGAN initialisation (Radford et al. 2015) of every conv / BatchNorm layer in module"""
    for m in module.modules():
        if isinstance(m, (nn.Conv2d, nn.ConvTranspose2d)):
            nn.init.normal_(m.weight, 0.0, 0.02)
        elif isinstance(m, nn.BatchNorm2d):
            nn.init.normal_(m.weight, 1.0, 0.02)
            nn.init.zeros_(m.bias)


def module_params(nets):
    """{"<prefix>.<name>": parameter} of the (state_dict prefix, module) pairs nets"""
    return {"%s.%s" % (tag, k): v.detach() for tag, mod in nets for k, v in mod.named_parameters()}


def pull_running_stats(eng, nets):
    """eng's BatchNorm running statistics -> the bn1..bn4 buffers of the (state_dict prefix, module) pairs nets"""
    runs = {"G": eng.run_G, "D": eng.run_D, "Q": eng.run_Q}
    with torch.no_grad():
        for tag, mod in nets:
            for i, bn in ((i, getattr(mod, "bn%d" % i, None)) for i in range(1, 5)):       # a critic may have none
                run = runs[tag].get(i - 1)
                if bn is not None and run is not None:
                    bn.running_mean.copy_(run[0].cpu())
                    bn.running_var.copy_(run[1].cpu())


def push_running_stats(eng, nets):
    """the BatchNorm running statistics of the (state_dict prefix, module) pairs nets -> eng (the inverse of
    pull_running_stats)"""
    runs = {"G": eng.run_G, "D": eng.run_D}
    with torch.no_grad():
        for tag, mod in nets:
            for i, r in runs[tag].items():
                bn = getattr(mod, "bn%d" % (i + 1))
                r[0].copy_(bn.running_mean)
                r[1].copy_(bn.running_var)


class EngineSync:
    """Parameter sync between a trainer's DcganEngine (self._engine) and its model's modules (self._nets(): (state_dict
    prefix, module) pairs); self._dirty marks module parameters newer than the engine's"""
    # device_dataset: keep train_iter's images in HBM as 8-bit codes (gm_b200.dcgan.DevicePool) and draw each train() batch on
    # the device, when the loader is eligible.  Off by default: train() then fetches every batch through the host loader.
    device_dataset = False

    def _sd(self):
        return module_params(self._nets())

    def _torch_tensors(self, grads=False):
        """the engine's parameters (grads=True: gradients) in torch's layouts under the modules' "<prefix>.<name>" names"""
        return self._engine.torch_grads() if grads else self._engine.torch_weights()

    def _pull(self):
        """engine -> module parameters (after training; before state_dict / save_model)"""
        if self._engine is None:
            return
        tw = self._torch_tensors()
        with torch.no_grad():
            for tag, mod in self._nets():
                for k, v in mod.named_parameters():
                    v.copy_(tw["%s.%s" % (tag, k)].to(v.device))
        pull_running_stats(self._engine, self._nets())

    def _device_pool(self):
        """train_iter's images as a DevicePool when device_dataset is on and the loader is eligible (kept for later train()
        calls), else None: the batches then come from the host loader"""
        if not self.device_dataset:
            return None
        self._pool = DevicePool.from_loader(self.train_iter, self.model.channels, getattr(self, "_pool", None))
        return self._pool

    def _fused_loss(self, mods, loss_val):
        """loss_val as a 0-dim loss whose backward() puts the engine's current gradients of the (tag, module) pairs `mods`
        on those modules' parameters"""
        tg = self._torch_tensors(grads=True)
        named = [(tag, k, p) for tag, mod in mods for k, p in mod.named_parameters()]
        params = [p for _, _, p in named]
        flat = torch.cat([tg["%s.%s" % (tag, k)].detach().reshape(-1).to(p.device) for tag, k, p in named])
        self._dirty = True                                            # the caller's optimizer will change the module parameters
        return GradHandoff.apply(flat.detach().requires_grad_(True), loss_val.detach().to(flat.device), flat_pairs(params, flat))


class DCGANTrainer(EngineSync):
    """ Object to hold data iterators, train a GAN variant (surface of src/ns_gan.py:77-290) """
    variant = "ns"

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.Glosses, self.Dlosses = [], []
        self.viz = viz
        self.num_epochs = 0
        self._engine = None
        self._dirty = True               # module parameters newer than the engine's
        self._step = 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        object.__setattr__(model.G, "_owner", self)
        object.__setattr__(model.D, "_owner", self)

    # ------------------------------------------------------------------ engine <-> module parameters
    def _nets(self):
        """(state_dict prefix, module) of every network the engine trains"""
        return [("G", self.model.G), ("D", self.model.D)]

    def _engine_synced(self):
        m = self.model
        if self._engine is None:
            self._engine = DcganEngine(m.hidden_dim, m.z_dim, m.channels, variant=self.variant, d_out_act=m.D.out_act,
                                       embed_dim=getattr(m.D, "embed_dim", None), disc_dim=getattr(m, "disc_dim", None),
                                       cont_dim=getattr(m, "cont_dim", None))
            self._dirty = True
        if self._dirty:
            self._engine.load_torch_weights(self._sd())
            self._dirty = False
        return self._engine

    # ------------------------------------------------------------------ reference surface
    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1):
        """ Trainer.train (src/ns_gan.py:94-170): same loop and logging on the fused conv step, or on the overriding
        train_D / train_G (_train_custom) """
        import torch.distributed as dist
        if self._has_custom_step():
            return self._train_custom(num_epochs, G_lr, D_lr, D_steps)
        eng = self._engine_synced()
        hpG, hpD = AdamHP.make(G_lr), AdamHP.make(D_lr, clamp=self._d_clamp())
        for net in (eng.G, eng.D):                                  # fresh optimizers per train() call (src/ns_gan.py:107-110)
            net.exp_avg.zero_(); net.exp_avg_sq.zero_(); net.step = 0
        world, rank = par.world_size(), par.rank_of()
        if world > 1:                                               # replicas start from rank 0's parameters
            for net in (eng.G, eng.D):
                dist.broadcast(net.params, src=0)
                net.refresh()
        # batch statistics (RaNS / Fisher loss moments, DRAGAN's image std) run over the global batch: NCCL SUM between passes
        eng.stats_reduce = par.sum_gradients if world > 1 else None
        self._pre_train(eng)
        seed = par.rank_seed(self._seed, rank)
        pool = self._device_pool()
        epoch_steps = int(np.ceil(len(self.train_iter) / D_steps))
        for epoch in range(1, num_epochs + 1):
            self.model.train()
            ring = torch.zeros(D_steps + 1, epoch_steps, device="cuda")
            for i in range(epoch_steps):
                for k in range(D_steps):
                    if pool is not None:                            # the first batch of a freshly shuffled loader, on the device
                        n = min(pool.batch_size, pool.n)
                        rows = eng.stage_pool(pool, n, seed ^ DevicePool.SEED_MIX, self._step * D_steps + k)
                    else:
                        images = self.process_batch(self.train_iter)
                        n = images.shape[0]
                        rows = eng.stage_images(images)
                    inv = par.inv_global_batch(n, world)
                    ring[k, i] = eng.d_grad(rows, n, inv_global_batch=inv, seed=seed, step=self._step * D_steps + k, stat_batch=n * world)
                    par.sum_gradients(eng.D.grads)                  # NCCL SUM of the flat D gradient (no-op on one GPU)
                    eng.apply(1, hpD)
                ring[D_steps, i] = eng.g_grad(n, inv_global_batch=inv, seed=seed, step=self._step)
                par.sum_gradients(eng.G.grads)
                eng.apply(0, hpG)
                self._after_g_step(eng, n, inv, seed)
                self._step += 1
            G_losses, D_losses = ring[D_steps].tolist(), ring[:D_steps].mean(dim=0).tolist()
            self.Glosses.extend(G_losses)
            self.Dlosses.extend(D_losses)
            print(self._epoch_line(eng, epoch, num_epochs, G_losses, D_losses))
            self.num_epochs += 1
        self._pull()

    # a trainer whose losses need more than one score per image from D (BEGAN's autoencoder) or more than G and D (InfoGAN's
    # coded input and Q) names what is missing here: an override of its steps is refused, not silently ignored
    _custom_step_limit = None

    def _has_custom_step(self):
        """True when a subclass overrides train_D / train_G (/ train_Q) with a method not marked @builtin_step"""
        steps = [getattr(type(self), m) for m in ("train_D", "train_G", "train_Q") if hasattr(type(self), m)]
        return not all(getattr(f, "_gm_builtin", False) for f in steps)

    def _train_custom(self, num_epochs, G_lr, D_lr, D_steps):
        """The reference loop over the overriding train_D / train_G: their torch losses run model.G / model.D as autograd
        nodes over the conv kernels; Adam (FusedAdam) steps the module parameters, which the next forward loads"""
        if self._custom_step_limit is not None:
            raise GmError("%s: an overridden train_D / train_G is not supported: %s" % (type(self).__name__, self._custom_step_limit))
        if par.world_size() > 1:
            raise GmError("an overridden train_D / train_G trains on one process; data-parallel training runs the built-in steps")
        eng = self._engine_synced()
        self.model.to(eng.device)                   # the reference's to_cuda(model) (src/ns_gan.py:81): Adam runs on the device

        def after_step():
            self._dirty = True                      # the module parameters are newer than the engine's
        G_optimizer = FusedAdam(self.model.G.parameters(), lr=G_lr)
        D_optimizer = FusedAdam(self.model.D.parameters(), lr=D_lr, clamp=self._d_clamp())
        reference_loop(self, num_epochs, G_optimizer, D_optimizer, D_steps, after_step)
        pull_running_stats(eng, self._nets())

    def _epoch_line(self, eng, epoch, num_epochs, G_losses, D_losses):
        return "Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f" % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses))

    def _after_g_step(self, eng, n, inv, seed):
        """per-step device work of a subclass after each G update (e.g. BEGAN's K control, InfoGAN's MI step) for the step's
        local batch n, gradient scale inv and Philox seed; enqueued, never synchronising"""

    def _pre_train(self, eng):
        """per-train() state of a subclass (e.g. Fisher GAN's multiplier), after the optimizers are reset"""

    def _d_clamp(self):
        """the bound c of the clamp to [-c, c] that every D Adam step of train() applies to all D parameters (WGAN's weight
        clipping, src/w_gan.py:158,241-243); 0 = none"""
        return 0.0

    def _loss(self, net, loss_val):
        return self._fused_loss([("G", self.model.G)] if net == 0 else [("D", self.model.D)], loss_val)

    @builtin_step
    def train_D(self, images):
        """ Run 1 step of training for discriminator (src/ns_gan.py:172-194): returns D_loss; .backward() delivers the gradients """
        images = to_cuda(images)
        eng = self._engine_synced()
        n = images.shape[0]
        noise = self.compute_noise(n, self.model.z_dim)
        loss = eng.d_grad(eng.stage_images(images.reshape(n, -1).float()), n, noise=noise.float().contiguous())
        return self._loss(1, loss.clone())

    @builtin_step
    def train_G(self, images):
        """ Run 1 step of training for generator (src/ns_gan.py:196-216) """
        eng = self._engine_synced()
        n = images.shape[0]
        noise = self.compute_noise(n, self.model.z_dim)
        loss = eng.g_grad(n, noise=noise.float().contiguous())
        return self._loss(0, loss.clone())

    def compute_noise(self, batch_size, z_dim):
        """ Compute random noise for the generator to learn to make images from (src/ns_gan.py:218-220) """
        return to_cuda(torch.randn(batch_size, z_dim))

    def process_batch(self, iterator):
        """ Generate a process batch to be input into the discriminator D (src/ns_gan.py:222-226) """
        images, _ = next(iter(iterator))
        return to_cuda(images.view(images.shape[0], -1)).float().contiguous()

    def generate_images(self, epoch, num_outputs=36, save=True):
        """ Sample a grid from G (src/ns_gan.py:228-262 without the plotting) """
        self.model.eval()
        noise = self.compute_noise(num_outputs, self.model.z_dim)
        images = self.model.G(noise)
        return images.view(num_outputs, self.model.channels, 64, 64)

    def viz_loss(self):
        print("viz_loss: matplotlib is not installed")

    def save_model(self, savepath):
        """ Save model state dictionary (src/ns_gan.py:283-285) """
        if not self._dirty:
            self._pull()
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        """ Load state dictionary into model (src/ns_gan.py:287-290) """
        self.model.load_state_dict(torch.load(loadpath))
        self._dirty = True


if __name__ == "__main__":
    imgs = (torch.rand(8192, 3, 64, 64) < 0.3).float()
    loader = torch.utils.data.DataLoader(torch.utils.data.TensorDataset(imgs, torch.zeros(8192)), batch_size=256, shuffle=True)
    model = DCGAN(image_size=64 * 64 * 3, hidden_dim=64, z_dim=100)
    trainer = DCGANTrainer(model=model, train_iter=loader, val_iter=loader, test_iter=loader, viz=False)
    trainer.train(num_epochs=1, G_lr=2e-4, D_lr=2e-4, D_steps=1)
