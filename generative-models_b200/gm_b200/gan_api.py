"""Host-side mirror of the reference's GAN class surface (src/ns_gan.py:35-290 and its
per-variant copies), backed by the CUDA train-step engine.

What a reference user sees is unchanged: `Generator`, `Discriminator`, an `XGAN`
container with `.G .D .z_dim .image_size .hidden_dim .shape`, and an `XTrainer` with
`train / train_D / train_G / compute_noise / process_batch / generate_images /
viz_loss / save_model / load_model` and the `Glosses / Dlosses / num_epochs / name`
attributes.  What changes is where the arithmetic runs: the nn.Linear parameters
become views into the engine's flat fp32 buffers and every forward / loss / backward /
Adam is a hand-written sm_90a kernel behind the C ABI.  No autograd on the hot path.
"""
import os
import weakref
from copy import deepcopy

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib
from . import parallel as par
from ._lib import AdamHP, GmError
from .engine import GanEngine

G_NET, D_NET = 0, 1


def to_cuda(x):
    """src/utils.py:10-14."""
    if torch.cuda.is_available():
        x = x.cuda()
    return x


def to_var(x):
    """src/utils.py:6-8."""
    return to_cuda(x).requires_grad_()


class _EngineBacked(nn.Module):
    """nn.Module whose Linear parameters alias an engine's flat fp32 buffer once a
    Trainer has attached it; forward runs the CUDA kernels (inference, no autograd)."""
    _engine = None
    _net = None
    _owner = None      # weakref to the Trainer that creates / grows the engine on demand

    def _attach(self, engine, net):
        object.__setattr__(self, "_engine", engine)
        object.__setattr__(self, "_net", net)

    def _engine_for(self, batch, what):
        """The engine able to hold `batch` rows; the owning Trainer creates or grows it lazily
        (the reference moves the model to the GPU in Trainer.__init__, src/ns_gan.py:81)."""
        owner = self._owner() if self._owner is not None else None
        if owner is not None and (self._engine is None or batch > (owner._max_batch or 0)):
            owner._ensure_engine(batch)
        if self._engine is None:
            raise GmError(what + " is not attached to a CUDA engine yet: construct the Trainer first "
                          "(there is no eager/CPU path)")
        self._engine.sync_if_stale()
        return self._engine


class Generator(_EngineBacked):
    """Generator. Input is noise, output is a generated image (src/ns_gan.py:35-46)."""

    def __init__(self, image_size, hidden_dim, z_dim):
        super().__init__()
        self.linear = nn.Linear(z_dim, hidden_dim)
        self.generate = nn.Linear(hidden_dim, image_size)

    def forward(self, x):
        x = to_cuda(x).float().contiguous()
        eng = self._engine_for(x.shape[0], "Generator")
        if torch.is_grad_enabled() and eng.supports_custom_loss:
            return _GForward.apply(x, eng, *self.parameters())     # custom-loss path (README.md:31)
        return eng.generate(x)


class Discriminator(_EngineBacked):
    """Discriminator. Input is an image, output is D's score (src/ns_gan.py:49-60)."""

    def __init__(self, image_size, hidden_dim, output_dim):
        super().__init__()
        if output_dim != 1:
            raise GmError("only output_dim=1 discriminators are built (as in every reference model)")
        self.linear = nn.Linear(image_size, hidden_dim)
        self.discriminate = nn.Linear(hidden_dim, output_dim)

    def forward(self, x):
        x = to_cuda(x).float().contiguous()
        eng = self._engine_for(x.shape[0], "Discriminator")
        if torch.is_grad_enabled() and eng.supports_custom_loss:
            return _DForward.apply(x, eng, *self.parameters())     # custom-loss path (README.md:31)
        return eng.discriminate(x)


class GANBase(nn.Module):
    """Container for G and D (src/ns_gan.py:63-74): keeps the hyper-parameters as
    attributes the way `self.__dict__.update(locals())` does in the reference."""

    def __init__(self, image_size, hidden_dim, z_dim, output_dim=1):
        super().__init__()
        self.__dict__.update(dict(image_size=image_size, hidden_dim=hidden_dim, z_dim=z_dim, output_dim=output_dim))
        self.G = Generator(image_size, hidden_dim, z_dim)
        self.D = Discriminator(image_size, hidden_dim, output_dim)
        self.shape = int(image_size ** 0.5)


class DeviceDataset:
    """Device-resident, bit-packed copy of a binarised image dataset + on-device batch sampling.

    The reference fetches every batch with `next(iter(DataLoader(shuffle=True)))`
    (src/ns_gan.py:222-226): a fresh random permutation of the whole dataset and a host
    `stack` + H2D copy per step — 27-34 % of its CPU step (SURVEY.md 2.2).  When the
    Trainer is handed a DataLoader over a TensorDataset of {0,1} images, the images are
    packed once to 1 bit/pixel (98 B/image) in HBM; a batch is then `batch_size` distinct
    random row indices drawn on the device and gathered + unpacked by the staging kernel."""

    def __init__(self, images, batch_size, drop_last=False):
        n = images.shape[0]
        flat = images.reshape(n, -1)
        self.n, self.x, self.batch_size = n, flat.shape[1], batch_size
        if self.x % 8:
            raise ValueError("image_size must be a multiple of 8")
        self.bits = self._pack(flat)            # [n, x/8] uint8 on the device, MSB first (np.packbits order)
        self.num_batches = n // batch_size if drop_last else -(-n // batch_size)
        self._gen = None
        self._source = images

    @staticmethod
    def _pack(flat, chunk_rows=32768):
        """{0,1} images -> 1 bit/pixel, packed ON the device chunk by chunk (a 262144-image fp32 dataset
        packs in ~0.1 s instead of seconds of host numpy); raises ValueError for non-binary data."""
        n, x = flat.shape
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else flat.device
        w = torch.tensor([128, 64, 32, 16, 8, 4, 2, 1], dtype=torch.int32, device=dev)
        out = torch.empty(n, x // 8, dtype=torch.uint8, device=dev)
        for i in range(0, n, chunk_rows):
            c = flat[i:i + chunk_rows].to(dev, non_blocking=True)
            one = c == 1
            if not bool((one | (c == 0)).all()):
                raise ValueError("DeviceDataset needs binarised {0,1} images")
            out[i:i + chunk_rows] = (one.view(-1, x // 8, 8).to(torch.int32) * w).sum(dim=2).to(torch.uint8)
        return out

    def seed(self, value):
        """Own device generator (data-parallel ranks must draw different batches)."""
        self._gen = torch.Generator(device=self.bits.device).manual_seed(int(value) & 0x7FFFFFFFFFFFFFFF)

    def __len__(self):
        return self.num_batches

    def sample(self):
        """indices of one shuffled batch (what the first batch of a fresh shuffling iterator holds)"""
        b = min(self.batch_size, self.n)
        return torch.randperm(self.n, device=self.bits.device, generator=self._gen)[:b].to(torch.int32)

    @staticmethod
    def from_loader(loader, cached=None):
        """`cached`: the DeviceDataset of an earlier train() call - reused when the loader still serves the
        same image tensor with the same batching (packing runs once per dataset, not once per train())."""
        ds = getattr(loader, "dataset", None)
        tensors = getattr(ds, "tensors", None)
        if tensors is None or getattr(loader, "batch_size", None) is None:
            return None
        drop = getattr(loader, "drop_last", False)
        if cached is not None and cached._source is tensors[0] and cached.batch_size == loader.batch_size and \
                cached.num_batches == (tensors[0].shape[0] // loader.batch_size if drop else -(-tensors[0].shape[0] // loader.batch_size)):
            return cached
        try:
            return DeviceDataset(tensors[0], loader.batch_size, drop)
        except ValueError:
            return None


def builtin_step(fn):
    """Marks a train_D / train_G implementation as one of the fused built-in losses.  A
    Trainer whose train_D / train_G is NOT marked (a user override, README.md:31) is trained
    by the reference loop over the custom-loss path instead of the fused step."""
    fn._gm_builtin = True
    return fn


def first_order(backward):
    """a create_graph=True backward through a CUDA node raises here, before the kernels run, instead of returning
    gradients that a second differentiation would see as constants"""
    def wrapper(ctx, *grads):
        if torch.is_grad_enabled():
            raise RuntimeError("the CUDA forward / backward nodes have no double backward (create_graph=True)")
        return backward(ctx, *grads)
    return wrapper


def _split_like(flat, params):
    out, off = [], 0
    for p in params:
        n = p.numel()
        out.append(flat[off:off + n].view_as(p).clone())
        off += n
    return out


class _GForward(torch.autograd.Function):
    """Generator.forward with a backward (src/ns_gan.py:43-46): both halves are the CUDA
    kernels; autograd only routes dL/dG(z) in and the parameter gradients out."""

    @staticmethod
    def forward(ctx, noise, engine, *params):
        ctx.engine, ctx.params = engine, params
        engine.g_generation += 1
        ctx.generation = engine.g_generation
        return engine.g_forward(noise)

    @staticmethod
    @once_differentiable        # the backward is a CUDA kernel chain: a create_graph=True caller gets an error, not a silently missing term
    def backward(ctx, dimages):
        eng = ctx.engine
        if eng.g_generation != ctx.generation:
            raise RuntimeError("Generator activations were overwritten by a later Generator.forward: "
                               "back-propagate a G output before calling G again")
        if getattr(ctx, "consumed", False):
            # gm_gan_g_backward turns the saved output into its upstream in place: a second pass would read that instead
            raise RuntimeError("Generator activations were consumed by this call's first backward: a G output can be "
                               "back-propagated once (retain_graph=True does not keep them)")
        ctx.consumed = True
        flat = eng.g_backward(dimages.float().contiguous())
        return (None, None, *_split_like(flat, ctx.params))


class _DForward(torch.autograd.Function):
    """Discriminator.forward with a backward (src/ns_gan.py:57-60).  Each call keeps its
    activations in one of the engine's row regions until its backward ran."""

    @staticmethod
    def forward(ctx, x, engine, *params):
        ctx.engine, ctx.params = engine, params
        ctx.slot = engine.d_calls % engine.num_slots()
        engine.d_calls += 1
        engine.d_generation[ctx.slot] = engine.d_calls
        ctx.generation = engine.d_calls
        return engine.d_forward(ctx.slot, x).view(-1, 1)

    @staticmethod
    @once_differentiable
    def backward(ctx, dscore):
        eng = ctx.engine
        if eng.d_generation[ctx.slot] != ctx.generation:
            raise RuntimeError("Discriminator activations were overwritten: at most %d Discriminator.forward "
                               "results can await their backward (construct the engine with a gradient-penalty "
                               "variant for more)" % eng.num_slots())
        flat, dx = eng.d_backward(ctx.slot, dscore.reshape(-1).float().contiguous(), ctx.needs_input_grad[0])
        return (dx, None, *_split_like(flat, ctx.params))


class FusedAdam(torch.optim.Optimizer):
    """torch.optim.Adam semantics (src/ns_gan.py:107-110) with the update done by
    gm_adam_step; used by the reference loop when train_D / train_G are user overrides."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, clamp=0.0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, clamp=clamp))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            hp = AdamHP.make(group["lr"], group["betas"], group["eps"], group["weight_decay"], group["clamp"])
            for p in group["params"]:
                if p.grad is None:
                    continue
                st = self.state[p]
                if not st:
                    st["step"], st["exp_avg"], st["exp_avg_sq"] = 0, torch.zeros_like(p.data), torch.zeros_like(p.data)
                st["step"] += 1
                _lib.adam_step(p.data, p.grad.contiguous(), st["exp_avg"], st["exp_avg_sq"], hp, st["step"])


def reference_loop(tr, num_epochs, G_optimizer, D_optimizer, D_steps, after_step=None):
    """The reference's loop verbatim (src/ns_gan.py:107-156) for a Trainer tr whose train_D / train_G were overridden: the
    override's torch loss drives the CUDA forward / backward kernels through model.G / model.D and their autograd nodes.
    after_step(), when given, runs after every optimizer step (the conv trainers mark their modules' parameters as newer
    than their engine's)."""
    epoch_steps = int(np.ceil(len(tr.train_iter) / D_steps))
    for epoch in range(1, num_epochs + 1):
        tr.model.train()
        G_losses, D_losses = [], []
        for _ in range(epoch_steps):
            D_step_loss = []
            for _ in range(D_steps):
                images = tr.process_batch(tr.train_iter)
                D_optimizer.zero_grad()
                D_loss = tr.train_D(images)
                D_loss.backward()
                D_optimizer.step()
                if after_step is not None:
                    after_step()
                D_step_loss.append(D_loss.detach())
            D_losses.append(torch.stack(D_step_loss).mean())
            G_optimizer.zero_grad()
            G_loss = tr.train_G(images)
            G_losses.append(G_loss.detach())
            G_loss.backward()
            G_optimizer.step()
            if after_step is not None:
                after_step()
        G_losses, D_losses = torch.stack(G_losses).tolist(), torch.stack(D_losses).tolist()
        tr.Glosses.extend(G_losses)
        tr.Dlosses.extend(D_losses)
        print("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f" % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses)))
        tr.num_epochs += 1
        if tr.viz:
            tr.generate_images(epoch)


def has_custom_compute_batch(tr):
    """True when tr's class overrides compute_batch (README.md:31) with a method not marked @builtin_step"""
    return not getattr(type(tr).compute_batch, "_gm_builtin", False)


def refuse_multi_rank():
    """an overridden compute_batch trains on one process: refused under a process group of more than one rank"""
    from . import parallel as par
    if par.world_size() > 1:
        raise GmError("an overridden compute_batch trains on one process; data-parallel training runs the built-in step")


def compute_batch_loop(tr, num_epochs, lr, weight_decay, two_losses, after_step=None):
    """The reference's train loop verbatim (src/vae.py:127-191 when compute_batch returns (recon, kl), src/ae.py:84-145 when
    it returns one loss) for a VAE-family trainer tr whose compute_batch was overridden: the override's torch loss drives the
    CUDA forward / backward kernels through the model's encoder / decoder autograd nodes, FusedAdam (coupled weight decay,
    as torch.optim.Adam) steps the module parameters, validation runs tr.evaluate (which calls the override) in eval mode.
    train_iter is read on the host.  after_step(), when given, runs after every optimizer step.  best_model is
    deepcopy(tr.model), a detached copy with its own inference engine."""
    optimizer = FusedAdam([p for p in tr.model.parameters() if p.requires_grad], lr=lr, weight_decay=weight_decay)
    for epoch in range(1, num_epochs + 1):
        tr.model.train()
        epoch_loss, epoch_recon, epoch_kl = [], [], []
        for batch in tr.train_iter:
            optimizer.zero_grad()
            if two_losses:
                recon_loss, kl_diverge = tr.compute_batch(batch)
                batch_loss = recon_loss + kl_diverge
            else:
                batch_loss = tr.compute_batch(batch)
            batch_loss.backward()
            optimizer.step()
            if after_step is not None:
                after_step()
            epoch_loss.append(batch_loss.item())
            if two_losses:
                epoch_recon.append(recon_loss.item())
                epoch_kl.append(kl_diverge.item())
        if two_losses:
            tr.kl_loss.extend(epoch_kl)
            tr.recon_loss.extend(epoch_recon)
        else:
            tr.recon_loss.extend(epoch_loss)
        tr.model.eval()
        val_loss = tr.evaluate(tr.val_iter)
        if val_loss < tr.best_val_loss:
            tr.best_model = deepcopy(tr.model)
            tr.best_val_loss = val_loss
        if two_losses:
            print("Epoch[%d/%d], Total Loss: %.4f, Reconst Loss: %.4f, KL Div: %.7f, Val Loss: %.4f"
                  % (epoch, num_epochs, np.mean(epoch_loss), np.mean(epoch_recon), np.mean(epoch_kl), val_loss))
        else:
            print("Epoch[%d/%d], Train Loss: %.4f, Val Loss: %.4f" % (epoch, num_epochs, np.mean(epoch_loss), val_loss))
        tr.num_epochs += 1
        if tr.viz:
            if two_losses:
                tr.sample_images(epoch)
            else:
                tr.reconstruct_images(tr.debugging_image, epoch)


def compute_batch_evaluate(tr, iterator, two_losses):
    """evaluate (src/vae.py:214-223, src/ae.py:162-164) over the overridden compute_batch: the mean per-batch loss"""
    loss = []
    for batch in iterator:
        out = tr.compute_batch(batch)
        loss.append((out[0] + out[1]).item() if two_losses else out.item())
    return float(np.mean(loss))


class SlotRing:
    """The per-call slots of one engine's encoder or decoder: take() hands them out round robin, numbering the calls; a
    backward whose slot a later call took, or whose engine was replaced (retire(): a larger batch), raises"""

    def __init__(self, n, what):
        self.n, self.what, self.calls, self.gen, self.retired = n, what, 0, [0] * n, False

    def take(self):
        self.calls += 1
        slot = (self.calls - 1) % self.n
        self.gen[slot] = self.calls
        return slot, self.calls

    def check(self, slot, gen):
        if self.retired:
            raise RuntimeError("%s activations were overwritten: the engine was rebuilt for a larger batch since this call"
                               % self.what)
        if self.gen[slot] != gen:
            raise RuntimeError("%s activations were overwritten: at most %d %s.forward results can await their backward"
                               % (self.what, self.n, self.what))

    def retire(self):
        self.retired = True


class _FusedLoss(torch.autograd.Function):
    """0-dim loss whose backward() hands the gradients the fused kernels already
    computed to the parameters' .grad (the reference calls loss.backward() then
    optimizer.step(), src/ns_gan.py:138-139)."""

    @staticmethod
    def forward(ctx, flat_params, loss_val, flat_grad, param_list):
        ctx.flat_grad, ctx.param_list = flat_grad, param_list
        return loss_val.clone()

    @staticmethod
    def backward(ctx, gout):
        off = 0
        for p in ctx.param_list:
            n = p.numel()
            g = ctx.flat_grad[off:off + n].view_as(p) * gout
            p.grad = g if p.grad is None else p.grad + g
            off += n
        return None, None, None, None


class _StepGraph:
    """One captured outer train step of a GANTrainerBase (see GANTrainerBase.cuda_graph)."""

    def __init__(self, trainer, eng):
        self.tr, self.eng, self.ready, self.graph = trainer, eng, False, None
        self.scratch = None

    @staticmethod
    def begin(tr):
        res = getattr(tr, "_resident", None)
        if not (tr.cuda_graph and res is not None and getattr(tr, "_world", 1) == 1 and tr._use_device_noise()):
            return None
        batch = min(res.batch_size, res.n)
        if batch > tr.cuda_graph_max_batch or type(tr)._fused_D is not GANTrainerBase._fused_D or type(tr)._fused_G is not GANTrainerBase._fused_G:
            return None
        eng = tr._ensure_engine(batch)
        eng._g_calls, eng._d_calls = tr._step, tr._dcount
        eng.use_device_step(True)              # Adam steps / Philox streams / sampler rounds now come from device counters
        return _StepGraph(tr, eng)

    def capture(self, D_steps, batch, hpD, hpG):
        tr, eng = self.tr, self.eng
        if tr._engine is not eng:              # the engine was re-created (grown) under us: stay eager
            return
        self.scratch = torch.zeros(D_steps + 1, device="cuda")
        torch.cuda.synchronize()
        try:
            g = torch.cuda.CUDAGraph()
            d0, s0 = tr._dcount, tr._step
            with torch.cuda.graph(g):
                for k in range(D_steps):
                    tr._fused_D(tr._resident.bits, hpD, batch=batch, loss_out=self.scratch[k])
                tr._fused_G(batch, hpG, loss_out=self.scratch[D_steps])
            tr._dcount, tr._step = d0, s0      # capturing executes nothing
            self.graph, self.ready, self.D_steps = g, True, D_steps
        except RuntimeError as exc:            # pragma: no cover  (capture not possible here: keep launching eagerly)
            print("[gm_b200] CUDA-graph capture of the train step failed (%s); continuing with eager launches" % str(exc)[:120])
            self.graph, self.ready = None, False

    def replay(self, ring_col):
        self.graph.replay()
        ring_col.copy_(self.scratch)
        self.tr._dcount += self.D_steps
        self.tr._step += 1

    def end(self):
        try:
            torch.cuda.synchronize()
            self.eng.use_device_step(False)
        except GmError:                        # pragma: no cover
            pass


class GANTrainerBase:
    """Object to hold data iterators, train a GAN variant (src/ns_gan.py:77-290)."""
    variant = "ns"
    d_out_act = "sigmoid"
    device_dataset = True     # keep a bit-packed copy of train_iter's dataset in HBM when possible

    def __init__(self, model, train_iter, val_iter, test_iter, viz=False):
        self.model = model
        self.name = model.__class__.__name__
        self.train_iter, self.val_iter, self.test_iter = train_iter, val_iter, test_iter
        self.Glosses, self.Dlosses = [], []
        self.viz = viz
        self.num_epochs = 0
        self._engine = None
        self._max_batch = None
        self._step = 0          # G updates so far / D updates so far: the Philox streams of train_G / train_D
        self._dcount = 0
        self._seed = int(torch.initial_seed() & 0x7FFFFFFF)
        self._needs_sync = True
        for mod in (getattr(model, "G", None), getattr(model, "D", None)):
            if isinstance(mod, _EngineBacked):
                object.__setattr__(mod, "_owner", weakref.ref(self))

    # ------------------------------------------------------------------ engine plumbing
    def _ensure_engine(self, batch):
        """Create (or grow) the engine; the model's Linear parameters become views of the
        engine's flat fp32 buffers (this is the reference's to_cuda(model), src/ns_gan.py:81)."""
        if self._engine is not None and batch <= self._max_batch and self._engine.variant == self._variant_name():
            return self._engine
        m = self.model
        old = self._engine
        batch = max(batch, self._max_batch or 0)
        eng = GanEngine(m.image_size, m.hidden_dim, m.z_dim, max_batch=max(batch, 64), variant=self._variant_name(),
                        d_out_act=self.d_out_act)
        for net, mod in ((G_NET, m.G), (D_NET, m.D)):
            params = list(mod.parameters())
            eng.load(net, [p.data for p in params])
            for p, v in zip(params, eng.views(net)):
                p.data = v                      # alias: nn.Parameter storage == engine master weights
            mod._attach(eng, net)
        if old is not None:
            for net in (G_NET, D_NET):
                eng.exp_avg[net].copy_(old.exp_avg[net])
                eng.exp_avg_sq[net].copy_(old.exp_avg_sq[net])
            eng.steps = list(old.steps)
        self._engine, self._max_batch = eng, max(batch, 64)
        self._needs_sync = False
        self._after_engine_created(eng)
        return eng

    def _after_engine_created(self, eng):
        pass

    # loss constants the reference passes as train_D / train_G kwargs (LAMBDA, K, C; a, b, c): set the class / instance
    # attribute `loss_consts` (e.g. dict(gp_lambda=5.0)) for the fused train() loop, or pass them to train_D / train_G
    loss_consts = {}

    def _set_consts(self, eng, **kw):
        want = dict(self.loss_consts)
        want.update(kw)
        if getattr(eng, "loss_consts", None) != dict(dict(gp_lambda=10.0, gp_k=1.0, dra_c=1.0, ls_a=0.0, ls_b=1.0, ls_c=1.0), **want):
            eng.set_loss_consts(**dict(dict(gp_lambda=10.0, gp_k=1.0, dra_c=1.0, ls_a=0.0, ls_b=1.0, ls_c=1.0), **want))

    def _draw_aux(self, images):
        """Extra random tensors train_D draws after the noise (WGAN-GP eps, DRAGAN delta/u)."""
        return None

    def _variant_name(self):
        return self.variant

    def _loss_tensor(self, net, loss_val):
        eng = self._engine
        params = list((self.model.G if net == G_NET else self.model.D).parameters())
        return _FusedLoss.apply(eng.params[net].detach().requires_grad_(True), loss_val, eng.grads[net], params)

    # ------------------------------------------------------------------ reference surface
    def train(self, num_epochs, G_lr=2e-4, D_lr=2e-4, D_steps=1, **extra):
        """Trainer.train (src/ns_gan.py:94-170): same loop, same logging; each train_D /
        train_G + backward + Adam step is one fused kernel sequence and losses are read
        back once per epoch instead of once per step."""
        if self._has_custom_step():
            return self._train_reference_loop(num_epochs, G_lr, D_lr, D_steps, float(extra.get("clip", 0.0) or 0.0))
        hpG, hpD = AdamHP.make(G_lr), AdamHP.make(D_lr, clamp=float(extra.get("clip", 0.0) or 0.0))
        epoch_steps = int(np.ceil(len(self.train_iter) / D_steps))
        self._resident = DeviceDataset.from_loader(self.train_iter, getattr(self, "_resident", None)) if self.device_dataset else None
        self._dp_begin()
        graph = None
        try:
            self._pre_train(num_epochs, hpG, hpD, D_steps, extra)
            graph = _StepGraph.begin(self)
            for epoch in range(1, num_epochs + 1):
                self.model.train()
                # the kernels write each step's loss straight into this epoch's device log
                ring = torch.zeros(D_steps + 1, epoch_steps, device="cuda")
                done = 0
                try:
                    for i in range(epoch_steps):
                        if graph is not None and graph.ready:
                            graph.replay(ring[:, i])                # one launch from the host: the whole outer step
                            done = i + 1
                            continue
                        for k in range(D_steps):
                            if self._resident is not None:          # on-device shuffle + gather, no host work
                                batch = min(self._resident.batch_size, self._resident.n)
                                self._fused_D(self._resident.bits, hpD, batch=batch, loss_out=ring[k, i])
                            else:
                                images = self.process_batch(self.train_iter)
                                batch = images.shape[0]
                                self._fused_D(images, hpD, loss_out=ring[k, i])
                        self._fused_G(batch, hpG, loss_out=ring[D_steps, i])
                        done = i + 1
                        if graph is not None and not graph.ready:
                            graph.capture(D_steps, batch, hpD, hpG)   # the first outer step ran eagerly (plans, attributes)
                finally:
                    # an interrupted epoch (KeyboardInterrupt in a notebook) still logs the steps it ran;
                    # one device->host read per epoch
                    G_losses = ring[D_steps, :done].tolist()
                    D_losses = ring[:D_steps, :done].mean(dim=0).tolist()
                    self.Glosses.extend(G_losses)
                    self.Dlosses.extend(D_losses)
                print("Epoch[%d/%d], G Loss: %.4f, D Loss: %.4f" % (epoch, num_epochs, np.mean(G_losses), np.mean(D_losses)))
                self.num_epochs += 1
                if self.viz:
                    self.generate_images(epoch)
        finally:
            if graph is not None:
                graph.end()
            self._dp_end()

    # CUDA-graph replay of the outer step (D_steps D updates + 1 G update) for launch-bound batch sizes - the reference's own
    # regime, batch 64 / 100 (src/ns_gan.py:311-314, src/utils.py:16): with the resident dataset and in-kernel noise nothing
    # in a step depends on host data, the engine keeps its step counters on the device (gm_gan_use_device_step) and every
    # step after the first is ONE graph launch.  Bit-identical to eager launches (tests/test_dropin_gpu.py) but MEASURED
    # SLOWER on an H100 (700 W limit; B = 64 through this loop: 0.428 ms/step replayed vs 0.175 ms/step eager): the step is
    # a chain of ~22 dependent kernels whose prologues already overlap through programmatic dependent launch, and every
    # graph launch adds its own start / drain
    # gap.  Hence off by default; `trainer.cuda_graph = True` turns it on (a host-bound caller, e.g. a slow CPU, gains).
    cuda_graph = False
    cuda_graph_max_batch = 8192

    # ------------------------------------------------------------------ data-parallel / fast-path state of one train() call
    def _dp_begin(self):
        """Data parallel when launched under torchrun with an initialised process group (SURVEY.md 8e): per-rank
        batches and noise, upstream gradients scaled by 1/(global batch), SUM of the flat D / G gradients fused
        into the Adam kernel.  Replicas start from rank 0's parameters.  On one GPU the split-K gradient gather
        is fused into the Adam kernel instead ("lazy gradients")."""
        self._world, self._rank = par.world_size(), par.rank_of()
        self._comm = None
        self._noise_gen = None
        if self._world > 1:
            bs = getattr(self.train_iter, "batch_size", None) or 64
            eng = self._ensure_engine(bs)
            self._broadcast_parameters(eng)
            n = sum(p.numel() for p in self.model.G.parameters()), sum(p.numel() for p in self.model.D.parameters())
            self._comm = par.make_peer_comm(max(n))
            # host-side draws (compute_noise overrides, the DataLoader fallback) must differ per rank
            self._noise_gen = torch.Generator().manual_seed((int(torch.initial_seed()) + 7919 * (self._rank + 1)) & 0x7FFFFFFFFFFFFFFF)
        self._lazy = self._world == 1 or self._comm is not None
        self.gradient_exchange = "none" if self._world == 1 else ("peer" if self._comm is not None else "nccl")

    def _broadcast_parameters(self, eng):
        import torch.distributed as dist
        for net in (G_NET, D_NET):
            dist.broadcast(eng.params[net], src=0)
        eng.sync_all()

    def _dp_end(self):
        """Always runs (try/finally): leave the engine with materialised gradients and no dangling communicator."""
        try:
            if self._engine is not None and getattr(self, "_d_begun", None) is not None and self._comm is not None:
                self._finish_d_exchange(self._engine)
        except GmError:          # pragma: no cover
            self._d_begun = None
        self._lazy = False
        self._noise_gen = None
        eng = self._engine
        if eng is not None:
            try:
                eng.set_lazy_grads(False)
                if getattr(eng, "_comm_attached", None) is not None:
                    eng.attach_comm(None)
                    eng._comm_attached = None
            except GmError:      # pragma: no cover  (a CUDA error is already propagating)
                pass
        if self._comm is not None:          # the exchange buffers live for one train() call
            try:
                torch.cuda.synchronize()
                self._comm.close()
            finally:
                self._comm = None

    def _has_custom_step(self):
        return not (getattr(type(self).train_D, "_gm_builtin", False) and getattr(type(self).train_G, "_gm_builtin", False))

    def _train_reference_loop(self, num_epochs, G_lr, D_lr, D_steps, clip):
        """reference_loop for Trainers whose train_D / train_G were overridden"""
        bs = getattr(self.train_iter, "batch_size", None) or next(iter(self.train_iter))[0].shape[0]
        self._ensure_engine(bs)
        G_optimizer = FusedAdam(self.model.G.parameters(), lr=G_lr)
        D_optimizer = FusedAdam(self.model.D.parameters(), lr=D_lr, clamp=clip)
        reference_loop(self, num_epochs, G_optimizer, D_optimizer, D_steps)

    def _pre_train(self, num_epochs, hpG, hpD, D_steps, extra):
        # fresh optimizers each train() call, like src/ns_gan.py:107-110; parameters may have
        # been touched from outside since the last call -> refresh the operand copies once
        if self._engine is not None:
            self._engine.reset_optimizer()
        self._needs_sync = True

    def _sync_once(self, eng):
        if self._needs_sync:
            eng.sync_all()
            self._needs_sync = False

    # in-kernel Philox noise unless the user wants the reference's CPU stream (torch.manual_seed replay):
    # set `trainer.device_noise = False`, or override / replace compute_noise (always honoured)
    device_noise = True

    def _use_device_noise(self):
        if not self.device_noise:
            return False
        return getattr(self.compute_noise, "__func__", None) is GANTrainerBase.compute_noise and \
            getattr(self._draw_aux, "__func__", None) in (GANTrainerBase._draw_aux, type(self)._draw_aux)

    def _philox_seed(self):
        return par.rank_seed(self._seed, getattr(self, "_rank", 0))

    def _fused_D(self, images, hp, gather_idx=None, batch=None, loss_out=None):
        """One D update.  `images`: a [B, x] batch, or (with `batch`) the resident bit-packed pool the engine
        samples from on the device, or (with gather_idx) pool + explicit row indices."""
        pool = batch is not None and gather_idx is None
        if batch is None:
            batch = images.shape[0] if gather_idx is None else gather_idx.shape[0]
        eng = self._ensure_engine(batch)
        self._finish_d_exchange(eng)             # a D exchange begun by the previous D sub-step (D_steps > 1)
        self._sync_once(eng)
        self._set_consts(eng)
        world = getattr(self, "_world", 1)
        eng.set_lazy_grads(getattr(self, "_lazy", False))
        if getattr(self, "_comm", None) is not None and getattr(eng, "_comm_attached", None) is not self._comm:
            eng.attach_comm(self._comm)          # batch statistics over the global batch
            eng._comm_attached = self._comm
        inv = par.inv_global_batch(batch, world)
        dev = self._use_device_noise()
        noise = None if dev else self.compute_noise(batch, self.model.z_dim)
        kw = dict(noise=noise, inv_global_batch=inv, seed=self._philox_seed(), step=self._dcount, loss_out=loss_out)
        if pool or gather_idx is not None:
            if pool:
                eng.set_sampler(self._resident.n, self._philox_seed() ^ 0x5DEECE66D)
            aux = None if dev else self._draw_aux(torch.empty(batch, self.model.image_size, device="meta"))
            loss = eng.d_grad(images, fmt="bits", gather_idx=gather_idx, batch=batch, aux=aux, **kw)
        else:
            eng.set_sampler(0)
            loss = eng.d_grad(images, aux=None if dev else self._draw_aux(images), **kw)
        if loss_out is None:
            loss = loss.clone()
        self._dcount += 1
        comm = getattr(self, "_comm", None)
        if comm is not None and self.split_exchange:
            # publish the D gradient now; the wait + sum + Adam half runs after the G step's generator forward (_fused_G),
            # which does not depend on the D update and absorbs the NVLink latency and the ranks' arrival skew
            eng.exchange_begin(D_NET, comm)
            self._d_begun = hp
        else:
            self._dp_apply(eng, D_NET, hp)
        return loss

    def _fused_G(self, batch, hp, loss_out=None):
        eng = self._ensure_engine(batch)
        self._sync_once(eng)
        self._set_consts(eng)
        noise = None if self._use_device_noise() else self.compute_noise(batch, self.model.z_dim)
        world = getattr(self, "_world", 1)
        if getattr(self, "_d_begun", None) is not None:
            eng.g_forward_stage(batch, noise=noise, seed=self._philox_seed(), step=self._step)     # independent of the D update
            self._finish_d_exchange(eng)
            loss = eng.g_grad_staged(batch, inv_global_batch=par.inv_global_batch(batch, world), loss_out=loss_out)
        else:
            loss = eng.g_grad(batch, noise=noise, inv_global_batch=par.inv_global_batch(batch, world), seed=self._philox_seed(),
                              step=self._step, loss_out=loss_out)
        if loss_out is None:
            loss = loss.clone()
        self._dp_apply(eng, G_NET, hp)
        self._step += 1
        return loss

    # two-phase gradient exchange (gm_gan_exchange_begin ... gm_gan_apply_allreduce with the G forward in between) under data
    # parallelism: bitwise the same replicas; kept off by default (the fused kernel has fewer launches and sync points)
    split_exchange = False

    def _finish_d_exchange(self, eng):
        hp = getattr(self, "_d_begun", None)
        if hp is not None:
            self._d_begun = None
            eng.apply_allreduce(D_NET, hp, self._comm)

    def _dp_apply(self, eng, net, hp):
        """optimizer.step(); under data parallelism preceded by the SUM of the flat gradient - fused into
        the Adam kernel over peer mappings when available, else NCCL all-reduce."""
        comm = getattr(self, "_comm", None)
        if comm is not None:
            eng.apply_allreduce(net, hp, comm)
            return
        if getattr(self, "_world", 1) > 1:
            par.sum_gradients(eng.grads[net])
        eng.apply(net, hp)

    @builtin_step
    def train_D(self, images, **consts):
        """Run 1 step of training for the discriminator (src/ns_gan.py:172-194): returns
        the loss; `.backward()` delivers the D gradients to model.D's parameters."""
        images = to_cuda(images)
        eng = self._ensure_engine(images.shape[0])
        eng.sync_if_stale()
        self._set_consts(eng, **consts)
        eng.set_lazy_grads(False)       # .backward() reads the flat gradient: it must be formed by d_grad itself
        eng.set_sampler(0)
        noise = self.compute_noise(images.shape[0], self.model.z_dim)
        loss = eng.d_grad(images.float().contiguous(), noise=noise.float().contiguous(), aux=self._draw_aux(images),
                          seed=self._seed, step=self._step)
        return self._loss_tensor(D_NET, loss)

    @builtin_step
    def train_G(self, images, **consts):
        """Run 1 step of training for the generator (src/ns_gan.py:196-216)."""
        batch = images.shape[0]
        eng = self._ensure_engine(batch)
        eng.sync_if_stale()
        self._set_consts(eng, **consts)
        eng.set_lazy_grads(False)
        noise = self.compute_noise(batch, self.model.z_dim)
        loss = eng.g_grad(batch, noise=noise.float().contiguous(), seed=self._seed, step=self._step)
        self._step += 1
        return self._loss_tensor(G_NET, loss)

    def compute_noise(self, batch_size, z_dim):
        """Compute random noise for the generator (src/ns_gan.py:218-220): CPU RNG then
        H2D, so a torch.manual_seed run draws the same numbers as the reference."""
        return to_cuda(torch.randn(batch_size, z_dim, generator=getattr(self, "_noise_gen", None)))

    def process_batch(self, iterator):
        """Generate a processed batch for D (src/ns_gan.py:222-226)."""
        images, _ = next(iter(iterator))
        images = to_cuda(images.view(images.shape[0], -1)).float().contiguous()
        return images

    def generate_images(self, epoch, num_outputs=36, save=True):
        """Sample a grid from G (src/ns_gan.py:228-262); saving needs torchvision, plotting
        needs matplotlib — both optional here."""
        self.model.eval()
        noise = self.compute_noise(num_outputs, self.model.z_dim)
        images = self.model.G(noise)
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
        """Loss curves (src/ns_gan.py:264-281); needs matplotlib."""
        try:
            import matplotlib.pyplot as plt
        except ImportError:
            print("viz_loss: matplotlib is not installed")
            return
        plt.plot(np.linspace(1, self.num_epochs, len(self.Dlosses)), self.Dlosses, "r")
        plt.plot(np.linspace(1, self.num_epochs, len(self.Dlosses)), self.Glosses, "g")
        plt.legend(["Discriminator", "Generator"])
        plt.title(self.name)
        plt.show()

    def save_model(self, savepath):
        """Save model state dictionary (src/ns_gan.py:283-285); same keys as the reference."""
        torch.save(self.model.state_dict(), savepath)

    def load_model(self, loadpath):
        """Load state dictionary into model (src/ns_gan.py:287-290)."""
        state = torch.load(loadpath)
        self.model.load_state_dict(state)
        if self._engine is not None:
            self._engine.sync_shadows(G_NET)
            self._engine.sync_shadows(D_NET)
