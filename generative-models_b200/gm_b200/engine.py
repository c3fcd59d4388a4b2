"""GanEngine — owns the flat fp32 parameter / gradient / Adam-state tensors (torch
allocations) and drives the C-ABI train-step engine on them."""
import ctypes as C

import torch

from . import _lib
from ._lib import AdamHP, GanDesc, VaeDesc, GmError, VARIANTS, OUT_ACTS, IMG_FMTS, PRECISIONS, check, lib, _ptr, _stream

G, D = 0, 1


class GanEngine:
    """One MLP GAN (z -> hidden -> image ; image -> hidden -> 1) on one GPU.

    Flat layouts follow nn.Module.parameters() order of the reference modules
    (src/ns_gan.py:40-41,54-55): [linear.weight, linear.bias, generate|discriminate.weight, .bias].
    """

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, max_batch=64, variant="ns",
                 d_out_act="sigmoid", device=None, precision="bf16"):
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.image_size, self.hidden_dim, self.z_dim = image_size, hidden_dim, z_dim
        self.max_batch = max_batch
        self.variant = variant
        self.precision = precision
        d = GanDesc(image_size, hidden_dim, z_dim, max_batch, VARIANTS[variant], OUT_ACTS[d_out_act], PRECISIONS[precision])
        self.g = C.c_void_p()
        check(self.h, lib().gm_gan_create(self.h, C.byref(d), C.byref(self.g)))
        self.n = [lib().gm_gan_param_count(self.g, G), lib().gm_gan_param_count(self.g, D)]
        kw = dict(device=self.device, dtype=torch.float32)
        self.params = [torch.zeros(n, **kw) for n in self.n]
        self.grads = [torch.zeros(n, **kw) for n in self.n]
        self.exp_avg = [torch.zeros(n, **kw) for n in self.n]
        self.exp_avg_sq = [torch.zeros(n, **kw) for n in self.n]
        self.loss_buf = torch.zeros(2, **kw)
        for net in (G, D):
            check(self.h, lib().gm_gan_bind(self.g, net, _ptr(self.params[net]), _ptr(self.grads[net]),
                                            _ptr(self.exp_avg[net]), _ptr(self.exp_avg_sq[net])))
        H, X, Z = hidden_dim, image_size, z_dim
        self.shapes = [[(H, Z), (H,), (X, H), (X,)], [(H, X), (H,), (1, H), (1,)]]
        if variant == "began":      # D is an autoencoder: encoder [h, x], decoder [x, h]
            self.shapes[1] = [(H, X), (H,), (X, H), (X,)]
        self.steps = [0, 0]

    def __del__(self):
        try:
            if getattr(self, "g", None):
                lib().gm_gan_destroy(self.g)
                self.g = None
        except Exception:
            pass

    # ---- parameter views -------------------------------------------------
    def views(self, net, flat=None):
        flat = self.params[net] if flat is None else flat
        out, off = [], 0
        for shp in self.shapes[net]:
            n = 1
            for s in shp:
                n *= s
            out.append(flat[off:off + n].view(shp))
            off += n
        return out

    def load(self, net, tensors):
        """Copy [W1, b1, W2, b2] into the flat fp32 master and refresh the bf16 copies."""
        for dst, src in zip(self.views(net), tensors):
            dst.copy_(torch.as_tensor(src, dtype=torch.float32).reshape(dst.shape))
        self.sync_shadows(net)

    def sync_shadows(self, net):
        check(self.h, lib().gm_gan_sync_shadows(self.g, net, _stream()))

    def sync_all(self):
        """Refresh both nets' bf16 operand copies from the fp32 masters (call after anything
        outside the engine — torch.optim, load_state_dict, clamp_ — touched the parameters)."""
        self.sync_shadows(G)
        self.sync_shadows(D)

    sync_if_stale = sync_all

    def track_versions(self, param_lists):
        self._tracked = param_lists

    def discriminate(self, images, fmt="f32"):
        n = images.shape[0]
        out = torch.empty(n, 1, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_discriminate(self.g, _ptr(images.contiguous()), IMG_FMTS[fmt], n, _ptr(out), _stream()))
        return out

    def reset_optimizer(self):
        for net in (G, D):
            self.exp_avg[net].zero_()
            self.exp_avg_sq[net].zero_()
        self.steps = [0, 0]

    # ---- the hot path ----------------------------------------------------
    def d_grad(self, images, noise=None, aux=None, fmt="f32", gather_idx=None, batch=None, inv_global_batch=None,
               seed=0, step=0, loss_out=None):
        """train_D + backward (src/ns_gan.py:172-194,138). Returns the device loss (0-dim view of loss_buf, or
        of `loss_out`, a 0-dim fp32 device tensor the kernel writes instead: per-epoch loss logs without a copy)."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        inv = 1.0 / B if inv_global_batch is None else inv_global_batch
        dst = self.loss_buf[0] if loss_out is None else loss_out
        check(self.h, lib().gm_gan_d_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, _ptr(noise),
                                          _ptr(aux), inv, seed, step, _ptr(dst), _stream()))
        return dst

    def d_stage(self, images, fmt="f32", gather_idx=None, batch=None, step=0):
        """process_batch of the next d_grad ahead of time (the following d_grad with the same batch skips its staging)."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        check(self.h, lib().gm_gan_d_stage(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, step, _stream()))

    def g_grad(self, batch, noise=None, inv_global_batch=None, seed=0, step=0, loss_out=None):
        """train_G + backward (src/ns_gan.py:196-216,155)."""
        inv = 1.0 / batch if inv_global_batch is None else inv_global_batch
        dst = self.loss_buf[1] if loss_out is None else loss_out
        check(self.h, lib().gm_gan_g_grad(self.g, batch, _ptr(noise), inv, seed, step, _ptr(dst), _stream()))
        return dst

    def g_forward_stage(self, batch, noise=None, seed=0, step=0):
        """First half of g_grad: the generator forward only (independent of the D update; lets a data-parallel
        host overlap it with the D-gradient exchange running on another stream)."""
        check(self.h, lib().gm_gan_g_forward_stage(self.g, batch, _ptr(noise), seed, step, _stream()))

    def g_grad_staged(self, batch, inv_global_batch=None, loss_out=None):
        """Second half of g_grad after g_forward_stage: D on the fake rows, loss, backward through D and G."""
        inv = 1.0 / batch if inv_global_batch is None else inv_global_batch
        dst = self.loss_buf[1] if loss_out is None else loss_out
        check(self.h, lib().gm_gan_g_grad_staged(self.g, batch, inv, _ptr(dst), _stream()))
        return dst

    def use_device_step(self, on=True):
        """Device-step mode (include/gm_b200.h: gm_gan_use_device_step): Adam step counts, Philox streams and the
        sampler round come from device counters, so a captured CUDA graph of one train step replays as successive
        steps.  Turning it on seeds the counters from this engine's host-side step counts; turning it off reads
        them back."""
        buf = (C.c_ulonglong * 4)()
        if on:
            buf[0], buf[1] = self.steps[0], self.steps[1]
            buf[2], buf[3] = getattr(self, "_g_calls", 0), getattr(self, "_d_calls", 0)
            check(self.h, lib().gm_gan_use_device_step(self.g, 1, buf, _stream()))
            self._device_step = True
        elif getattr(self, "_device_step", False):
            check(self.h, lib().gm_gan_device_steps(self.g, buf, _stream()))
            self.steps = [int(buf[0]), int(buf[1])]
            self._g_calls, self._d_calls = int(buf[2]), int(buf[3])
            check(self.h, lib().gm_gan_use_device_step(self.g, 0, None, _stream()))
            self._device_step = False

    def device_steps(self):
        buf = (C.c_ulonglong * 4)()
        check(self.h, lib().gm_gan_device_steps(self.g, buf, _stream()))
        return [int(v) for v in buf]

    def set_loss_consts(self, gp_lambda=10.0, gp_k=1.0, dra_c=1.0, ls_a=0.0, ls_b=1.0, ls_c=1.0):
        """LAMBDA / K / C of the gradient penalties, a / b / c of LSGAN (the reference's train_D / train_G kwargs)."""
        lc = _lib.LossConsts(gp_lambda, gp_k, dra_c, ls_a, ls_b, ls_c)
        check(self.h, lib().gm_gan_set_loss_consts(self.g, C.byref(lc)))
        self.loss_consts = dict(gp_lambda=gp_lambda, gp_k=gp_k, dra_c=dra_c, ls_a=ls_a, ls_b=ls_b, ls_c=ls_c)

    def set_sampler(self, n_pool, seed=0):
        """On-device batch sampling: d_grad(images=pool, gather_idx=None, batch=B, step=s) then reads the first B
        rows of a fresh pseudo-random permutation of the pool per step (src/ns_gan.py:222-226)."""
        check(self.h, lib().gm_gan_set_sampler(self.g, int(n_pool), int(seed) & 0xFFFFFFFFFFFFFFFF))

    def sample_indices(self, batch, step):
        out = torch.empty(batch, device=self.device, dtype=torch.int32)
        check(self.h, lib().gm_gan_sample_indices(self.g, batch, int(step), _ptr(out), _stream()))
        return out

    BUFFERS = {"Zb": 0, "Hg": 1, "Xall": 2, "Aall": 3, "DHall": 4, "DA2": 5, "DHg": 6}

    def debug_read(self, which, row0, rows, cols, plane=0):
        """An internal bf16 activation buffer as fp32 [rows, cols] (plane 0: hi + lo in split mode, 1: hi, 2: lo); tests only."""
        out = torch.empty(rows, cols, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_debug_read(self.g, self.BUFFERS[which] + 16 * plane, row0, rows, cols, _ptr(out), _stream()))
        return out

    def debug_noise(self, batch, seed, step, g_step=False):
        """The on-device Philox noise of (seed, step) as the bf16 operand values, [batch, z] fp32."""
        out = torch.empty(batch, self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_debug_noise(self.g, batch, int(seed), int(step), 1 if g_step else 0, _ptr(out), _stream()))
        return out

    def apply(self, net, hp):
        """optimizer.step() (src/ns_gan.py:139,156)."""
        self.steps[net] += 1
        check(self.h, lib().gm_gan_apply(self.g, net, C.byref(hp), self.steps[net], _stream()))

    def scores(self, n):
        out = torch.empty(n, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_scores(self.g, _ptr(out), n, _stream()))
        return out

    def generate(self, noise):
        n = noise.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_generate(self.g, _ptr(noise.contiguous().float()), n, _ptr(out), _stream()))
        return out

    def apply_allreduce(self, net, hp, comm):
        """Data-parallel optimizer.step(): SUM all-reduce of the gradient over the peer mappings of
        `comm` (parallel.PeerComm) fused with Adam, one kernel per rank."""
        self.steps[net] += 1
        check(self.h, lib().gm_gan_apply_allreduce(self.g, net, C.byref(hp), self.steps[net], comm.c, _stream()))

    def exchange_begin(self, net, comm):
        """First half of apply_allreduce: publish the gradient to the peers without waiting (work that does not depend on
        the update can be enqueued before the matching apply_allreduce)."""
        check(self.h, lib().gm_gan_exchange_begin(self.g, net, comm.c, _stream()))

    def attach_comm(self, comm):
        """Batch statistics (RaNS / Fisher / DRAGAN / BEGAN) over the global batch of all ranks of `comm`
        (parallel.PeerComm); None detaches."""
        check(self.h, lib().gm_gan_attach_comm(self.g, comm.c if comm is not None else None))

    def set_lazy_grads(self, on=True):
        """Single-GPU fast path: d_grad / g_grad leave split-K partials and apply() gathers + updates
        in one kernel; self.grads[net] is then valid only after apply() (or materialize_grads())."""
        check(self.h, lib().gm_gan_set_lazy_grads(self.g, 1 if on else 0, _stream()))

    def materialize_grads(self):
        check(self.h, lib().gm_gan_materialize_grads(self.g, _stream()))

    # ---- custom-loss path (README.md:31): forward / backward halves as separate calls
    g_generation = 0
    d_calls = 0

    @property
    def supports_custom_loss(self):
        return self.variant not in ("began",)        # BEGAN's D is an autoencoder (src/be_gan.py:63-76)

    @property
    def d_generation(self):
        if not hasattr(self, "_d_generation"):
            self._d_generation = [0] * self.num_slots()
        return self._d_generation

    def num_slots(self):
        return lib().gm_gan_num_slots(self.g)

    def d_forward(self, slot, x):
        n = x.shape[0]
        out = torch.empty(n, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_d_forward(self.g, slot, _ptr(x), n, _ptr(out), _stream()))
        return out

    def d_backward(self, slot, dscore, need_dx):
        """-> (flat D gradient (engine buffer, overwritten by the next call), dL/dx or None)"""
        n = dscore.shape[0]
        dx = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32) if need_dx else None
        check(self.h, lib().gm_gan_d_backward(self.g, slot, n, _ptr(dscore), _ptr(dx), _stream()))
        return self.grads[1], dx

    def g_forward(self, noise):
        n = noise.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_g_forward(self.g, _ptr(noise), n, _ptr(out), _stream()))
        return out

    def g_backward(self, dimages):
        check(self.h, lib().gm_gan_g_backward(self.g, dimages.shape[0], _ptr(dimages), _stream()))
        return self.grads[0]

    def began_state(self, values=None):
        """BEGAN device state (list of 11 floats, see include/gm_b200.h); pass values to set."""
        buf = (C.c_float * 11)()
        if values is not None:
            for i, v in enumerate(values):
                buf[i] = v
            check(self.h, lib().gm_gan_began_state(self.g, buf, 1, _stream()))
            return list(values)
        check(self.h, lib().gm_gan_began_state(self.g, buf, 0, _stream()))
        return list(buf)

    def began_init(self, K, batch, world=1):
        inv = 1.0 / (batch * world)
        return self.began_state([K, inv, -K * inv, 0.0, 0.0, float("inf"), 0.0, 1.0, inv, inv, 0.0])

    def began_control(self, gamma, lam, patience):
        check(self.h, lib().gm_gan_began_control(self.g, gamma, lam, float(patience), _stream()))

    def fisher_state(self, lam=None, rho=None):
        buf = (C.c_float * 2)()
        if lam is not None:
            buf[0], buf[1] = lam, rho
            check(self.h, lib().gm_gan_fisher_state(self.g, buf, 1, _stream()))
            return lam, rho
        check(self.h, lib().gm_gan_fisher_state(self.g, buf, 0, _stream()))
        return buf[0], buf[1]


class InfoGanEngine(GanEngine):
    """GanEngine + the auxiliary network Q and the mutual-information step of InfoGAN
    (src/info_gan.py:78-94,269-304).  The generator input is z + disc_dim + cont_dim wide."""

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, disc_dim=10, cont_dim=10, max_batch=64, device=None,
                 precision="bf16"):
        if (disc_dim, cont_dim) != (10, 10):
            raise GmError("the fused Q head is built for disc_dim = cont_dim = 10 (the reference's setting)")
        super().__init__(image_size, hidden_dim, z_dim + disc_dim + cont_dim, max_batch, variant="info", device=device,
                         precision=precision)
        self.noise_dim, self.code_z = z_dim + disc_dim + cont_dim, z_dim
        nq = lib().gm_gan_q_param_count(self.g)
        kw = dict(device=self.device, dtype=torch.float32)
        self.q_params, self.q_grads = torch.zeros(nq, **kw), torch.zeros(nq, **kw)
        self.q_exp_avg, self.q_exp_avg_sq = torch.zeros(nq, **kw), torch.zeros(nq, **kw)
        self.g_mi_exp_avg, self.g_mi_exp_avg_sq = torch.zeros(self.n[G], **kw), torch.zeros(self.n[G], **kw)
        check(self.h, lib().gm_gan_bind_q(self.g, _ptr(self.q_params), _ptr(self.q_grads), _ptr(self.q_exp_avg),
                                          _ptr(self.q_exp_avg_sq), _ptr(self.g_mi_exp_avg), _ptr(self.g_mi_exp_avg_sq)))
        H, X = hidden_dim, image_size
        self.q_shapes = [(H, X), (H,), (disc_dim + cont_dim, H), (disc_dim + cont_dim,)]
        self.mi_steps = 0

    def q_views(self, flat=None):
        flat = self.q_params if flat is None else flat
        out, off = [], 0
        for shp in self.q_shapes:
            n = 1
            for s in shp:
                n *= s
            out.append(flat[off:off + n].view(shp))
            off += n
        return out

    def load_q(self, tensors):
        for dst, src in zip(self.q_views(), tensors):
            dst.copy_(torch.as_tensor(src, dtype=torch.float32).reshape(dst.shape))
        self.sync_shadows_q()

    def sync_shadows_q(self):
        check(self.h, lib().gm_gan_sync_shadows_q(self.g, _stream()))

    def sync_all(self):
        super().sync_all()
        self.sync_shadows_q()

    sync_if_stale = sync_all

    def reset_optimizer(self):
        super().reset_optimizer()
        for t in (self.q_exp_avg, self.q_exp_avg_sq, self.g_mi_exp_avg, self.g_mi_exp_avg_sq):
            t.zero_()
        self.mi_steps = 0

    def q_grad(self, batch, noise, inv_global_batch=None):
        """train_Q + backward (src/info_gan.py:269-304,204): G and Q gradients, MI loss."""
        inv = 1.0 / batch if inv_global_batch is None else inv_global_batch
        if not hasattr(self, "mi_loss_buf"):
            self.mi_loss_buf = torch.zeros(1, device=self.device)
        check(self.h, lib().gm_gan_q_grad(self.g, batch, _ptr(noise), self.code_z, inv, _ptr(self.mi_loss_buf), _stream()))
        return self.mi_loss_buf[0]

    def apply_mi(self, hp):
        self.mi_steps += 1
        check(self.h, lib().gm_gan_apply_mi(self.g, C.byref(hp), self.mi_steps, _stream()))


class VaeEngine:
    """One MLP VAE (x -> hidden -> (mu, log_var) ; z -> hidden -> x) on one GPU.  The flat
    layout puts the two latent heads next to each other (one 400 -> 2z GEMM):
    [enc.linear.W, .b, enc.mu.W, enc.log_var.W, enc.mu.b, enc.log_var.b, dec.linear.W, .b, dec.recon.W, .b]."""
    NAMES = ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.log_var.weight",
             "encoder.mu.bias", "encoder.log_var.bias", "decoder.linear.weight", "decoder.linear.bias",
             "decoder.recon.weight", "decoder.recon.bias"]

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, max_batch=64, device=None, precision="bf16"):
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.image_size, self.hidden_dim, self.z_dim, self.max_batch = image_size, hidden_dim, z_dim, max_batch
        self.precision = precision
        d = VaeDesc(image_size, hidden_dim, z_dim, max_batch, PRECISIONS[precision])
        self.g = C.c_void_p()
        check(self.h, lib().gm_vae_create(self.h, C.byref(d), C.byref(self.g)))
        n = lib().gm_vae_param_count(self.g)
        kw = dict(device=self.device, dtype=torch.float32)
        self.params, self.grads = torch.zeros(n, **kw), torch.zeros(n, **kw)
        self.exp_avg, self.exp_avg_sq = torch.zeros(n, **kw), torch.zeros(n, **kw)
        self.loss_buf = torch.zeros(2, **kw)
        check(self.h, lib().gm_vae_bind(self.g, _ptr(self.params), _ptr(self.grads), _ptr(self.exp_avg), _ptr(self.exp_avg_sq)))
        X, H, Z = image_size, hidden_dim, z_dim
        self.shapes = [(H, X), (H,), (Z, H), (Z, H), (Z,), (Z,), (H, Z), (H,), (X, H), (X,)]
        self.steps = 0

    def __del__(self):
        try:
            if getattr(self, "g", None):
                lib().gm_vae_destroy(self.g)
                self.g = None
        except Exception:
            pass

    def views(self, flat=None):
        """{reference parameter name: view into the flat buffer}"""
        flat = self.params if flat is None else flat
        out, off = {}, 0
        for name, shp in zip(self.NAMES, self.shapes):
            n = 1
            for s in shp:
                n *= s
            out[name] = flat[off:off + n].view(shp)
            off += n
        return out

    def load(self, tensors):
        v = self.views()
        for name, src in tensors.items():
            v[name].copy_(torch.as_tensor(src, dtype=torch.float32).reshape(v[name].shape))
        self.sync_shadows()

    def sync_shadows(self):
        check(self.h, lib().gm_vae_sync_shadows(self.g, _stream()))

    sync_all = sync_shadows

    def reset_optimizer(self):
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self.steps = 0

    def grad(self, images, eps=None, fmt="f32", gather_idx=None, batch=None, seed=0, step=0):
        """compute_batch + backward (src/vae.py:157-161). Returns the device tensor [recon, kl]."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        check(self.h, lib().gm_vae_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, _ptr(eps), 1.0, seed, step,
                                        _ptr(self.loss_buf), _stream()))
        return self.loss_buf

    def set_sampler(self, n_pool, batches_per_epoch, seed=0, batch_size=0):
        """On-device epoch shuffling: grad(images=pool, gather_idx=None, batch=B, step=s) reads batch
        s % batches_per_epoch of the permutation of epoch s // batches_per_epoch (src/vae.py:150); batch_size = the
        loader's nominal batch when the last batch of an epoch is shorter."""
        check(self.h, lib().gm_vae_set_sampler(self.g, int(n_pool), int(batches_per_epoch), int(batch_size),
                                               int(seed) & 0xFFFFFFFFFFFFFFFF))

    def set_lazy_grads(self, on=True):
        """Single-GPU fast path: grad() leaves split-K partials, apply() gathers + updates in one kernel; self.grads is
        then valid only after apply() (or materialize_grads())."""
        check(self.h, lib().gm_vae_set_lazy_grads(self.g, 1 if on else 0, _stream()))

    def materialize_grads(self):
        check(self.h, lib().gm_vae_materialize_grads(self.g, _stream()))

    def last_eps(self, batch):
        out = torch.empty(batch, self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_last_eps(self.g, _ptr(out), batch, _stream()))
        return out

    def sample_indices(self, batch, step, batches_per_epoch, n_pool, seed):
        """host evaluation of the epoch sampler's draw for `step` (tests)"""
        import numpy as np
        out = np.empty(batch, dtype=np.int32)
        bpe = max(int(batches_per_epoch), 1)
        check(self.h, lib().gm_sampler_indices_host(int(n_pool), int(seed), int(step) // bpe, (int(step) % bpe) * batch, batch,
                                                    C.c_void_p(out.ctypes.data)))
        return torch.from_numpy(out).to(self.device)

    def apply(self, hp):
        self.steps += 1
        check(self.h, lib().gm_vae_apply(self.g, C.byref(hp), self.steps, _stream()))

    def forward(self, images, eps=None, fmt="f32", want_images=True, want_latent=True, want_losses=False, seed=0, step=0):
        n = images.shape[0]
        kw = dict(device=self.device, dtype=torch.float32)
        out = torch.empty(n, self.image_size, **kw) if want_images else None
        ml = torch.empty(n, 2 * self.z_dim, **kw) if want_latent else None
        ls = torch.empty(2, **kw) if want_losses else None
        check(self.h, lib().gm_vae_forward(self.g, _ptr(images.contiguous()), IMG_FMTS[fmt], n, _ptr(eps), seed, step,
                                           _ptr(out), _ptr(ml), _ptr(ls), _stream()))
        mu = ml[:, :self.z_dim] if ml is not None else None
        lv = ml[:, self.z_dim:] if ml is not None else None
        return out, mu, lv, ls

    def decode(self, z):
        n = z.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_decode(self.g, _ptr(z.contiguous().float()), n, _ptr(out), _stream()))
        return out

    # ------------------------------------------------------------------ per-call encoder / decoder (user-written losses)
    def num_slots(self):
        return lib().gm_vae_num_slots(self.g)

    def encoder_forward(self, slot, x):
        """Encoder.forward on slot's buffers: x [n, image_size] fp32 -> (mu, log_var) [n, z] fp32"""
        n = x.shape[0]
        ml = torch.empty(n, 2 * self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_encoder_forward(self.g, slot, _ptr(x.contiguous()), n, _ptr(ml), _stream()))
        return ml[:, :self.z_dim], ml[:, self.z_dim:]

    def encoder_backward(self, slot, n, dmu, dlog_var):
        """-> {encoder parameter name: gradient} of encoder_forward's call on slot"""
        grads = torch.empty_like(self.params)
        dml = torch.cat([dmu.float(), dlog_var.float()], dim=1).contiguous()
        check(self.h, lib().gm_vae_encoder_backward(self.g, slot, n, _ptr(dml), _ptr(grads), _stream()))
        return {k: v for k, v in self.views(grads).items() if k.startswith("encoder.")}

    def decoder_forward(self, slot, z):
        """Decoder.forward on slot's buffers: z [n, z] fp32 -> images [n, image_size] fp32"""
        n = z.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_decoder_forward(self.g, slot, _ptr(z.contiguous()), n, _ptr(out), _stream()))
        return out

    def decoder_backward(self, slot, n, dimages, need_dz):
        """-> ({decoder parameter name: gradient}, dL/dz [n, z] fp32 or None) of decoder_forward's call on slot"""
        grads = torch.empty_like(self.params)
        dz = torch.empty(n, self.z_dim, device=self.device, dtype=torch.float32) if need_dz else None
        check(self.h, lib().gm_vae_decoder_backward(self.g, slot, n, _ptr(dimages.float().contiguous()), _ptr(grads), _ptr(dz),
                                                    _stream()))
        return {k: v for k, v in self.views(grads).items() if k.startswith("decoder.")}, dz

    def slot_bytes(self):
        """device bytes one encoder slot and one decoder slot hold (allocated on the first per-call use)"""
        XP, HP, ZP, B = (self.image_size + 16) // 16 * 16, (self.hidden_dim + 16) // 16 * 16, (self.z_dim + 64) // 64 * 64, self.max_batch
        return 2 * B * (XP + HP) + 4 * B * 64, 2 * B * (ZP + HP + XP)
