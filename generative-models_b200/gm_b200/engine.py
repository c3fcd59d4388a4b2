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

    BUFFERS = {"Zb": 0, "Hg": 1, "Xall": 2, "Aall": 3, "DHall": 4, "DA2": 5, "DHg": 6, "HQ0": 7, "HQ1": 8}

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
    @property
    def supports_custom_loss(self):
        """True where Discriminator.forward is the scalar-score node (gm_gan_d_*); BEGAN's D is an autoencoder
        (src/be_gan.py:63-76) with nodes of its own (ae_forward / ae_backward)"""
        return self.variant not in ("began",)

    supports_custom_g = True       # Generator.forward is a node on every variant (gm_gan_g_*)

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

    def ae_forward(self, slot, x):
        """BEGAN's Discriminator.forward (the autoencoder) on slot's row region: x [n, image_size] -> recon, fp32"""
        n = x.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_ae_forward(self.g, slot, _ptr(x), n, _ptr(out), _stream()))
        return out

    def ae_backward(self, slot, drecon, need_dx):
        """-> (flat D gradient (engine buffer, overwritten by the next call), dL/dx or None) of ae_forward's call on slot"""
        n = drecon.shape[0]
        dx = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32) if need_dx else None
        check(self.h, lib().gm_gan_ae_backward(self.g, slot, n, _ptr(drecon), _ptr(dx), _stream()))
        return self.grads[1], dx

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

    # ---- per-call Q (user-written train_Q)
    def num_q_slots(self):
        return lib().gm_gan_num_q_slots(self.g)

    def q_forward(self, slot, x):
        """Q.forward on slot's buffers: x [n, image_size] fp32 -> codes [n, disc + cont] fp32 (logits | continuous)"""
        n = x.shape[0]
        out = torch.empty(n, self.q_shapes[3][0], device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_gan_q_forward(self.g, slot, _ptr(x), n, _ptr(out), _stream()))
        return out

    def q_backward(self, slot, dcodes, need_dx):
        """-> (flat Q gradient (q_grads, overwritten by the next call), dL/dx or None) of q_forward's call on slot"""
        n = dcodes.shape[0]
        dx = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32) if need_dx else None
        check(self.h, lib().gm_gan_q_backward(self.g, slot, n, _ptr(dcodes), _ptr(dx), _stream()))
        return self.q_grads, dx


class VaeEngine:
    """One MLP VAE (x -> hidden -> (mu, log_var) ; z -> hidden -> x) on one GPU.  The flat
    layout puts the two latent heads next to each other (one 400 -> 2z GEMM):
    [enc.linear.W, .b, enc.mu.W, enc.log_var.W, enc.mu.b, enc.log_var.b, dec.linear.W, .b, dec.recon.W, .b]."""
    NAMES = ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.log_var.weight",
             "encoder.mu.bias", "encoder.log_var.bias", "decoder.linear.weight", "decoder.linear.bias",
             "decoder.recon.weight", "decoder.recon.bias"]

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, max_batch=64, device=None, precision="bf16"):
        X, H, Z = image_size, hidden_dim, z_dim
        self._open(image_size, hidden_dim, z_dim, max_batch, device, precision, lambda h, d, out: lib().gm_vae_create(h, d, out),
                   [(H, X), (H,), (Z, H), (Z, H), (Z,), (Z,), (H, Z), (H,), (X, H), (X,)])

    def _open(self, image_size, hidden_dim, z_dim, max_batch, device, precision, create, shapes):
        """create(ctx, desc, out) one engine of the gm_vae family, bind its flat fp32 buffers; shapes: the tensors of the
        flat layout in NAMES order"""
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.image_size, self.hidden_dim, self.z_dim, self.max_batch = image_size, hidden_dim, z_dim, max_batch
        self.precision = precision
        d = VaeDesc(image_size, hidden_dim, z_dim, max_batch, PRECISIONS[precision])
        self.g = C.c_void_p()
        check(self.h, create(self.h, C.byref(d), C.byref(self.g)))
        n = lib().gm_vae_param_count(self.g)
        kw = dict(device=self.device, dtype=torch.float32)
        self.params, self.grads = torch.zeros(n, **kw), torch.zeros(n, **kw)
        self.exp_avg, self.exp_avg_sq = torch.zeros(n, **kw), torch.zeros(n, **kw)
        self.loss_buf = torch.zeros(2, **kw)
        check(self.h, lib().gm_vae_bind(self.g, _ptr(self.params), _ptr(self.grads), _ptr(self.exp_avg), _ptr(self.exp_avg_sq)))
        self.shapes = shapes
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

    BUFFERS = {"Xin": 0, "H1": 1, "Zb": 2, "H3": 3, "DA4": 4, "DA3": 5, "DML": 6, "DA1": 7}

    def debug_read(self, which, row0, rows, cols):
        """An internal bf16 buffer of the last grad() as fp32 [rows, cols] (hi + lo in split mode); tests only."""
        out = torch.empty(rows, cols, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_debug_read(self.g, self.BUFFERS[which], row0, rows, cols, _ptr(out), _stream()))
        return out

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


class BirVaeEngine(VaeEngine):
    """One MLP BIR-VAE (x -> hidden -> mu ; z = mu + eps ; z -> hidden -> x) on one GPU: the VAE engine in its BIR mode
    (gm_bir_vae_create).  Flat layout [enc.linear.W, .b, enc.mu.W, .b, dec.linear.W, .b, dec.recon.W, .b].  eps_std is
    the standard deviation of eps (the reference's set_var, src/bir_vae.py:82,91)."""
    NAMES = ["encoder.linear.weight", "encoder.linear.bias", "encoder.mu.weight", "encoder.mu.bias",
             "decoder.linear.weight", "decoder.linear.bias", "decoder.recon.weight", "decoder.recon.bias"]

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, eps_std=1.0, max_batch=64, device=None, precision="bf16"):
        self.eps_std = float(eps_std)
        X, H, Z = image_size, hidden_dim, z_dim
        self._open(image_size, hidden_dim, z_dim, max_batch, device, precision,
                   lambda h, d, out: lib().gm_bir_vae_create(h, d, self.eps_std, out),
                   [(H, X), (H,), (Z, H), (Z,), (H, Z), (H,), (X, H), (X,)])

    def grad(self, images, eps=None, prior=None, lam=1000.0, fmt="f32", gather_idx=None, batch=None, seed=0, step=0):
        """compute_batch + backward (src/bir_vae.py:148-188). Returns the device tensor [mse, mmd]."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        check(self.h, lib().gm_bir_vae_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, _ptr(eps), _ptr(prior),
                                            float(lam), seed, step, _ptr(self.loss_buf), _stream()))
        return self.loss_buf

    def forward(self, images, eps=None, prior=None, lam=1000.0, fmt="f32", want_images=True, want_latent=True,
                want_losses=False, seed=0, step=0):
        """-> (images or None, mu or None, losses [mse, mmd] or None)"""
        n = images.shape[0]
        kw = dict(device=self.device, dtype=torch.float32)
        out = torch.empty(n, self.image_size, **kw) if want_images else None
        mu = torch.empty(n, self.z_dim, **kw) if want_latent else None
        ls = torch.empty(2, **kw) if want_losses else None
        check(self.h, lib().gm_bir_vae_forward(self.g, _ptr(images.contiguous()), IMG_FMTS[fmt], n, _ptr(eps), _ptr(prior),
                                               float(lam), seed, step, _ptr(out), _ptr(mu), _ptr(ls), _stream()))
        return out, mu, ls

    def last_latent(self, batch):
        """(z, p) [batch, z] fp32 of the last grad() / forward()"""
        z = torch.empty(batch, self.z_dim, device=self.device, dtype=torch.float32)
        p = torch.empty_like(z)
        check(self.h, lib().gm_bir_vae_last_latent(self.g, _ptr(z), _ptr(p), batch, _stream()))
        return z, p

    def encoder_forward(self, slot, x):
        """Encoder.forward on slot's buffers: x [n, image_size] fp32 -> mu [n, z] fp32"""
        n = x.shape[0]
        mu = torch.empty(n, self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_vae_encoder_forward(self.g, slot, _ptr(x.contiguous()), n, _ptr(mu), _stream()))
        return mu

    def encoder_backward(self, slot, n, dmu):
        """-> {encoder parameter name: gradient} of encoder_forward's call on slot"""
        grads = torch.empty_like(self.params)
        check(self.h, lib().gm_vae_encoder_backward(self.g, slot, n, _ptr(dmu.float().contiguous()), _ptr(grads), _stream()))
        return {k: v for k, v in self.views(grads).items() if k.startswith("encoder.")}


class AaeEngine(VaeEngine):
    """One MLP adversarial autoencoder on one GPU: the VAE engine in its AAE mode (gm_aae_create).  Encoder x -> hidden ->
    z (deterministic), Decoder z -> hidden -> x, and a latent discriminator Dz z -> hidden -> 1 with flat parameters,
    gradient and Adam state of its own (d_params, ...) and optimizer_G's moments over the encoder (enc_g_exp_avg, ...).
    One train step: recon_grad, apply (optimizer_R over encoder + decoder), d_grad, apply_d, g_grad, apply_g."""
    NAMES = BirVaeEngine.NAMES
    D_NAMES = ["discriminator.linear.weight", "discriminator.linear.bias", "discriminator.discriminate.weight",
               "discriminator.discriminate.bias"]

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, max_batch=64, device=None, precision="bf16"):
        if precision != "bf16":
            raise GmError("the AAE engine runs in bf16 only (got precision=%r)" % (precision,))
        X, H, Z = image_size, hidden_dim, z_dim
        self._open(image_size, hidden_dim, z_dim, max_batch, device, precision, lambda h, d, out: lib().gm_aae_create(h, d, out),
                   [(H, X), (H,), (Z, H), (Z,), (H, Z), (H,), (X, H), (X,)])
        nd = lib().gm_aae_d_param_count(self.g)
        kw = dict(device=self.device, dtype=torch.float32)
        self.d_params, self.d_grads = torch.zeros(nd, **kw), torch.zeros(nd, **kw)
        self.d_exp_avg, self.d_exp_avg_sq = torch.zeros(nd, **kw), torch.zeros(nd, **kw)
        ne = H * X + H + Z * H + Z                 # the encoder prefix of the flat layout
        self.n_enc = ne
        self.enc_g_exp_avg, self.enc_g_exp_avg_sq = torch.zeros(ne, **kw), torch.zeros(ne, **kw)
        check(self.h, lib().gm_aae_bind_d(self.g, _ptr(self.d_params), _ptr(self.d_grads), _ptr(self.d_exp_avg),
                                          _ptr(self.d_exp_avg_sq), _ptr(self.enc_g_exp_avg), _ptr(self.enc_g_exp_avg_sq)))
        self.d_shapes = [(H, Z), (H,), (1, H), (1,)]
        self.d_loss_buf, self.g_loss_buf = torch.zeros(1, **kw), torch.zeros(1, **kw)
        self.d_steps, self.g_steps = 0, 0

    # ---- the latent discriminator's parameters
    def d_views(self, flat=None):
        """{discriminator parameter name: view into the flat D buffer}"""
        flat = self.d_params if flat is None else flat
        out, off = {}, 0
        for name, shp in zip(self.D_NAMES, self.d_shapes):
            n = 1
            for s in shp:
                n *= s
            out[name] = flat[off:off + n].view(shp)
            off += n
        return out

    def views(self, flat=None):
        """{parameter name: view}: the encoder / decoder of the main buffer (or of `flat`), and with no `flat` the
        discriminator's views of d_params too"""
        out = super().views(flat)
        if flat is None:
            out.update(self.d_views())
        return out

    def load(self, tensors):
        main = {k: v for k, v in tensors.items() if not k.startswith("discriminator.")}
        dv = self.d_views()
        for name, src in tensors.items():
            if name.startswith("discriminator."):
                dv[name].copy_(torch.as_tensor(src, dtype=torch.float32).reshape(dv[name].shape))
        VaeEngine.load(self, main)
        self.sync_shadows_d()

    def sync_shadows_d(self):
        check(self.h, lib().gm_aae_sync_shadows_d(self.g, _stream()))

    def sync_all(self):
        self.sync_shadows()
        self.sync_shadows_d()

    sync_if_stale = sync_all

    def reset_optimizer(self):
        """zero the three Adam states: optimizer_R (encoder + decoder), optimizer_D and optimizer_G (encoder)"""
        super().reset_optimizer()
        for t in (self.d_exp_avg, self.d_exp_avg_sq, self.enc_g_exp_avg, self.enc_g_exp_avg_sq):
            t.zero_()
        self.d_steps, self.g_steps = 0, 0

    # ---- the three phases of one train step
    def recon_grad(self, images, fmt="f32", gather_idx=None, batch=None, step=0):
        """phase 1, recon = sum (x - D(E(x)))^2 and its gradient.  Returns the device tensor [recon] (a view of loss_buf)."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        check(self.h, lib().gm_aae_recon_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, int(step),
                                              _ptr(self.loss_buf), _stream()))
        return self.loss_buf[:1]

    def d_grad(self, batch, prior=None, seed=0, step=0):
        """phase 2 on the batch recon_grad staged: D_loss and Dz's gradient (d_grads); prior [batch, z] or the device draw"""
        if prior is not None:
            prior = prior.float().contiguous()
        check(self.h, lib().gm_aae_d_grad(self.g, batch, _ptr(prior), int(seed), int(step), _ptr(self.d_loss_buf), _stream()))
        return self.d_loss_buf

    def g_grad(self, batch):
        """phase 3 on phase 2's encoding: G_loss and the encoder prefix of grads"""
        check(self.h, lib().gm_aae_g_grad(self.g, batch, _ptr(self.g_loss_buf), _stream()))
        return self.g_loss_buf

    def apply_d(self, hp):
        self.d_steps += 1
        check(self.h, lib().gm_aae_apply_d(self.g, C.byref(hp), self.d_steps, _stream()))

    def apply_g(self, hp):
        self.g_steps += 1
        check(self.h, lib().gm_aae_apply_g(self.g, C.byref(hp), self.g_steps, _stream()))

    def last_prior(self, batch):
        out = torch.empty(batch, self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_aae_last_prior(self.g, _ptr(out), batch, _stream()))
        return out

    def forward(self, images, fmt="f32", want_images=True, want_latent=True, want_losses=False):
        """-> (images or None, z or None, losses [recon] or None)"""
        n = images.shape[0]
        kw = dict(device=self.device, dtype=torch.float32)
        out = torch.empty(n, self.image_size, **kw) if want_images else None
        z = torch.empty(n, self.z_dim, **kw) if want_latent else None
        ls = torch.empty(1, **kw) if want_losses else None
        check(self.h, lib().gm_aae_forward(self.g, _ptr(images.contiguous()), IMG_FMTS[fmt], n, _ptr(out), _ptr(z), _ptr(ls),
                                           _stream()))
        return out, z, ls

    BUFFERS = dict(VaeEngine.BUFFERS, ZD=8, AD=9, DHD=10)

    encoder_forward = BirVaeEngine.encoder_forward
    encoder_backward = BirVaeEngine.encoder_backward

    # ---- the per-call latent D (user-written train_D / train_G)
    def num_d_slots(self):
        return lib().gm_aae_num_d_slots(self.g)

    def d_forward(self, slot, z):
        """Dz.forward on slot's rows: z [n, z] fp32 -> scores [n] fp32"""
        n = z.shape[0]
        out = torch.empty(n, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_aae_d_forward(self.g, slot, _ptr(z.float().contiguous()), n, _ptr(out), _stream()))
        return out

    def d_backward(self, slot, dscores, need_dz):
        """-> ({discriminator parameter name: gradient} (views of d_grads, overwritten by the next call), dL/dz or None)"""
        n = dscores.shape[0]
        dz = torch.empty(n, self.z_dim, device=self.device, dtype=torch.float32) if need_dz else None
        check(self.h, lib().gm_aae_d_backward(self.g, slot, n, _ptr(dscores.reshape(-1).float().contiguous()), _ptr(dz), _stream()))
        return self.d_views(self.d_grads), dz


class ClassIds:
    """Class labels checked against an engine's num_classes and held as an int32 tensor on its device (CvaeEngine.class_ids)"""
    __slots__ = ("t", "num_classes")

    def __init__(self, t, num_classes):
        self.t, self.num_classes = t, num_classes

    def __len__(self):
        return self.t.numel()


def class_ids(labels, num_classes, device, n=None):
    """labels (class ids in [0, num_classes): an integer tensor, array or sequence of shape [m] or [m, 1], with m == n when
    n is given) -> ClassIds on device.  Anything else - a one-hot matrix included - raises GmError here, on the host,
    before the labels are uploaded or a kernel runs."""
    import numpy as np
    def count(m):
        if n is not None and m != n:
            raise GmError("%d labels for %d rows" % (m, n))
    if isinstance(labels, ClassIds):
        if labels.num_classes != num_classes or labels.t.device != device:
            raise GmError("labels were checked for %d classes on %s, not %d on %s"
                          % (labels.num_classes, labels.t.device, num_classes, device))
        count(len(labels))
        return labels
    t = labels if torch.is_tensor(labels) else torch.as_tensor(np.asarray(labels))
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise GmError("labels must be integer class ids (got dtype %s)" % t.dtype)
    if not (t.dim() == 1 or (t.dim() == 2 and t.shape[1] == 1)):
        raise GmError("labels must be class ids of shape [n] or [n, 1], not one-hot or other rows (got shape %s)"
                      % (tuple(t.shape),))
    t = t.reshape(-1)
    count(t.numel())
    if t.numel() == 0:
        raise GmError("labels are empty")
    if t.numel() >= 2 ** 31:
        raise GmError("more than 2^31 labels")
    lo, hi = int(t.min()), int(t.max())
    if lo < 0 or hi >= num_classes:
        raise GmError("labels must be in [0, %d) (got values in [%d, %d])" % (num_classes, lo, hi))
    return ClassIds(t.to(device=device, dtype=torch.int32).contiguous(), num_classes)


class CvaeEngine(VaeEngine):
    """One MLP conditional VAE (x, y -> hidden -> (mu, log_var) ; z, y -> hidden -> x) on one GPU: the VAE engine in its
    CVAE mode (gm_cvae_create).  The flat layout is the VAE's, with encoder.linear.weight (H, X + C) and
    decoder.linear.weight (H, Z + C): the one-hot columns follow the x (z) columns.  Every entry that takes labels takes
    integer class ids or a ClassIds from class_ids()."""

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, num_classes=10, max_batch=64, device=None, precision="bf16"):
        if precision != "bf16":
            raise GmError("the CVAE engine runs in bf16 only (got precision=%r)" % (precision,))
        self.num_classes = int(num_classes)
        X, H, Z, K = image_size, hidden_dim, z_dim, self.num_classes
        self._open(image_size, hidden_dim, z_dim, max_batch, device, precision,
                   lambda h, d, out: lib().gm_cvae_create(h, d, self.num_classes, out),
                   [(H, X + K), (H,), (Z, H), (Z, H), (Z,), (Z,), (H, Z + K), (H,), (X, H), (X,)])

    def class_ids(self, labels, n=None):
        """labels checked for this engine (exactly n of them when n is given) -> ClassIds on its device"""
        return class_ids(labels, self.num_classes, self.device, n)

    def set_sampler(self, n_pool, batches_per_epoch, seed=0, batch_size=0):
        super().set_sampler(n_pool, batches_per_epoch, seed, batch_size)
        self._pool_n = int(n_pool)

    def grad(self, images, labels, eps=None, fmt="f32", gather_idx=None, batch=None, seed=0, step=0):
        """compute_batch + backward on (images, labels). Returns the device tensor [recon, kl].  With gather_idx or the
        epoch sampler, labels is the pool's label array, read at each gathered row."""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        pool = getattr(self, "_pool_n", 0)
        # one label per image the kernels may read: the whole image pool with gather_idx or the sampler, else the batch
        y = self.class_ids(labels, images.shape[0] if gather_idx is not None else pool if pool > 0 else B)
        check(self.h, lib().gm_cvae_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(y.t), _ptr(gather_idx), B, _ptr(eps), seed, step,
                                         _ptr(self.loss_buf), _stream()))
        return self.loss_buf

    def forward(self, images, labels, eps=None, fmt="f32", want_images=True, want_latent=True, want_losses=False, seed=0, step=0):
        n = images.shape[0]
        y = self.class_ids(labels, n)
        kw = dict(device=self.device, dtype=torch.float32)
        out = torch.empty(n, self.image_size, **kw) if want_images else None
        ml = torch.empty(n, 2 * self.z_dim, **kw) if want_latent else None
        ls = torch.empty(2, **kw) if want_losses else None
        check(self.h, lib().gm_cvae_forward(self.g, _ptr(images.contiguous()), IMG_FMTS[fmt], _ptr(y.t), n, _ptr(eps), seed, step,
                                            _ptr(out), _ptr(ml), _ptr(ls), _stream()))
        mu = ml[:, :self.z_dim] if ml is not None else None
        lv = ml[:, self.z_dim:] if ml is not None else None
        return out, mu, lv, ls

    def decode(self, z, labels):
        n = z.shape[0]
        y = self.class_ids(labels, n)
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_cvae_decode(self.g, _ptr(z.contiguous().float()), _ptr(y.t), n, _ptr(out), _stream()))
        return out

    def encoder_forward(self, slot, x, labels):
        """Encoder.forward on slot's buffers: x [n, image_size] fp32, labels [n] -> (mu, log_var) [n, z] fp32"""
        n = x.shape[0]
        y = self.class_ids(labels, n)
        ml = torch.empty(n, 2 * self.z_dim, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_cvae_encoder_forward(self.g, slot, _ptr(x.contiguous()), _ptr(y.t), n, _ptr(ml), _stream()))
        return ml[:, :self.z_dim], ml[:, self.z_dim:]

    def decoder_forward(self, slot, z, labels):
        """Decoder.forward on slot's buffers: z [n, z] fp32, labels [n] -> images [n, image_size] fp32"""
        n = z.shape[0]
        y = self.class_ids(labels, n)
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_cvae_decoder_forward(self.g, slot, _ptr(z.contiguous()), _ptr(y.t), n, _ptr(out), _stream()))
        return out

    def slot_bytes(self):
        """device bytes one encoder slot and one decoder slot hold (allocated on the first per-call use)"""
        K = self.num_classes
        XP, HP, B = (self.image_size + K + 16) // 16 * 16, (self.hidden_dim + 16) // 16 * 16, self.max_batch
        ZP = (self.z_dim + K + 64) // 64 * 64
        return 2 * B * (XP + HP) + 4 * B * 64, 2 * B * (ZP + HP + XP)


def mmd_gaussian(z, p, lam=1.0, want_grad=True):
    """gm_mmd_gaussian on fp32 CUDA tensors z, p [B, Z]: -> (mmd [1] device tensor, dmmd/dz [B, Z] or None)"""
    if z.shape != p.shape or z.dim() != 2:
        raise GmError("mmd_gaussian: z and p must both be [batch, z_dim] (got %s, %s)" % (tuple(z.shape), tuple(p.shape)))
    z, p = z.float().contiguous(), p.float().contiguous()
    out = torch.empty(1, device=z.device, dtype=torch.float32)
    dz = torch.empty_like(z) if want_grad else None
    h = _lib.ctx(z.device.index)
    check(h, lib().gm_mmd_gaussian(h, _ptr(z), _ptr(p), z.shape[0], z.shape[1], float(lam), _ptr(out), _ptr(dz), _stream()))
    return out, dz


class BayesGanEngine(GanEngine):
    """One MLP Bayesian GAN on one GPU: the GAN engine in its Bayes mode (gm_bgan_create), num_g generator samples and
    one discriminator with the NS energies, every net moved by SGHMC (include/gm_b200.h).  params[G] stacks the samples
    [sample 0 | sample 1 | ...], `stride` floats apart, each in GanEngine's G layout; views(G, sample=j) are sample j's
    tensors.  momentum[net] is SGHMC's v (bound in the exp_avg slot); there is no second moment."""

    def __init__(self, image_size=784, hidden_dim=400, z_dim=20, num_g=10, max_batch=64, device=None, precision="bf16"):
        if precision != "bf16":
            raise GmError("the Bayesian GAN engine runs in bf16 only (got precision=%r)" % (precision,))
        if not 1 <= int(num_g) <= 16:
            raise GmError("num_g must be in [1, 16] (got %r)" % (num_g,))
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.image_size, self.hidden_dim, self.z_dim, self.max_batch = image_size, hidden_dim, z_dim, max_batch
        self.variant, self.precision, self.num_g = "ns", precision, int(num_g)
        d = GanDesc(image_size, hidden_dim, z_dim, max_batch, VARIANTS["ns"], OUT_ACTS["sigmoid"], PRECISIONS[precision])
        self.g = C.c_void_p()
        check(self.h, lib().gm_bgan_create(self.h, C.byref(d), self.num_g, C.byref(self.g)))
        self.stride = lib().gm_bgan_g_stride(self.g)
        self.n = [lib().gm_gan_param_count(self.g, G), lib().gm_gan_param_count(self.g, D)]
        kw = dict(device=self.device, dtype=torch.float32)
        self.params = [torch.zeros(n, **kw) for n in self.n]
        self.grads = [torch.zeros(n, **kw) for n in self.n]
        self.momentum = [torch.zeros(n, **kw) for n in self.n]
        self.loss_buf = torch.zeros(2, **kw)
        for net in (G, D):
            check(self.h, lib().gm_gan_bind(self.g, net, _ptr(self.params[net]), _ptr(self.grads[net]),
                                            _ptr(self.momentum[net]), None))
        H, X, Z = hidden_dim, image_size, z_dim
        self.shapes = [[(H, Z), (H,), (X, H), (X,)], [(H, X), (H,), (1, H), (1,)]]

    def views(self, net, flat=None, sample=0):
        """[W1, b1, W2, b2] of D, or of generator sample `sample`, as views into `flat` (default: the parameters)"""
        flat = self.params[net] if flat is None else flat
        if net == G:
            if not 0 <= sample < self.num_g:
                raise GmError("sample %d outside [0, %d)" % (sample, self.num_g))
            flat = flat[sample * self.stride:(sample + 1) * self.stride]
        return GanEngine.views(self, net, flat)

    def load(self, net, tensors, sample=0):
        """Copy [W1, b1, W2, b2] into D or into generator sample `sample` and refresh the bf16 copies."""
        for dst, src in zip(self.views(net, sample=sample), tensors):
            dst.copy_(torch.as_tensor(src, dtype=torch.float32).reshape(dst.shape))
        self.sync_shadows(net)

    def reset_optimizer(self):
        """v <- 0 for both nets (SGHMC's momentum starts at rest)"""
        for m in self.momentum:
            m.zero_()

    def d_grad(self, images, noise=None, fmt="f32", gather_idx=None, batch=None, seed=0, step=0, loss_out=None):
        """U_D and D's gradient; noise [num_g * batch, z] (sample-major) or the device's Philox draw"""
        B = batch if batch is not None else (gather_idx.numel() if gather_idx is not None else images.shape[0])
        dst = self.loss_buf[0] if loss_out is None else loss_out
        check(self.h, lib().gm_bgan_d_grad(self.g, _ptr(images), IMG_FMTS[fmt], _ptr(gather_idx), B, _ptr(noise), int(seed),
                                           int(step), _ptr(dst), _stream()))
        return dst

    def g_grad(self, batch, noise=None, seed=0, step=0, loss_out=None):
        """mean_j U_j and each sample's gradient in its slice of grads[G]"""
        dst = self.loss_buf[1] if loss_out is None else loss_out
        check(self.h, lib().gm_bgan_g_grad(self.g, batch, _ptr(noise), int(seed), int(step), _ptr(dst), _stream()))
        return dst

    def apply(self, net, hp, seed=0, step=0):
        """one SGHMC update of net (hp: _lib.SghmcHP) and the refresh of its operand copies"""
        check(self.h, lib().gm_bgan_apply(self.g, net, C.byref(hp), int(seed), int(step), _stream()))

    def sghmc_noise(self, net, seed, step):
        """the xi apply(net, seed=seed, step=step) draws, over the net's whole flat block (tests)"""
        out = torch.empty(self.n[net], device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_bgan_sghmc_noise(self.g, net, int(seed), int(step), _ptr(out), _stream()))
        return out

    def generate(self, sample, noise):
        """Generator.forward of sample `sample`: noise [n, z] -> images [n, image_size]"""
        n = noise.shape[0]
        out = torch.empty(n, self.image_size, device=self.device, dtype=torch.float32)
        check(self.h, lib().gm_bgan_generate(self.g, int(sample), _ptr(noise.contiguous().float()), n, _ptr(out), _stream()))
        return out

    supports_custom_loss = False
    supports_custom_g = False
