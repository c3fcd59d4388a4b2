"""DcganEngine — NSGAN train step with DCGAN convolutional G / D (BASELINE configs[4]: 64x64x3 images, batch 8192
per GPU, data-parallel gradient all-reduce) on the sm_90a kernels of libgm_b200.so.

The reference has no convolutional model: its README recommends DCGAN (README.md:68) and lists it as To-Do
(README.md:96).  What is kept from the reference is the Trainer contract (src/ns_gan.py:94-216): train_D / train_G
with the non-saturating losses, D(images) and D(G(z)) as separate forward calls, Adam on G and on D, flattened
[B, image_size] images at the class boundary (src/ns_gan.py:222-226).  The architecture is the DCGAN of the paper the
README cites (Radford et al. 2015) with the reference's sigmoid outputs:

  G: z -> ConvT(z, 8h, 4, 1, 0) BN ReLU -> ConvT(8h, 4h, 4, 2, 1) BN ReLU -> ConvT(4h, 2h) BN ReLU -> ConvT(2h, h) BN ReLU
       -> ConvT(h, 3, 4, 2, 1) -> sigmoid                                   [B, 64, 64, 3]
  D: Conv(3, h, 4, 2, 1) LeakyReLU(0.2) -> Conv(h, 2h) BN LReLU -> Conv(2h, 4h) BN LReLU -> Conv(4h, 8h) BN LReLU
       -> Conv(8h, 1, 4, 1, 0) -> sigmoid                                   [B, 1]

variant="wgp" (WGAN-GP, src/w_gp_gan.py:177-239) trains D as a critic without BatchNorm — LeakyReLU on conv 1-4, output
relu(s) (src/w_gp_gan.py:61) or s (d_out_act="none") — and adds the gradient penalty at x_hat = eps x + (1 - eps) G(z),
whose double backward is closed form because the critic is piecewise linear (wgp_critic_grad, DESIGN.md §6b).  variant="dra"
(DRAGAN, src/dra_gan.py:174-225) trains the same critic with a sigmoid output and the penalty at x_hat around the real data
(dra_critic_grad); "ra" and "fisher" (src/ra_gan.py:204-205, src/fisher_gan.py:214-223) keep the batch-norm D and run
their batch statistics in separate loss passes that stats_reduce can sum over data-parallel ranks.  variant="be" (BEGAN,
src/be_gan.py:212-258) makes D an autoencoder: the D trunk above with a linear embed_dim-wide conv 5 as the encoder, the
generator stack with a linear output as the decoder, L1 reconstruction losses (gm_l1_rows) and K and the plateau scheduler
as device state (be_state, gm_began_control).  variant="info" (InfoGAN, src/info_gan.py:130-325) feeds G [z | one-hot |
continuous code] drawn on the device (gm_info_noise_rows) and adds Q, a second D trunk with a linear code head, trained with
G by the MI step (q_grad, gm_info_loss_rows) and MI_optimizer's own Adam state for G (apply_mi).  variant="vae" (the VAE
of src/vae.py:47-212 with conv nets) makes D the encoder - the D trunk with a linear head of 2 z outputs, mu then log_var -
and G the decoder; vae_grad runs compute_batch + (recon + kl).backward() with the reparameterisation and KL
(gm_vae_latent_rows, gm_vae_dlatent_rows) and the sum of squared errors through the sigmoid output (gm_sse_sigmoid_rows) on
the device, and train=False forwards (model.eval()) run every BatchNorm on its running statistics (gm_bn_forward_eval).
variant="ae" (the autoencoder of src/ae.py:38-160) is that encoder with one linear head of z outputs and the code relu(h)
in place of the reparameterisation (gm_ae_latent_rows, gm_ae_dlatent_rows), the same decoder and loss (ae_grad).  The row
losses mm, w, ls and f_* take LSGAN's targets ls_a, ls_b, ls_c from the engine (gm_loss_rows_c).

Everything on the device is NHWC bf16 as row-major matrices [B*H*W, C]: a convolution is gm_im2col_k4s2 + one wgmma
GEMM (gm_gemm_bf16), a transposed convolution one GEMM + gm_col2im_k4s2, BatchNorm / activations are gm_bn_* over the
same matrices, the loss is the MLP path's loss kernel on the conv D's logits (gm_loss_rows), Adam is gm_adam_step.
This module only sequences those C-ABI calls and owns the buffers (host language of the reference: Python).
Weights are kept in GEMM layout — conv [Cout, (kh, kw, ci)], transposed conv [(kh, kw, co), Cin] — and converted to /
from torch's Conv2d / ConvTranspose2d layouts at the state_dict boundary (torch_weights / load_torch_weights / torch_grads).
"""
import ctypes as C

import torch

from . import _lib
from ._lib import GmError, OUT_ACTS, VARIANTS, check, lib, _ptr, _stream, gemm_bf16, adam_step

SLOPE = 0.2
BN_EPS = 1e-5
BN_MOMENTUM = 0.1
ACT_NONE, ACT_RELU, ACT_LRELU = 0, 1, 2
C2I_NONE, C2I_SIGMOID, C2I_LRELU_GRAD, C2I_SIGMOID_GRAD = 0, 1, 2, 3


def _im2col(x, B, H, W, Cc, col):
    h = _lib.ctx()
    check(h, lib().gm_im2col_k4s2(h, _ptr(x), B, H, W, Cc, x.stride(0), _ptr(col), col.stride(0), _stream()))


def _col2im(col, B, Hi, Wi, Cc, y, mode=C2I_NONE, aux=None):
    h = _lib.ctx()
    check(h, lib().gm_col2im_k4s2(h, _ptr(col), col.stride(0), B, Hi, Wi, Cc, _ptr(y), y.stride(0), mode, _ptr(aux),
                                  aux.stride(0) if aux is not None else 0, SLOPE, _stream()))


def _im2col_lrelu_mask(x, B, H, W, Cc, m, col):
    h = _lib.ctx()
    check(h, lib().gm_im2col_k4s2_lrelu_mask(h, _ptr(x), B, H, W, Cc, x.stride(0), _ptr(m), m.stride(0), SLOPE, _ptr(col), col.stride(0),
                                             _stream()))


def _lrelu_mask(x, m, out):
    h = _lib.ctx()
    check(h, lib().gm_lrelu_mask_rows(h, _ptr(x), x.stride(0), _ptr(m), m.stride(0), x.shape[0], x.shape[1], SLOPE, _ptr(out),
                                      out.stride(0), _stream()))


def _bn_fwd(x, gamma, beta, act, y, stats, running):
    h = _lib.ctx()
    check(h, lib().gm_bn_forward(h, _ptr(x), x.shape[0], x.shape[1], x.stride(0), _ptr(gamma), _ptr(beta), BN_EPS, act, SLOPE,
                                 _ptr(y), y.stride(0), _ptr(stats), _ptr(running), BN_MOMENTUM, _stream()))


def _bn_fwd_eval(x, gamma, beta, act, y, running):
    h = _lib.ctx()
    check(h, lib().gm_bn_forward_eval(h, _ptr(x), x.shape[0], x.shape[1], x.stride(0), _ptr(gamma), _ptr(beta), _ptr(running), BN_EPS, act,
                                      SLOPE, _ptr(y), y.stride(0), _stream()))


def _bn_bwd(dy, x, stats, gamma, beta, act, dx, dgb):
    h = _lib.ctx()
    check(h, lib().gm_bn_backward(h, _ptr(dy), _ptr(x), x.shape[0], x.shape[1], x.stride(0), _ptr(stats), _ptr(gamma), _ptr(beta),
                                  act, SLOPE, _ptr(dx), dx.stride(0), _ptr(dgb), _stream()))


class _Net:
    """Flat fp32 master parameters of one network + gradient / Adam state + bf16 GEMM operand copies."""

    def __init__(self, shapes, device):
        self.names = [n for n, _ in shapes]
        self.shapes = dict(shapes)
        self.offsets, off = {}, 0
        for n, shp in shapes:
            cnt = 1
            for s in shp:
                cnt *= s
            self.offsets[n] = (off, cnt)
            off += (cnt + 3) // 4 * 4                         # 16-byte aligned sub-tensors
        self.total = off
        kw = dict(device=device, dtype=torch.float32)
        self.params, self.grads = torch.zeros(off, **kw), torch.zeros(off, **kw)
        self.exp_avg, self.exp_avg_sq = torch.zeros(off, **kw), torch.zeros(off, **kw)
        self.step = 0
        self.bf, self.bf_t = {}, {}
        pad8 = lambda v: (v + 7) // 8 * 8                  # noqa: E731  (TMA rows are 16-byte multiples)
        for n, shp in shapes:
            if len(shp) == 2:
                self.bf[n] = torch.zeros(shp[0], pad8(shp[1]), device=device, dtype=torch.bfloat16)[:, :shp[1]]
                self.bf_t[n] = torch.zeros(shp[1], pad8(shp[0]), device=device, dtype=torch.bfloat16)[:, :shp[0]]

    def view(self, n, flat=None):
        off, cnt = self.offsets[n]
        return (self.params if flat is None else flat)[off:off + cnt].view(self.shapes[n])

    def refresh(self):
        h = _lib.ctx()
        for n in self.bf:
            w = self.view(n)
            check(h, lib().gm_cast_bf16(h, _ptr(w), w.shape[0], w.shape[1], _ptr(self.bf[n]), self.bf[n].stride(0),
                                        _ptr(self.bf_t[n]), self.bf_t[n].stride(0), _stream()))

    def adam(self, hp, lr_scale=None):
        self.step += 1
        adam_step(self.params, self.grads, self.exp_avg, self.exp_avg_sq, hp, self.step, lr_scale)
        self.refresh()


class DevicePool:
    """A training set held in HBM as one byte per value, batches drawn on the device (DESIGN.md §6b).

    Image datasets hold few distinct values (k/255 from ToTensor, {0, 1} when binarised, (k/255 - 0.5)/0.5 normalised), and
    every value reaches the kernels as bf16.  So a dataset with at most 256 distinct bf16 bit patterns is stored as codes
    [n, 4096 ch] uint8 in NHWC order plus table [256], the bf16 bit patterns as int16: table[codes] is what stage_images makes
    of the images, bit for bit (-0.0 and +0.0 are distinct patterns).  DcganEngine.stage_pool turns rows of the on-device
    Feistel permutation (kernels.cuh: Sampler) into a batch; indices_host evaluates the same permutation on the host."""
    SEED_MIX = 0x5DEECE66D       # sampler seed = the trainer's Philox seed ^ SEED_MIX: the two streams are keyed apart

    def __init__(self, codes, table, channels, batch_size, drop_last, source):
        self.codes, self.table, self.ch = codes, table, channels
        self.n, self.row_vals = codes.shape
        self.batch_size, self.drop_last, self._source = batch_size, drop_last, source
        self.num_batches = self.n // batch_size if drop_last else -(-self.n // batch_size)

    def __len__(self):
        return self.num_batches

    @staticmethod
    def pack(images, channels, device=None, chunk_rows=4096):
        """images [n, ch*64*64] (NCHW flattened) or [n, ch, 64, 64] -> (codes [n, 4096 ch] uint8 NHWC, table [256] int16),
        or None when the bf16 values hold more than 256 distinct bit patterns.  The values become bf16 as process_batch +
        stage_images make them (.float(), then bf16).  Runs chunk by chunk on `device` (default: the images' own)."""
        n = images.shape[0]
        dev = images.device if device is None else torch.device(device)

        def bits(i):                                   # the chunk's bf16 bit patterns in NHWC order, int32
            c = images[i:i + chunk_rows].to(dev, non_blocking=True).float().reshape(-1, channels, 64, 64)
            return c.permute(0, 2, 3, 1).to(torch.bfloat16).contiguous().view(torch.int16).to(torch.int32).reshape(c.shape[0], -1)

        uniq = torch.empty(0, dtype=torch.int32, device=dev)
        for i in range(0, n, chunk_rows):
            uniq = torch.unique(torch.cat([uniq, torch.unique(bits(i))]))
            if uniq.numel() > 256:
                return None
        codes = torch.empty(n, 4096 * channels, dtype=torch.uint8, device=dev)
        for i in range(0, n, chunk_rows):
            codes[i:i + chunk_rows] = torch.searchsorted(uniq, bits(i)).to(torch.uint8)
        table = torch.zeros(256, dtype=torch.int16, device=dev)
        table[:uniq.numel()] = uniq.to(torch.int16)
        return codes, table

    @staticmethod
    def from_loader(loader, channels, cached=None, budget=None):
        """A pool of loader's images, or None when the loader is not eligible (the caller then keeps the host path): a
        DataLoader over a TensorDataset whose first tensor holds 64*64*channels values per row, drawn by a RandomSampler
        without replacement over the whole dataset, with at most 256 distinct bf16 values and codes within `budget` bytes
        (default: half the free device memory).  `cached`, the pool of an earlier train() call, is returned while the loader
        serves the same tensor with the same batch size and drop_last."""
        from torch.utils.data import DataLoader, RandomSampler, TensorDataset
        if not isinstance(loader, DataLoader) or not isinstance(loader.dataset, TensorDataset) or loader.batch_size is None:
            return None
        smp = loader.sampler
        if type(smp) is not RandomSampler or smp.replacement or smp._num_samples is not None:
            return None
        images = loader.dataset.tensors[0]
        n = images.shape[0]
        if n == 0 or n > 0x7FFFFFFF or images.numel() != n * 4096 * channels:
            return None
        if cached is not None and cached._source is images and cached.batch_size == loader.batch_size and \
                cached.drop_last == loader.drop_last and cached.ch == channels:
            return cached
        if budget is None:
            budget = torch.cuda.mem_get_info()[0] // 2
        if n * 4096 * channels > budget:
            return None
        dev = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else images.device
        packed = DevicePool.pack(images, channels, dev)
        if packed is None:
            return None
        return DevicePool(packed[0], packed[1], channels, loader.batch_size, loader.drop_last, images)

    def indices_host(self, seed, round, offset, count):
        """the pool rows perm_{seed,round}(offset + r), r < count, that gm_stage_pool_rows draws (int64 CPU tensor)"""
        out = (C.c_int * count)()
        rc = lib().gm_sampler_indices_host(self.n, int(seed), int(round), int(offset), int(count), out)
        if rc != 0:
            raise GmError("gm_sampler_indices_host: bad argument (rc=%d)" % rc)
        return torch.tensor(list(out), dtype=torch.int64)


class DcganEngine:
    """One DCGAN (64x64xchannels images) on one GPU; see the module docstring."""

    def __init__(self, hidden_dim=64, z_dim=100, channels=3, variant="ns", device=None, d_out_act=None, embed_dim=None, disc_dim=None,
                 cont_dim=None):
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        if hidden_dim % 16 or hidden_dim <= 0:
            raise GmError("hidden_dim (the base channel width) must be a positive multiple of 16")
        if variant not in ("ns", "mm", "w", "ls", "wgp", "ra", "fisher", "dra", "be", "info", "vae", "ae") and not variant.startswith("f_"):
            raise GmError("the conv path supports the row-wise losses (ns, mm, w, ls, f_*), ra, fisher, wgp, dra, be, info, vae and ae")
        if embed_dim is not None and (variant != "be" or embed_dim <= 0):
            raise GmError("embed_dim is the positive embedding width of BEGAN's autoencoder D (variant='be')")
        if variant == "info":
            disc_dim, cont_dim = 10 if disc_dim is None else int(disc_dim), 10 if cont_dim is None else int(cont_dim)
            if disc_dim < 1 or cont_dim < 1:
                # the reference's cross entropy / MSE over zero codes is NaN (src/info_gan.py:295-299)
                raise GmError("InfoGAN needs disc_dim >= 1 and cont_dim >= 1")
        elif disc_dim is not None or cont_dim is not None:
            raise GmError("disc_dim and cont_dim are the code widths of InfoGAN (variant='info')")
        if variant in ("vae", "ae"):
            # the VAE's encoder ends in the linear mu / log_var heads (src/vae.py:55-61), the autoencoder's in the linear layer
            # that its ReLU code follows (src/ae.py:38-39)
            if d_out_act is not None:
                raise GmError("the %s encoder's head is linear; d_out_act is a discriminator option" % variant.upper())
            d_out_act = "none"
        elif variant == "be":
            # BEGAN's D is an autoencoder whose reconstruction is linear (src/be_gan.py:73-76)
            if d_out_act not in (None, "none"):
                raise GmError("the BEGAN autoencoder's output is linear (d_out_act='none')")
            d_out_act = "none"
        elif variant == "wgp":
            # WGAN-GP critic: no BatchNorm (one sample's input gradient must not depend on the batch, WGAN-GP paper §4),
            # output relu(s) as src/w_gp_gan.py:61 or the linear s
            d_out_act = "relu" if d_out_act is None else d_out_act
            if d_out_act not in ("relu", "none"):
                raise GmError("the WGAN-GP conv critic's output is relu or none")
        elif d_out_act not in (None, "sigmoid"):
            raise GmError("the conv discriminator of the %s loss ends in a sigmoid" % variant)
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.hd, self.z, self.ch, self.variant = hidden_dim, z_dim, channels, variant
        self.d_out_act = d_out_act or "sigmoid"
        self.d_bn = variant not in ("wgp", "dra")                # BatchNorm in D's layers 2-4; the penalised critics have none
        self.gp_lambda = 10.0                                    # LAMBDA of src/w_gp_gan.py:177, src/dra_gan.py:174
        self.gp_k, self.dra_c = 1.0, 1.0                         # K, C of src/dra_gan.py:174
        self.ls_a, self.ls_b, self.ls_c = 0.0, 1.0, 1.0          # LSGAN's targets a, b, c (src/ls_gan.py:173,197)
        self.fisher = torch.tensor([0.0, 1e-6], device=self.device)   # Fisher's (LAMBDA, RHO), src/fisher_gan.py:117-118
        # stats_reduce(buf): SUM a float64 statistic buffer over the data-parallel ranks in place (RaNS / Fisher loss
        # moments, DRAGAN's image std, BEGAN's L1 sums); None on one process.  stat_batch (d_grad) is then the global batch.
        self.stats_reduce = None
        # InfoGAN: G's input is [z | one-hot (nd) | continuous code (nc)] (src/info_gan.py:51,325); zin = G's input width
        self.nd, self.nc = (disc_dim, cont_dim) if variant == "info" else (0, 0)
        self.zin = z_dim + self.nd + self.nc
        self.zp = (self.zin + 1 + 7) // 8 * 8                    # noise rows: [z | 1 | pad], 16-byte rows
        hd = hidden_dim
        self.gc = [8 * hd, 4 * hd, 2 * hd, hd, channels]        # generator channels after each layer
        self.dc = [hd, 2 * hd, 4 * hd, 8 * hd]                  # discriminator channels after conv 1..4
        def g_stack(pfx, zin):                                   # the generator's transposed-conv stack on zin input columns
            out = [(pfx + "l1.weight", (16 * self.gc[0], zin))]
            for i in range(1, 5):
                out.append((pfx + "l%d.weight" % (i + 1), (16 * self.gc[i], self.gc[i - 1])))
            for i in range(4):
                out += [(pfx + "bn%d.weight" % (i + 1), (self.gc[i],)), (pfx + "bn%d.bias" % (i + 1), (self.gc[i],))]
            return out

        def d_stack(pfx, nout):                                  # the discriminator's conv stack with nout output rows
            out = [(pfx + "l1.weight", (self.dc[0], 16 * channels))]
            for i in range(1, 4):
                out.append((pfx + "l%d.weight" % (i + 1), (self.dc[i], 16 * self.dc[i - 1])))
            out.append((pfx + "l5.weight", (nout, 16 * self.dc[3])))
            for i in range(1, 4) if self.d_bn else ():
                out += [(pfx + "bn%d.weight" % (i + 1), (self.dc[i],)), (pfx + "bn%d.bias" % (i + 1), (self.dc[i],))]
            return out

        self.e = z_dim if embed_dim is None else int(embed_dim)  # BEGAN's embedding width (N_h = N_z in the BEGAN paper)
        self.ep = (self.e + 15) // 16 * 16                       # embedding rows: [e | 0 pad], N of a bf16-output GEMM
        # encoder head rows, the N of the fp32 row-major head GEMM: VAE [mu | log_var | 0 pad], autoencoder [h | 0 pad]
        self.mp = ((z_dim if variant == "ae" else 2 * z_dim) + 15) // 16 * 16
        if variant == "be":
            # D = encoder (the DCGAN D trunk, l5: e outputs, zero-padded to ep rows) + decoder (the generator stack with e
            # in place of z, l1's input columns zero-padded to ep); the torch views trim the padding (_TRIM)
            self._trim = {"D.encoder.l5.weight": self.e, "D.decoder.l1.weight": self.e}
            d_shapes = d_stack("encoder.", self.ep) + g_stack("decoder.", self.ep)
        elif variant == "vae":
            # the VAE's encoder: l5 is the mu head (rows [0, z)) stacked on the log_var head (rows [z, 2z)), zero-padded to mp
            # rows (the N of the fp32 row-major head GEMM)
            self._trim = {"D.l5.weight": 2 * z_dim}
            d_shapes = d_stack("", self.mp)
        elif variant == "ae":
            # the autoencoder's encoder: l5 is the linear head of z outputs, zero-padded to mp rows
            self._trim = {"D.l5.weight": z_dim}
            d_shapes = d_stack("", self.mp)
        else:
            self._trim = {"D.l5.weight": 1}
            d_shapes = d_stack("", 16)                           # 1 real output channel (row 0), padded to the MMA's N = 16
        self.G, self.D = _Net(g_stack("", self.zin), self.device), _Net(d_shapes, self.device)
        self.run_G = {i: torch.zeros(2, self.gc[i], device=self.device) for i in range(4)}
        self.run_D = {i: torch.zeros(2, self.dc[i], device=self.device) for i in range(1, 4) if self.d_bn}
        self.run_dec = {i: torch.zeros(2, self.gc[i], device=self.device) for i in range(4)} if variant == "be" else {}
        # InfoGAN's Q (src/info_gan.py:78-94): its own D trunk (BatchNorm on conv 2-4) and a linear conv 5 with nd + nc
        # outputs, zero-padded to qp rows (the N of the fp32 row-major head GEMM); MI_optimizer's own Adam moments for G
        self.Q, self.run_Q, self.qp = None, {}, 0
        if variant == "info":
            self.qp = (self.nd + self.nc + 15) // 16 * 16
            self._trim["Q.l5.weight"] = self.nd + self.nc
            self.Q = _Net(d_stack("", self.qp), self.device)
            self.run_Q = {i: torch.zeros(2, self.dc[i], device=self.device) for i in range(1, 4)}
            self.g_mi_avg, self.g_mi_avg_sq = torch.zeros_like(self.G.params), torch.zeros_like(self.G.params)
            self.mi_loss = torch.zeros(1, device=self.device)
            self.codes_ = {}
        for r in list(self.run_G.values()) + list(self.run_D.values()) + list(self.run_dec.values()) + list(self.run_Q.values()):
            r[1].fill_(1.0)
        self.loss_buf = torch.zeros(4, device=self.device)      # [D loss, G loss, loss-kernel scratch (sum ds, ..)]
        # BEGAN's device state, the layout of gm_gan_began_state: [K, inv_b, -K inv_b, DX, DG, plateau best, plateau bad
        # count, lr scale, inv_b, inv_b, convergence]; the conv path passes its gradient scales per call ([1], [2], [8], [9] unused)
        self.be_state = torch.zeros(11, device=self.device)
        if variant == "be":
            self.began_init(0.0, 1)
        self.vae_loss = torch.zeros(2, device=self.device)       # VAE: (recon, kl) of the last vae_grad, this process's sums
        self.ae_loss = torch.zeros(1, device=self.device)        # autoencoder: recon of the last ae_grad, this process's sum
        self._bufs = {}
        self._calls = {"d": 0, "g": 0}                           # custom_d_forward / custom_g_forward calls so far
        self._slot_gen = {"d": [0] * self.D_SLOTS, "g": [0] * self.G_SLOTS}   # the call that holds each slot
        self.init_weights()

    # ------------------------------------------------------------------ parameters
    def init_weights(self, seed=1234):
        """DCGAN initialisation (N(0, 0.02) conv weights, N(1, 0.02) BN scale, zero BN shift)."""
        g = torch.Generator().manual_seed(seed)
        for net in self.nets():
            for n in net.names:
                v = net.view(n)
                if n.endswith("bias"):
                    v.zero_()
                elif n.split(".")[-2].startswith("bn"):
                    v.copy_(1.0 + 0.02 * torch.randn(v.shape, generator=g))
                else:
                    v.copy_(0.02 * torch.randn(v.shape, generator=g))
        self.zero_padding()
        for net in self.nets():
            net.refresh()

    def nets(self):
        """G, D and (InfoGAN) Q"""
        return (self.G, self.D) if self.Q is None else (self.G, self.D, self.Q)

    def zero_padding(self):
        """zero the padding of D's padded weights (the 1-channel output layer's rows 1..15; BEGAN's embedding rows / columns
        beyond e; InfoGAN's Q head rows beyond nd + nc; the VAE encoder's head rows beyond 2 z): their gradients are then zero,
        so they stay zero and the padded GEMM columns read zeros"""
        if self.variant == "be":
            self.D.view("encoder.l5.weight")[self.e:].zero_()
            self.D.view("decoder.l1.weight")[:, self.e:].zero_()
        else:
            self.D.view("l5.weight")[self._trim["D.l5.weight"]:].zero_()
        if self.Q is not None:
            self.Q.view("l5.weight")[self.nd + self.nc:].zero_()

    def _torch_views(self, which):
        """{torch-style name: view of the G / D tensor in torch's layout} over the flat params (which="params"), grads
        (which="grads") or, for which = {"G" / "D" / "Q": flat buffer in that net's layout}, over those buffers only.
        Conv weights are [Cout, (kh, kw, ci)] here and [Cout, Cin, kh, kw] in torch; transposed-conv weights (G, BEGAN's
        decoder) are [(kh, kw, co), Cin] here and [Cin, Cout, kh, kw] in torch; BatchNorm vectors match.  Padded weights are
        trimmed on torch's dim 0 (_trim: D.l5 keeps output channel 0 of its 16 rows, BEGAN's encoder l5 / decoder l1 the e
        embedding channels, InfoGAN's Q.l5 its nd + nc code outputs)."""
        out = {}
        for tag, net in zip("GDQ", self.nets()):
            flat = which.get(tag) if isinstance(which, dict) else getattr(net, which)
            if flat is None:
                continue
            for n in net.names:
                w = net.view(n, flat)
                key = "%s.%s" % (tag, n)
                if n.split(".")[-2].startswith("l"):
                    if tag == "G" or n.startswith("decoder."):
                        w = w.view(4, 4, w.shape[0] // 16, w.shape[1]).permute(3, 2, 0, 1)
                    else:
                        w = w.view(w.shape[0], 4, 4, w.shape[1] // 16).permute(0, 3, 1, 2)
                    w = w[:self._trim[key]] if key in self._trim else w
                out[key] = w
        return out

    def torch_weights(self):
        """{torch-style name: tensor in torch's Conv2d / ConvTranspose2d / BatchNorm2d layout} (CPU fp32)."""
        return {k: v.detach().cpu().contiguous() for k, v in self._torch_views("params").items()}

    def torch_grads(self):
        """{torch-style name: the current G / D (/ Q) gradient in torch's layout} (views of the device gradients)."""
        return self._torch_views("grads")

    def load_torch_weights(self, sd):
        for k, v in self._torch_views("params").items():
            v.copy_(sd[k].float())
        for net in self.nets():
            net.refresh()

    def _buf(self, key, rows, cols, dtype=torch.bfloat16):
        t = self._bufs.get(key)
        if t is None or t.shape[0] < rows or t.shape[1] != cols:
            t = torch.empty(rows, cols, device=self.device, dtype=dtype)
            self._bufs[key] = t
        return t[:rows]

    # ------------------------------------------------------------------ generator
    def g_forward(self, n, noise=None, seed=0, stream_id=0, tag="g", net=None, pfx="", x_rows=None, out_mode=C2I_SIGMOID, run=None,
                  train=True):
        """G(z) for n samples -> (images [n*4096, ch] NHWC bf16, saved activations).  The same transposed-conv stack runs
        BEGAN's decoder: net / pfx name its weights (default G), x_rows [n, >= K] bf16 are its input rows instead of the
        noise rows, out_mode is the final col2im's (C2I_NONE: linear output) and run its BatchNorm running statistics.
        InfoGAN without caller noise draws [z | one-hot | continuous] on the device (gm_info_noise_rows); its fp32 copy, the
        MI loss's targets, is left in self.codes_[tag].  train=False (inference mode, the VAE's model.eval()) normalises with the
        running statistics and leaves them unchanged; its activations are not for g_backward."""
        net = self.G if net is None else net
        run = self.run_G if run is None else run
        K = net.shapes[pfx + "l1.weight"][1]
        if x_rows is None:
            x_rows = self._buf(tag + "z", n, self.zp)
            if self.variant == "info" and noise is None:
                codes = self.codes_[tag] = self._buf(tag + "codes", n, self.zin, torch.float32)
                check(self.h, lib().gm_info_noise_rows(self.h, _ptr(x_rows), self.zp, _ptr(codes), n, self.z, self.nd, self.nc, int(seed),
                                                       int(stream_id), _stream()))
            else:
                check(self.h, lib().gm_noise_rows(self.h, _ptr(noise), _ptr(x_rows), n, self.zin, self.zp, int(seed), int(stream_id),
                                                  _stream()))
        sv = {"z": x_rows, "n": n}
        gc = self.gc
        c = self._buf(tag + "c0", n, 16 * gc[0])
        gemm_bf16(x_rows, net.bf[pfx + "l1.weight"], c, "nt", K=K)                          # [n, (kh,kw,co)] = NHWC [n*16, 8h]
        x = c.view(n * 16, gc[0])
        hw = 4
        for i in range(4):
            a = self._buf(tag + "a%d" % i, x.shape[0], gc[i])
            st = self._buf(tag + "st%d" % i, 2, gc[i], torch.float32)
            if train:
                _bn_fwd(x, net.view(pfx + "bn%d.weight" % (i + 1)), net.view(pfx + "bn%d.bias" % (i + 1)), ACT_RELU, a, st, run[i])
            else:
                _bn_fwd_eval(x, net.view(pfx + "bn%d.weight" % (i + 1)), net.view(pfx + "bn%d.bias" % (i + 1)), ACT_RELU, a, run[i])
            sv["c%d" % i], sv["a%d" % i], sv["st%d" % i] = x, a, st
            col = self._buf(tag + "col%d" % i, a.shape[0], 16 * gc[i + 1])
            gemm_bf16(a, net.bf[pfx + "l%d.weight" % (i + 2)], col, "nt")
            y = self._buf(tag + "c%d" % (i + 1), n * 4 * hw * hw, gc[i + 1])
            _col2im(col, n, hw, hw, gc[i + 1], y, out_mode if i == 3 else C2I_NONE)
            x, hw = y, 2 * hw
        sv["img"] = x
        return x, sv

    def g_backward(self, sv, dpre, net=None, pfx="", grads=None, need_wgrad=True, need_dx=False, tag="g", dx_dtype=torch.bfloat16):
        """dpre [n*4096, ch] = dL/d(pre-sigmoid output) -> flat G gradient (self.G.grads, zeroed first).  For BEGAN's decoder
        (net / pfx, see g_forward) dpre is dL/d(linear output) and the weight gradients go to the flat D-layout `grads` when
        need_wgrad; need_dx returns dL/d(input rows) [n, K] (K = l1's input columns) instead, bf16 (BEGAN's embedding
        gradient) or dx_dtype=torch.float32 (the VAE's dL/dz) (one more GEMM, with l1's transposed copy)."""
        n, gc = sv["n"], self.gc
        net = self.G if net is None else net
        if grads is None and need_wgrad:
            grads = net.grads
            grads.zero_()
        d, hw = dpre, 64
        for i in range(3, -1, -1):
            hw //= 2                                                                      # input grid of transposed conv i+2
            a, c, st = sv["a%d" % i], sv["c%d" % i], sv["st%d" % i]
            dcol = self._buf("gdcol%d" % i, a.shape[0], 16 * gc[i + 1])
            _im2col(d, n, 2 * hw, 2 * hw, gc[i + 1], dcol)                                # gradient of col2im
            if need_wgrad:
                gemm_bf16(dcol, a, net.view(pfx + "l%d.weight" % (i + 2), grads), "tn")   # [16 Cout, Cin] = dcol^T a
            da = self._buf("gda%d" % i, a.shape[0], gc[i])
            gemm_bf16(dcol, net.bf_t[pfx + "l%d.weight" % (i + 2)], da, "nt")             # da = dcol Wm
            dc = self._buf("gdc%d" % i, a.shape[0], gc[i])
            dgb = self._buf("gdgb%d" % i, 2, gc[i], torch.float32)
            _bn_bwd(da, c, st, net.view(pfx + "bn%d.weight" % (i + 1)), net.view(pfx + "bn%d.bias" % (i + 1)), ACT_RELU, dc, dgb)
            if need_wgrad:
                net.view(pfx + "bn%d.bias" % (i + 1), grads).copy_(dgb[0])
                net.view(pfx + "bn%d.weight" % (i + 1), grads).copy_(dgb[1])
            d = dc
        w1 = pfx + "l1.weight"
        if need_wgrad:
            gemm_bf16(d.view(n, 16 * gc[0]), sv["z"], net.view(w1, grads), "tn", N=net.shapes[w1][1])   # [(kh,kw,co), z]
        if not need_dx:
            return grads
        dx = self._buf(tag + ("dx" if dx_dtype == torch.bfloat16 else "dx32"), n, net.shapes[w1][1], dx_dtype)
        gemm_bf16(d.view(n, 16 * gc[0]), net.bf_t[w1], dx, "nt")                             # [n, ep] = d Wm
        return dx

    # ------------------------------------------------------------------ discriminator
    def d_forward(self, img, n, logits, tag, pfx="", net=None, run=None, train=True):
        """D(img) for n NHWC images; logits: fp32 view [16, ld] (row 0 receives the n logits), or a bf16 [n, ep] buffer that
        receives BEGAN's linear embedding (pfx "encoder.").  The same trunk runs InfoGAN's Q: net / run name its weights and
        BatchNorm running statistics (default D's), and Q's head writes fp32 rows [n, qp] into logits; the VAE encoder's head
        writes fp32 rows [n, mp].  train=False (the VAE's model.eval()) normalises with the running statistics and leaves them
        unchanged.  Returns saved activations."""
        dc = self.dc
        net = self.D if net is None else net
        run = self.run_D if run is None else run
        sv = {"n": n, "img": img}
        x, hw, cin = img, 64, self.ch
        for i in range(4):
            hw //= 2
            col = self._buf(tag + "col%d" % i, n * hw * hw, 16 * cin)
            _im2col(x, n, 2 * hw, 2 * hw, cin, col)
            c = self._buf(tag + "c%d" % i, n * hw * hw, dc[i])
            sv["col%d" % i] = col
            if i == 0 or not self.d_bn:
                gemm_bf16(col, net.bf[pfx + "l%d.weight" % (i + 1)], c, "nt", act=3, act_slope=SLOPE)   # conv + LeakyReLU epilogue
                y = c
            else:
                gemm_bf16(col, net.bf[pfx + "l%d.weight" % (i + 1)], c, "nt")
                y = self._buf(tag + "y%d" % i, c.shape[0], dc[i])
                st = self._buf(tag + "st%d" % i, 2, dc[i], torch.float32)
                if train:
                    _bn_fwd(c, net.view(pfx + "bn%d.weight" % (i + 1)), net.view(pfx + "bn%d.bias" % (i + 1)), ACT_LRELU, y, st, run[i])
                else:
                    _bn_fwd_eval(c, net.view(pfx + "bn%d.weight" % (i + 1)), net.view(pfx + "bn%d.bias" % (i + 1)), ACT_LRELU, y, run[i])
                sv["c%d" % i], sv["st%d" % i] = c, st
            sv["y%d" % i] = y
            x, cin = y, dc[i]
        flat = x.view(n, 16 * dc[3])
        sv["flat"] = flat
        # D: fp32 [16, ld] with row 0 = logits (transposed store); Q and the VAE encoder: fp32 rows [n, qp] / [n, mp]; BEGAN:
        # the bf16 embedding rows [n, ep]
        gemm_bf16(flat, net.bf[pfx + "l5.weight"], logits, "nt",
                  transpose=logits.dtype == torch.float32 and net is not self.Q and self.variant not in ("vae", "ae"))
        return sv

    def d_backward(self, sv, ds, grads, need_wgrad=True, need_dimg=False, tag="d", pfx="", dimg_mode=C2I_SIGMOID_GRAD, net=None):
        """ds [n] fp32 = dL/dlogit, or a bf16 [n, ep] upstream gradient of BEGAN's embedding (pfx "encoder.") or of InfoGAN's
        Q head (net = self.Q, [n, qp]).  Accumulates nothing: writes this pass's D (Q) gradient into `grads` (flat, that net's
        layout) when need_wgrad; returns dL/d(pre-sigmoid generator output) (dimg_mode C2I_SIGMOID_GRAD) or dL/d(image)
        (C2I_NONE) when need_dimg."""
        n, dc, D = sv["n"], self.dc, self.D if net is None else net
        if ds.dtype == torch.bfloat16:
            dy5 = ds
        else:
            dy5 = self._buf(tag + "dy5", n, 16)
            check(self.h, lib().gm_pack_col0(self.h, _ptr(ds), n, _ptr(dy5), 16, _stream()))
        if need_wgrad:
            gemm_bf16(dy5, sv["flat"], D.view(pfx + "l5.weight", grads), "tn")            # [16 (ep), 128h]
        if not self.d_bn:
            betas = self._betas(sv, dy5, tag)
            if need_wgrad:
                for i in range(4):
                    gemm_bf16(betas[i], sv["col%d" % i], D.view("l%d.weight" % (i + 1), grads), "tn")
            return self._dimg(sv, betas[0], tag, dimg_mode) if need_dimg else None
        dflat = self._buf(tag + "dflat", n, 16 * dc[3])
        gemm_bf16(dy5, D.bf_t[pfx + "l5.weight"], dflat, "nt", K=dy5.shape[1])
        d, hw = dflat.view(n * 16, dc[3]), 4
        for i in range(3, 0, -1):
            c, st, col = sv["c%d" % i], sv["st%d" % i], sv["col%d" % i]
            dcv = self._buf(tag + "dc%d" % i, c.shape[0], dc[i])
            dgb = self._buf(tag + "dgb%d" % i, 2, dc[i], torch.float32)
            _bn_bwd(d, c, st, D.view(pfx + "bn%d.weight" % (i + 1)), D.view(pfx + "bn%d.bias" % (i + 1)), ACT_LRELU, dcv, dgb)
            if need_wgrad:
                D.view(pfx + "bn%d.bias" % (i + 1), grads).copy_(dgb[0])
                D.view(pfx + "bn%d.weight" % (i + 1), grads).copy_(dgb[1])
                gemm_bf16(dcv, col, D.view(pfx + "l%d.weight" % (i + 1), grads), "tn")    # [Cout, 16 Cin]
            dcol = self._buf(tag + "dcol%d" % i, col.shape[0], col.shape[1])
            gemm_bf16(dcv, D.bf_t[pfx + "l%d.weight" % (i + 1)], dcol, "nt")
            dprev = self._buf(tag + "dprev%d" % i, n * 4 * hw * hw, dc[i - 1])
            # layer i's input is y_{i-1}: a BN layer's output (its backward applies LeakyReLU') or, for i == 1, lrelu(c_0)
            _col2im(dcol, n, hw, hw, dc[i - 1], dprev, C2I_LRELU_GRAD if i == 1 else C2I_NONE, sv["y0"] if i == 1 else None)
            d, hw = dprev, 2 * hw
        if need_wgrad:
            gemm_bf16(d, sv["col0"], D.view(pfx + "l1.weight", grads), "tn")              # [h, 16 ch]
        if not need_dimg:
            return None
        return self._dimg(sv, d, tag, dimg_mode, pfx, D)

    def _dimg(self, sv, d, tag, mode=C2I_SIGMOID_GRAD, pfx="", net=None):
        """d = dL/d(conv 1 output) -> dL/d(image) (mode C2I_NONE) or dL/d(pre-sigmoid generator output) (C2I_SIGMOID_GRAD)"""
        n = d.shape[0] // 1024
        net = self.D if net is None else net
        dcol = self._buf(tag + "dcol0", d.shape[0], 16 * self.ch)
        gemm_bf16(d, net.bf_t[pfx + "l1.weight"], dcol, "nt")
        dpre = self._buf(tag + ("dpre" if mode == C2I_SIGMOID_GRAD else "dimg"), n * 4096, self.ch)
        _col2im(dcol, n, 32, 32, self.ch, dpre, mode, sv["img"] if mode == C2I_SIGMOID_GRAD else None)
        return dpre

    def _betas(self, sv, dy5, tag):
        """Input-gradient chain of the batch-norm-free critic: dy5 [rows, 16] (column 0 = dL/dlogit per image) -> the
        pre-activation gradients [beta_1, .., beta_4] of conv 1..4 as NHWC rows (beta_l = LReLU'(y_l) * W_{l+1}^T beta_{l+1})."""
        n, dc, D = sv["n"], self.dc, self.D
        dflat = self._buf(tag + "dflat", n, 16 * dc[3])
        gemm_bf16(dy5, D.bf_t["l5.weight"], dflat, "nt", K=16)
        betas = [None, None, None, self._buf(tag + "beta3", n * 16, dc[3])]
        _lrelu_mask(dflat.view(n * 16, dc[3]), sv["y3"], betas[3])
        hw = 4
        for i in range(3, 0, -1):
            col = sv["col%d" % i]
            dcol = self._buf(tag + "dcol%d" % i, col.shape[0], col.shape[1])
            gemm_bf16(betas[i], D.bf_t["l%d.weight" % (i + 1)], dcol, "nt")
            betas[i - 1] = self._buf(tag + "beta%d" % (i - 1), n * 4 * hw * hw, dc[i - 1])
            _col2im(dcol, n, hw, hw, dc[i - 1], betas[i - 1], C2I_LRELU_GRAD, sv["y%d" % (i - 1)])
            hw *= 2
        return betas

    # ------------------------------------------------------------------ the train step (src/ns_gan.py:126-156)
    def _image_arg(self, images):
        """images [n, ch*64*64] or [n, ch, 64, 64] -> fp32 [n, ch*64*64] on the device, contiguous and 16-byte aligned"""
        n = images.shape[0]
        if images.numel() != n * 4096 * self.ch:
            raise GmError("expected %d-channel 64x64 images, got shape %s" % (self.ch, tuple(images.shape)))
        x = images.to(self.device).reshape(n, -1).float().contiguous()
        return x if x.data_ptr() % 16 == 0 else x.clone()

    def image_to_rows(self, images, out_rows=None, dst=None):
        """images (see _image_arg) -> NHWC bf16 rows [n*4096, ch] (gm_image_to_rows): x rounded to bf16, or with out_rows
        (G's stored sigmoid output rows) x * f * (1 - f) rounded once.  dst: the rows to write (default a new tensor)."""
        x = self._image_arg(images)
        n = x.shape[0]
        dst = torch.empty(n * 4096, self.ch, device=self.device, dtype=torch.bfloat16) if dst is None else dst
        check(self.h, lib().gm_image_to_rows(self.h, _ptr(x), _ptr(out_rows), n, self.ch, _ptr(dst), _stream()))
        return dst

    def rows_to_image(self, rows, n):
        """NHWC bf16 rows of n images -> fp32 [n, ch*64*64] (NCHW flattened), exact (gm_rows_to_image)"""
        out = torch.empty(n, 4096 * self.ch, device=self.device)
        check(self.h, lib().gm_rows_to_image(self.h, _ptr(rows), n, self.ch, _ptr(out), _stream()))
        return out

    def stage_images(self, images):
        """[n, ch*64*64] flat (the reference's process_batch layout: NCHW flattened, src/ns_gan.py:225) or
        [n, ch, 64, 64] -> NHWC bf16 rows [n*4096, ch]."""
        return self.image_to_rows(images)

    def stage_pool(self, pool, n, seed, round, offset=0, idx_out=None):
        """n images of a DevicePool drawn on the device -> NHWC bf16 rows [n*4096, ch] (a reused buffer), the rows stage_images
        makes of pool images perm_{seed,round}(offset + r), r < n (gm_stage_pool_rows).  idx_out: int32 [>= n] device tensor
        that receives the drawn pool indices."""
        if pool.ch != self.ch:
            raise GmError("the pool holds %d-channel images; this engine takes %d channels" % (pool.ch, self.ch))
        x = self._buf("pool_x", n * 4096, self.ch)
        check(self.h, lib().gm_stage_pool_rows(self.h, _ptr(pool.codes), pool.n, pool.row_vals, _ptr(pool.table), int(seed), int(round),
                                               int(offset), int(n), _ptr(x), _ptr(idx_out), _stream()))
        return x

    # the per-row loss each variant's rows share: WGAN-GP's are W's and DRAGAN's NS's (the penalty is separate); the G steps of
    # RaNS and Fisher are NS's and W's -mean(D(G(z))) (src/ra_gan.py, src/fisher_gan.py train_G); InfoGAN's D and G steps
    # are NS's (src/info_gan.py:223-267)
    _ROW_LOSS = {"wgp": "w", "dra": "ns", "ra": "ns", "fisher": "w", "info": "ns"}

    def _loss_rows(self, logits, n, g_step, inv, ds, loss):
        variant = VARIANTS[self._ROW_LOSS.get(self.variant, self.variant)]
        lc = _lib.LossConsts(self.gp_lambda, self.gp_k, self.dra_c, self.ls_a, self.ls_b, self.ls_c)
        check(self.h, lib().gm_loss_rows_c(self.h, variant, OUT_ACTS[self.d_out_act], _ptr(logits), n, g_step, inv, C.byref(lc), _ptr(ds),
                                           None, loss, _stream()))

    def _reduce_stats(self, buf):
        if self.stats_reduce is not None:
            self.stats_reduce(buf)

    def fisher_state(self, lam=None, rho=None):
        """Fisher GAN's multiplier and penalty weight (LAMBDA, RHO) on the device: set (both given) or read"""
        if lam is not None:
            self.fisher.copy_(torch.tensor([float(lam), float(rho)]))
            return float(lam), float(rho)
        lam, rho = self.fisher.tolist()
        return lam, rho

    def loss_stats(self, logits, n, stat_batch, stats):
        """RaNS / Fisher statistics of the D-step logits [real n | fake n] into stats (float64 [8]): phase 0, the ranks'
        sum, then (RaNS) phase 1 on the global phase-0 sums and its sum"""
        v = VARIANTS[self.variant]
        check(self.h, lib().gm_loss_stats(self.h, v, OUT_ACTS[self.d_out_act], _ptr(logits), n, stat_batch, 0, None, _ptr(stats), _stream()))
        self._reduce_stats(stats[:4])
        if self.variant == "ra":
            check(self.h, lib().gm_loss_stats(self.h, v, OUT_ACTS[self.d_out_act], _ptr(logits), n, stat_batch, 1, _ptr(stats),
                                              _ptr(stats[4:]), _stream()))
            self._reduce_stats(stats[4:])

    def loss_rows_stats(self, logits, n, stat_batch, stats, inv, ds, loss):
        """pass 2 of the RaNS / Fisher D loss on global statistics: ds [2n], loss [4] ([0] the D loss, [2] Fisher's Omega);
        Fisher's LAMBDA (self.fisher[0]) moves by -RHO Omega"""
        check(self.h, lib().gm_loss_rows_stats(self.h, VARIANTS[self.variant], OUT_ACTS[self.d_out_act], _ptr(logits), n, inv, _ptr(stats),
                                               stat_batch, _ptr(self.fisher), _ptr(ds), None, _ptr(loss), _stream()))

    def d_grad(self, img_real, n, noise=None, inv_global_batch=None, seed=0, step=0, gp_lambda=None, eps=None, gp_k=None, dra_c=None,
               delta=None, u=None, stat_batch=None):
        """train_D + backward (src/ns_gan.py:172-194,138; src/w_gp_gan.py:177-220 for wgp, src/dra_gan.py:174-225 for dra,
        src/ra_gan.py:186-207 for ra, src/fisher_gan.py:193-229 for fisher): img_real NHWC rows of n images (stage_images).
        Writes the flat D gradient (self.D.grads) and loss_buf[0].  WGAN-GP and DRAGAN: gp_lambda (None = self.gp_lambda).
        WGAN-GP: eps [n] fp32 (None = on-device Philox keyed by (seed, step)).  DRAGAN: gp_k, dra_c (None = self.gp_k,
        self.dra_c), delta [n] and u [n, ch*64*64] (the reference's NCHW-flattened layout) or None for Philox.  RaNS, Fisher
        and DRAGAN: stat_batch = the batch the statistics run over (None = n; the global batch under stats_reduce)."""
        if self.variant in ("vae", "ae"):
            raise GmError("the %s has no D step: its train step is %s_grad" % (self.variant.upper(), self.variant))
        inv = 1.0 / n if inv_global_batch is None else inv_global_batch
        lam = self.gp_lambda if gp_lambda is None else float(gp_lambda)
        stat_batch = n if stat_batch is None else int(stat_batch)
        fake, _ = self.g_forward(n, noise, seed, 2 * step)
        if self.variant == "be":
            return self._began_d_grad(img_real, fake, n, inv, stat_batch)
        if self.variant == "wgp":
            return self.wgp_critic_grad(img_real, fake, n, inv, lam, eps, seed, step)
        if self.variant == "dra":
            return self.dra_critic_grad(img_real, fake, n, inv, lam, self.gp_k if gp_k is None else float(gp_k),
                                        self.dra_c if dra_c is None else float(dra_c), delta, u, seed, step, stat_batch)
        lr_, lf_ = self._buf("logits_r", 16, n, torch.float32), self._buf("logits_f", 16, n, torch.float32)
        sr = self.d_forward(img_real, n, lr_, "dr")
        sf = self.d_forward(fake, n, lf_, "df")
        logits = self._buf("logits", 1, 2 * n, torch.float32)[0]           # [real | fake], what the loss kernel walks
        logits[:n].copy_(lr_[0])
        logits[n:].copy_(lf_[0])
        ds = self._buf("ds", 1, 2 * n, torch.float32)[0]
        if self.variant in ("ra", "fisher"):
            stats = self._buf("loss_stats", 1, 8, torch.float64)[0]
            lossv = self._buf("loss_stat_out", 1, 4, torch.float32)[0]
            self.loss_stats(logits, n, stat_batch, stats)
            self.loss_rows_stats(logits, n, stat_batch, stats, inv, ds, lossv)
            self.loss_buf[0].copy_(lossv[0])
            self.loss_stats_, self.fisher_omega_ = stats, lossv[2]
        else:
            self._loss_rows(logits, n, 0, inv, ds, _ptr(self.loss_buf))
        g2 = self._buf("dgrad2", 1, self.D.total, torch.float32)[0]
        self.D.grads.zero_()
        g2.zero_()
        self.d_backward(sr, ds[:n], self.D.grads, tag="dr")
        self.d_backward(sf, ds[n:], g2, tag="df")
        self.D.grads.add_(g2)
        self.scores_ = logits
        return self.loss_buf[0]

    def _stack_x3(self, img_real, fake, n):
        """NHWC rows [real | fake | x_hat] of n images each for the penalised critics; the caller writes x_hat's rows"""
        R = n * 4096
        x3 = self._buf("gp_x3", 3 * R, self.ch)
        x3[:R].copy_(img_real)
        x3[R:2 * R].copy_(fake)
        return x3

    def wgp_critic_grad(self, img_real, fake, n, inv, lam, eps=None, seed=0, step=0):
        """The critic half of the WGAN-GP D step for given real and generated NHWC image rows: D_loss = mean(D(G(z))) -
        mean(D(x)) + lam mean_b (||grad D(x_hat_b)|| - 1)^2 at x_hat = eps x + (1 - eps) G(z) (src/w_gp_gan.py:186-218),
        the penalty's double backward in closed form (DESIGN.md §6b)."""
        R = n * 4096
        x3 = self._stack_x3(img_real, fake, n)
        eps_used = self._buf("gp_eps", 1, n, torch.float32)[0]
        if eps is not None:
            eps = eps.reshape(n).float().contiguous()
        check(self.h, lib().gm_gp_interp_rows(self.h, _ptr(x3), self.ch, _ptr(x3[R:]), self.ch, n, 4096, self.ch, _ptr(eps), _ptr(eps_used),
                                              int(seed), int(2 * step), _ptr(x3[2 * R:]), self.ch, _stream()))
        self.gp_eps_ = eps_used
        return self._penalised_critic_grad(x3, n, inv, lam)

    def dra_std_sums(self, img_real, n, sums):
        """this process's (sum x, sum x^2) of the real images (NHWC rows of n images) into sums (float64 [2])"""
        cols = 4096 * self.ch
        check(self.h, lib().gm_dra_std_sums(self.h, _ptr(img_real), n, cols, cols, _ptr(sums), _stream()))

    def dra_critic_grad(self, img_real, fake, n, inv, lam, K=1.0, C=1.0, delta=None, u=None, seed=0, step=0, stat_batch=None):
        """The critic half of the DRAGAN D step (src/dra_gan.py:174-225) for given real and generated NHWC image rows:
        x_hat = delta x + (1 - delta)(x + C std(x) u) around the real data, std over the stat_batch images behind
        stats_reduce, then the NS rows on real / fake and the penalty lam mean (||grad sigmoid(D(x_hat))|| - K)^2."""
        R, cols = n * 4096, 4096 * self.ch
        x3 = self._stack_x3(img_real, fake, n)
        sums = self._buf("dra_sums", 1, 2, torch.float64)[0]
        self.dra_std_sums(x3[:R], n, sums)
        self._reduce_stats(sums)
        rnd = None
        if delta is not None or u is not None:
            if delta is None or u is None:
                raise GmError("DRAGAN's delta and u are given together or not at all")
            u = u.reshape(n, self.ch, 64, 64).permute(0, 2, 3, 1).reshape(-1)       # NCHW-flattened -> the NHWC rows' order
            rnd = torch.cat([delta.reshape(n).float(), u.float()]).to(self.device).contiguous()
        count = float(n if stat_batch is None else stat_batch) * cols
        check(self.h, lib().gm_dra_xhat_rows(self.h, _ptr(x3), n, cols, cols, _ptr(sums), count, float(C), _ptr(rnd), int(seed), int(2 * step),
                                             _ptr(x3[2 * R:]), cols, _stream()))
        self.dra_sums_ = sums
        return self._penalised_critic_grad(x3, n, inv, lam, K)

    def _penalised_critic_grad(self, x3, n, inv, lam, K=1.0):
        """The D gradient of a batch-norm-free critic with a gradient penalty at x_hat (DESIGN.md §6b) from the stacked NHWC
        rows x3 = [real | fake | x_hat] of n images each.  WGAN-GP: W rows, relu / linear output, penalty on ||grad D||;
        DRAGAN: NS rows on the sigmoid output, penalty on ||grad sigmoid(s)|| = sigma' ||grad s|| with target K."""
        dc, D, ch = self.dc, self.D, self.ch
        R = n * 4096
        dra = self.variant == "dra"
        # 1. primal forward of the 3n images; the LeakyReLU outputs y_l carry the masks
        logits = self._buf("gp_logits", 16, 3 * n, torch.float32)
        sv = self.d_forward(x3, 3 * n, logits, "dw")
        # 2. upstream dL/dlogit: the loss rows for real / fake (loss_buf[0]), and the x_hat rows' seed - WGAN-GP: 1[s > 0]
        #    (relu output) or 1, the loss kernel's train_G row (-d, gradient -act'(s) * inv) with inv = -1; DRAGAN: 1, so
        #    that the chain below is J = ds/dx_hat and the sigmoid enters through the penalty kernel
        ds = self._buf("gp_ds", 1, 3 * n, torch.float32)[0]
        self._loss_rows(logits[0], n, 0, inv, ds, _ptr(self.loss_buf))
        if dra:
            ds[2 * n:].fill_(1.0)
        else:
            self._loss_rows(logits[0, 2 * n:], n, 1, -1.0, ds[2 * n:], _ptr(self._buf("gp_seed_loss", 1, 4, torch.float32)))
        dy5 = self._buf("dwdy5", 3 * n, 16)
        check(self.h, lib().gm_pack_col0(self.h, _ptr(ds), 3 * n, _ptr(dy5), 16, _stream()))
        betas = self._betas(sv, dy5, "dw")
        # 2b. image gradient g at x_hat and 3. the penalty: loss_buf[0] += lam mean (||g|| - K)^2, tangent seed r
        g = self._dimg(sv, betas[0][2 * n * 1024:], "gp", C2I_NONE)
        r = self._buf("gp_r", R, ch)
        norms = self._buf("gp_norm", 1, n, torch.float32)[0]
        if dra:
            check(self.h, lib().gm_dra_penalty(self.h, _ptr(g), ch, _ptr(x3[2 * R:]), ch, _ptr(logits[0, 2 * n:]), n, 4096, ch, lam, K, inv,
                                               1.0 / n, _ptr(r), ch, _ptr(norms), _ptr(self.loss_buf), _stream()))
        else:
            check(self.h, lib().gm_gp_penalty(self.h, _ptr(g), ch, n, 4096, ch, lam, inv, 1.0 / n, _ptr(r), ch, _ptr(norms),
                                              _ptr(self.loss_buf), _stream()))
        # 4. tangent pass t_0 = r, t_l = LReLU'(y_l) * conv_l(t_{l-1}) under x_hat's masks.  im2col(t_{l-1}) overwrites
        #    x_hat's rows of the saved column matrices (and t_4 x_hat's rows of y_4 = the last layer's input), so that
        # 5. each layer's weight gradient is ONE GEMM over the 3n images: W part (activations) + penalty (tangents).
        _im2col(r, n, 64, 64, ch, sv["col0"][2 * n * 1024:])
        hw = 32
        for i in range(4):
            off = 2 * n * hw * hw
            u = self._buf("gp_u%d" % i, n * hw * hw, dc[i])
            gemm_bf16(sv["col%d" % i][off:], D.bf["l%d.weight" % (i + 1)], u, "nt")
            y_hat = sv["y%d" % i][off:]
            if i < 3:
                _im2col_lrelu_mask(u, n, hw, hw, dc[i], y_hat, sv["col%d" % (i + 1)][2 * n * (hw // 2) ** 2:])
            else:
                _lrelu_mask(u, y_hat, y_hat)
            hw //= 2
        D.grads.zero_()
        gemm_bf16(dy5, sv["flat"], D.view("l5.weight", D.grads), "tn")
        for i in range(4):
            gemm_bf16(betas[i], sv["col%d" % i], D.view("l%d.weight" % (i + 1), D.grads), "tn")
        self.scores_ = logits[0, :2 * n]
        self.gp_norms_, self.gp_logits_, self.gp_r_ = norms, logits[0, 2 * n:], r   # per-image ||g||, x_hat logits, tangent seed
        return self.loss_buf[0]

    def g_grad(self, n, noise=None, inv_global_batch=None, seed=0, step=0):
        """train_G + backward (src/ns_gan.py:196-216,155): G gradients only."""
        if self.variant in ("vae", "ae"):
            raise GmError("the %s has no G step: its train step is %s_grad" % (self.variant.upper(), self.variant))
        inv = 1.0 / n if inv_global_batch is None else inv_global_batch
        fake, gsv = self.g_forward(n, noise, seed, 2 * step + 1)
        if self.variant == "be":
            return self._began_g_grad(fake, gsv, n, inv)
        logits = self._buf("logits_g", 16, n, torch.float32)
        sf = self.d_forward(fake, n, logits, "df")
        ds = self._buf("ds_g", 1, n, torch.float32)[0]
        self._loss_rows(logits, n, 1, inv, ds, C.c_void_p(self.loss_buf.data_ptr() + 4))
        dpre = self.d_backward(sf, ds, None, need_wgrad=False, need_dimg=True, tag="df")
        self.g_backward(gsv, dpre)
        return self.loss_buf[1]

    def apply(self, net, hp=None):
        """Adam on G (net 0) or D (net 1) with hp.  The VAE's and the autoencoder's apply(hp) steps both: their one optimizer
        over encoder and decoder (src/vae.py:139-142, src/ae.py:98-101) is elementwise, so an Adam step per net with the same
        step count is that optimizer exactly."""
        if self.variant in ("vae", "ae"):
            hp = net if hp is None else hp
            self.D.adam(hp)
            self.G.adam(hp)
            return
        # BEGAN: both learning rates carry the plateau scale be_state[7]; the reference's two schedulers see the same
        # measure with the same settings (src/be_gan.py:133-136,194-195), so one scale is exact
        (self.G if net == 0 else self.D).adam(hp, self.be_state[7:8] if self.variant == "be" else None)

    # ------------------------------------------------------------------ InfoGAN (src/info_gan.py:269-304)
    # The MI step's Philox streams: bit 63 set, so that no D draw (2 step) or G draw (2 step + 1) of any step reaches them
    MI_STREAM = 1 << 63

    def q_grad(self, n, noise=None, inv_global_batch=None, seed=0, step=0, lam=1.0):
        """train_Q + MI_loss.backward() (src/info_gan.py:269-304): fresh codes (noise [n, zin] fp32, or Philox keyed by (seed,
        MI_STREAM + step)), G(codes), Q(G(codes)) as fp32 rows, MI_loss = lam (CE(discrete, argmax one-hot) + MSE(continuous,
        code)).  The gradient reaches Q and G (G's output is not detached): writes Q.grads and G.grads (both carry
        lam inv_global_batch) and mi_loss[0] (lam times this process's mean)."""
        if self.variant != "info":
            raise GmError("q_grad is InfoGAN's MI step (variant='info')")
        inv = 1.0 / n if inv_global_batch is None else inv_global_batch
        if noise is not None:
            noise = noise.reshape(n, self.zin).float().contiguous()
        fake, gsv = self.g_forward(n, noise, seed, self.MI_STREAM + int(step))
        codes = self.codes_["g"] if noise is None else noise
        qrows = self._buf("q_rows", n, self.qp, torch.float32)
        sv = self.d_forward(fake, n, qrows, "q", net=self.Q, run=self.run_Q)
        dq = self._buf("q_dq", n, self.qp)
        check(self.h, lib().gm_info_loss_rows(self.h, _ptr(qrows), self.qp, _ptr(codes), self.zin, self.z, n, self.nd, self.nc, inv * lam,
                                              _ptr(dq), self.qp, _ptr(self.mi_loss), _stream()))
        if lam != 1.0:
            self.mi_loss.mul_(lam)
        dpre = self.d_backward(sv, dq, self.Q.grads, need_dimg=True, tag="q", net=self.Q)
        self.g_backward(gsv, dpre)
        # the step's stored tensors: codes, Q's rows and their gradient, dL/d(pre-sigmoid G output), the saved activations
        self.q_saved_ = dict(codes=codes, q=qrows, dq=dq, dpre=dpre, qsv=sv, gsv=gsv, fake=fake)
        return self.mi_loss[0]

    def apply_mi(self, hp):
        """MI_optimizer.step() (src/info_gan.py:148,205): Adam over G with MI_optimizer's own moments (not G.exp_avg /
        exp_avg_sq, which are G_optimizer's) and over Q, one step count for both; refreshes both operand copies"""
        self.Q.adam(hp)
        adam_step(self.G.params, self.G.grads, self.g_mi_avg, self.g_mi_avg_sq, hp, self.Q.step)
        self.G.refresh()

    def infer_codes(self, images):
        """Q(images) (src/info_gan.py:90-94): flat [n, ch*64*64] (NCHW flattened) -> (discrete logits [n, nd], continuous
        [n, nc]) fp32"""
        n = images.shape[0]
        qrows = self._buf("qi_rows", n, self.qp, torch.float32)
        self.d_forward(self.stage_images(images), n, qrows, "qi", net=self.Q, run=self.run_Q)
        return qrows[:, :self.nd].clone(), qrows[:, self.nd:self.nd + self.nc].clone()

    # ------------------------------------------------------------------ VAE (src/vae.py:94-106,193-212)
    # Forward-only draws of eps (vae_forward without a caller eps): a stream with bit 56 set, which no train step (stream =
    # step) reaches; vae_reparam_kernel offsets Philox by 64 stream_id, so the stream stays below 2^58
    VAE_FWD_STREAM = 1 << 56

    def _vae_only(self, what):
        if self.variant != "vae":
            raise GmError("%s is the VAE's (variant='vae')" % what)

    def _vae_latent(self, mulv, n, eps, seed, stream_id, kl, tag):
        """gm_vae_latent_rows on the encoder head's rows mulv [n, mp]: (the decoder's bf16 input rows [n, zp] = [z | 1 | 0],
        the eps used [n, z] fp32); kl[0] = this process's sum of the KL terms"""
        zrows = self._buf(tag + "z", n, self.zp)
        eps_used = self._buf(tag + "eps", n, self.z, torch.float32)
        if eps is not None:
            eps = eps.reshape(n, self.z).to(self.device, torch.float32).contiguous()
        check(self.h, lib().gm_vae_latent_rows(self.h, _ptr(mulv), self.mp, _ptr(eps), _ptr(eps_used), _ptr(zrows), self.zp, n, self.z,
                                               int(seed), int(stream_id), _ptr(kl), _stream()))
        return zrows, eps_used

    def sse_sigmoid_rows(self, out, x, n, scale, grad, total):
        """the VAE's reconstruction term on n NHWC images: total[0] = sum (x - out)^2, grad = 2 scale (out - x) out (1 - out)"""
        check(self.h, lib().gm_sse_sigmoid_rows(self.h, _ptr(out), _ptr(x), n, 4096 * self.ch, float(scale), _ptr(grad), _ptr(total),
                                                _stream()))

    def vae_grad(self, img_rows, n, eps=None, seed=0, step=0):
        """compute_batch + (recon + kl).backward() (src/vae.py:150-161,193-212) for n NHWC image rows (stage_images): the encoder
        forward with the heads as fp32 rows, z = mu + eps e^(lv/2) (eps [n, z] given, or Philox keyed by (seed, step)), the
        decoder, recon = sum (x - out)^2 and KL = sum 0.5 (mu^2 + e^lv - lv - 1).  Both losses are sums, so the gradients carry
        scale 1 and sum exactly over data-parallel ranks.  Writes G.grads (decoder), D.grads (encoder) and vae_loss = (recon,
        kl), this process's sums."""
        self._vae_only("vae_grad")
        z, mp = self.z, self.mp
        sums = self._buf("vae_sums", 1, 2, torch.float64)[0]
        mulv = self._buf("vae_mulv", n, mp, torch.float32)
        sve = self.d_forward(img_rows, n, mulv, "ve")
        zrows, eps_used = self._vae_latent(mulv, n, eps, seed, step, sums[1:2], "vae_")
        out, svd = self.g_forward(n, tag="vd", x_rows=zrows)
        dpre = self._buf("vae_dpre", n * 4096, self.ch)
        self.sse_sigmoid_rows(out, img_rows, n, 1.0, dpre, sums[0:1])
        dz = self.g_backward(svd, dpre, need_dx=True, tag="vd", dx_dtype=torch.float32)
        dml = self._buf("vae_dml", n, mp)
        check(self.h, lib().gm_vae_dlatent_rows(self.h, _ptr(mulv), mp, _ptr(dz), dz.stride(0), _ptr(eps_used), _ptr(dml), mp, n, z, 1.0,
                                                _stream()))
        self.d_backward(sve, dml, self.D.grads, tag="ve")
        self.vae_loss.copy_(sums)
        # the step's stored tensors: the head rows, eps, z rows, the reconstruction, dpre, dz, the head upstream, activations
        self.vae_saved_ = dict(mulv=mulv, eps=eps_used, zrows=zrows, out=out, dpre=dpre, dz=dz, dml=dml, sve=sve, svd=svd, sums=sums)
        return self.vae_loss

    def vae_forward(self, img_rows, n, eps=None, train=True, seed=0, step=0):
        """VAE.forward + compute_batch's losses without a backward (src/vae.py:94-98,193-208) for n NHWC image rows: (the
        reconstruction flat [n, ch*64*64] (NCHW flattened) fp32, mu [n, z], log_var [n, z], losses fp32 [2] = (recon, kl) sums).
        eps: [n, z] or None for Philox keyed by (seed, VAE_FWD_STREAM + step).  train=False runs every BatchNorm in inference
        mode (model.eval()); train=True takes batch statistics and updates the running statistics, as torch does."""
        self._vae_only("vae_forward")
        sums = self._buf("vaef_sums", 1, 2, torch.float64)[0]
        mulv = self._buf("vaef_mulv", n, self.mp, torch.float32)
        self.d_forward(img_rows, n, mulv, "vfe", train=train)
        zrows, _ = self._vae_latent(mulv, n, eps, seed, self.VAE_FWD_STREAM + int(step), sums[1:2], "vaef_")
        out, _ = self.g_forward(n, tag="vfd", x_rows=zrows, train=train)
        dpre = self._buf("vaef_dpre", n * 4096, self.ch)
        self.sse_sigmoid_rows(out, img_rows, n, 1.0, dpre, sums[0:1])
        rec = self.rows_to_image(out, n)
        return rec, mulv[:, :self.z].clone(), mulv[:, self.z:2 * self.z].clone(), sums.float()

    def encode(self, images, train=True):
        """Encoder.forward (src/vae.py:58-61): flat [n, ch*64*64] (NCHW flattened) -> (mu, log_var) fp32 [n, z]; the
        autoencoder's (src/ae.py:38-39): -> the code relu(h) fp32 [n, z], the values the decoder reads (bf16)"""
        n = images.shape[0]
        if self.variant == "ae":
            h = self._buf("aee_h", n, self.mp, torch.float32)
            self.d_forward(self.stage_images(images), n, h, "aee", train=train)
            return self._ae_latent(h, n, "aee_")[:, :self.z].float()
        self._vae_only("encode")
        mulv = self._buf("vaee_mulv", n, self.mp, torch.float32)
        self.d_forward(self.stage_images(images), n, mulv, "vee", train=train)
        return mulv[:, :self.z].clone(), mulv[:, self.z:2 * self.z].clone()

    def decode(self, z, train=True):
        """Decoder.forward (src/vae.py:74-77, src/ae.py:51-52): z [n, z] -> images flat [n, ch*64*64] (NCHW flattened) fp32"""
        if self.variant != "ae":
            self._vae_only("decode")
        n = z.shape[0]
        img, _ = self.g_forward(n, z.to(self.device, torch.float32).contiguous(), tag="vdd", train=train)
        return self.rows_to_image(img, n)

    # ------------------------------------------------------------------ autoencoder (src/ae.py:38-52,147-160)
    def _ae_only(self, what):
        if self.variant != "ae":
            raise GmError("%s is the autoencoder's (variant='ae')" % what)

    def _ae_latent(self, h, n, tag):
        """gm_ae_latent_rows on the encoder head's rows h [n, mp]: the decoder's bf16 input rows [n, zp] = [relu(h) | 1 | 0]"""
        zrows = self._buf(tag + "z", n, self.zp)
        check(self.h, lib().gm_ae_latent_rows(self.h, _ptr(h), self.mp, _ptr(zrows), self.zp, n, self.z, _stream()))
        return zrows

    def ae_grad(self, img_rows, n):
        """compute_batch + recon.backward() (src/ae.py:147-160) for n NHWC image rows (stage_images): the encoder forward with
        the head as fp32 rows h, the code relu(h), the decoder, recon = sum (x - out)^2 and the backward through all of them.
        The loss is a sum, so the gradients carry scale 1 and sum exactly over data-parallel ranks.  Writes G.grads (decoder),
        D.grads (encoder) and ae_loss[0] = recon, this process's sum."""
        self._ae_only("ae_grad")
        sums = self._buf("ae_sums", 1, 1, torch.float64)[0]
        h = self._buf("ae_h", n, self.mp, torch.float32)
        sve = self.d_forward(img_rows, n, h, "ae")
        zrows = self._ae_latent(h, n, "ae_")
        out, svd = self.g_forward(n, tag="ad", x_rows=zrows)
        dpre = self._buf("ae_dpre", n * 4096, self.ch)
        self.sse_sigmoid_rows(out, img_rows, n, 1.0, dpre, sums)
        dz = self.g_backward(svd, dpre, need_dx=True, tag="ad", dx_dtype=torch.float32)
        dh = self._buf("ae_dh", n, self.mp)
        check(self.h, lib().gm_ae_dlatent_rows(self.h, _ptr(h), self.mp, _ptr(dz), dz.stride(0), _ptr(dh), self.mp, n, self.z, _stream()))
        self.d_backward(sve, dh, self.D.grads, tag="ae")
        self.ae_loss.copy_(sums)
        # the step's stored tensors: the head rows, the code rows, the reconstruction, dpre, dz, the head upstream, activations
        self.ae_saved_ = dict(h=h, zrows=zrows, out=out, dpre=dpre, dz=dz, dh=dh, sve=sve, svd=svd)
        return self.ae_loss

    def ae_forward(self, img_rows, n, train=True):
        """Autoencoder.forward + compute_batch's loss without a backward (src/ae.py:66-67,147-160) for n NHWC image rows: (the
        reconstruction flat [n, ch*64*64] (NCHW flattened) fp32, the code [n, z] fp32, recon fp32 [1] = sum (x - out)^2).
        train=False runs every BatchNorm in inference mode (model.eval()); train=True takes batch statistics and updates the
        running statistics, as torch does."""
        self._ae_only("ae_forward")
        sums = self._buf("aef_sums", 1, 1, torch.float64)[0]
        h = self._buf("aef_h", n, self.mp, torch.float32)
        self.d_forward(img_rows, n, h, "afe", train=train)
        zrows = self._ae_latent(h, n, "aef_")
        out, _ = self.g_forward(n, tag="afd", x_rows=zrows, train=train)
        dpre = self._buf("aef_dpre", n * 4096, self.ch)
        self.sse_sigmoid_rows(out, img_rows, n, 1.0, dpre, sums)
        return self.rows_to_image(out, n), zrows[:, :self.z].float(), sums.float()

    # ------------------------------------------------------------------ BEGAN (src/be_gan.py:212-258)
    def began_state(self, values=None):
        """BEGAN device state (11 floats, the layout of gm_gan_began_state): set (values given) or read"""
        if values is not None:
            self.be_state.copy_(torch.tensor([float(v) for v in values]))
            return list(values)
        return self.be_state.tolist()

    def began_init(self, K, batch):
        """K, a fresh plateau scheduler (best = inf, lr scale 1) and the MLP layout's scale fields for `batch` images"""
        inv = 1.0 / batch
        return self.began_state([K, inv, -K * inv, 0.0, 0.0, float("inf"), 0.0, 1.0, inv, inv, 0.0])

    def began_control(self, gamma, lam, patience):
        """K <- clip(K + lam (gamma DX - DG), 0, 1), the convergence measure and the ReduceLROnPlateau pair on the device
        (src/be_gan.py:186-195), from the DX, DG of the last D step"""
        check(self.h, lib().gm_began_control(self.h, _ptr(self.be_state), float(gamma), float(lam), float(patience), _stream()))

    def l1_rows(self, r, x, n, inv, coef, grad, total):
        """BEGAN's L1 term on n NHWC images: grad = sign(r - x) inv (coef[0] if coef is given) as bf16, total[0] = sum |r - x|"""
        check(self.h, lib().gm_l1_rows(self.h, _ptr(r), _ptr(x), n, 4096 * self.ch, float(inv), _ptr(coef), _ptr(grad), _ptr(total),
                                       _stream()))

    def began_loss_final(self, sums, batch, g_step, loss):
        """sums (float64 [2]: this process's sum |D(x) - x|, sum |D(G(z)) - G(z)|) -> loss[0]: D step (summed over the ranks
        by stats_reduce first; batch = the global batch) DX - K DG with be_state[3], [4] = DX, DG; G step DG"""
        if not g_step:
            self._reduce_stats(sums)
        check(self.h, lib().gm_began_loss_final(self.h, _ptr(sums[0:1]), _ptr(sums[1:2]), int(batch), int(g_step), _ptr(self.be_state),
                                                _ptr(loss), _stream()))

    def autoencode(self, x, n, tag="be"):
        """D(x) = decoder(encoder(x)) for n NHWC images -> (reconstruction [n*4096, ch] bf16, encoder and decoder saved
        activations).  Each call takes its own BatchNorm batch statistics."""
        emb = self._buf(tag + "emb", n, self.ep)
        sve = self.d_forward(x, n, emb, tag + "e", "encoder.")
        rec, svd = self.g_forward(n, tag=tag + "d", net=self.D, pfx="decoder.", x_rows=emb, out_mode=C2I_NONE, run=self.run_dec)
        return rec, sve, svd

    def _autoencoder_backward(self, sve, svd, dr, grads, tag="be"):
        """dr = dL/d(reconstruction) -> the autoencoder's weight gradients into `grads` (flat D layout)"""
        demb = self.g_backward(svd, dr, self.D, "decoder.", grads, need_dx=True, tag=tag + "d")
        self.d_backward(sve, demb, grads, tag=tag + "e", pfx="encoder.")

    def _began_d_grad(self, img_real, fake, n, inv, stat_batch):
        """train_D + backward (src/be_gan.py:212-238): D_loss = DX - K DG.  The real and the generated half each run the
        autoencoder, the L1 kernel and the backward in turn (sharing buffers); the fake half's gradient carries -K inv with K
        read on the device.  The two sums then meet the ranks' (stats_reduce) in the loss finalisation."""
        sums = self._buf("be_sums", 1, 2, torch.float64)[0]
        g2 = self._buf("dgrad2", 1, self.D.total, torch.float32)[0]
        self.D.grads.zero_()
        g2.zero_()
        drs = []
        for k, (x, grads) in enumerate(((img_real, self.D.grads), (fake, g2))):
            rec, sve, svd = self.autoencode(x, n)
            dr = self._buf("be_dr%d" % k, n * 4096, self.ch)
            self.l1_rows(rec, x, n, inv if k == 0 else -inv, None if k == 0 else self.be_state[0:1], dr, sums[k:k + 1])
            self._autoencoder_backward(sve, svd, dr, grads)
            drs.append(dr)
        self.D.grads.add_(g2)
        self.began_loss_final(sums, stat_batch, 0, self.loss_buf[0:1])
        self.be_sums_, self.be_dr_ = sums, drs                       # this process's L1 sums (before stats_reduce), dL/dr
        return self.loss_buf[0]

    def _began_g_grad(self, fake, gsv, n, inv):
        """train_G + backward (src/be_gan.py:240-258): G_loss = mean_i sum |D(G(z)) - G(z)|, whose gradient reaches G(z) through
        D (T, the autoencoder's input-gradient chain without weight gradients) and directly through the target (-dr).  The
        gradients carry inv (1 / the global batch); the reported G loss is this process's mean, like every G loss of the conv
        path (only the D step's DX and DG are global: K and the lr scale must agree on every rank)."""
        sums = self._buf("be_sums_g", 1, 2, torch.float64)[0]
        rec, sve, svd = self.autoencode(fake, n)
        dr = self._buf("be_drg", n * 4096, self.ch)
        self.l1_rows(rec, fake, n, inv, None, dr, sums[1:2])
        self.began_loss_final(sums, n, 1, self.loss_buf[1:2])
        demb = self.g_backward(svd, dr, self.D, "decoder.", need_wgrad=False, need_dx=True, tag="bed")
        T = self.d_backward(sve, demb, None, need_wgrad=False, need_dimg=True, tag="bee", pfx="encoder.", dimg_mode=C2I_NONE)
        dpre = self._buf("be_dpre", n * 4096, self.ch)
        check(self.h, lib().gm_began_dfake_rows(self.h, _ptr(T), _ptr(dr), _ptr(fake), _ptr(dpre), n, 4096 * self.ch, _stream()))
        self.g_backward(gsv, dpre)
        # the step's stored tensors: dL/dr, the autoencoder's saved activations, the embedding gradient, T, dpre, G's activations
        self.be_drg_, self.be_g_saved_ = dr, dict(sve=sve, svd=svd, demb=demb, T=T, dpre=dpre, gsv=gsv, fake=fake)
        return self.loss_buf[1]

    def reconstruct(self, images):
        """BEGAN's D(images): flat [n, ch*64*64] (NCHW flattened) -> the reconstructions in the same layout (fp32)"""
        n = images.shape[0]
        rec, _, _ = self.autoencode(self.stage_images(images), n, "ber")
        return self.rows_to_image(rec, n)

    def generate(self, noise):
        n = noise.shape[0]
        img, _ = self.g_forward(n, noise.float().contiguous(), tag="gen")
        return self.rows_to_image(img, n)

    def discriminate(self, images):
        n = images.shape[0]
        logits = self._buf("logits_i", 16, n, torch.float32)
        self.d_forward(self.stage_images(images), n, logits, "di")
        return self._out_act(logits[0, :n].view(n, 1))

    def _out_act(self, s):
        return torch.sigmoid(s) if self.d_out_act == "sigmoid" else (torch.relu(s) if self.d_out_act == "relu" else s.clone())

    # ------------------------------------------------------------------ per-call forward / backward (user-written losses)
    # A user's train_D / train_G (README.md:31) calls model.D / model.G as its loss needs and back-propagates through the
    # drop-ins' autograd nodes (dc_gan._DcDForward / _DcGForward).  Each call keeps its saved activations in a slot of a ring,
    # D_SLOTS discriminator and G_SLOTS generator calls, allocated on first use; a backward whose slot a later call has taken
    # raises instead of reading that call's tensors.  The losses that need these are the ones whose D returns one score per
    # image, and the VAE's and autoencoder's compute_batch, whose encoder is D's trunk and head and whose decoder is G;
    # BEGAN's autoencoder D and InfoGAN's coded input and Q have none.
    D_SLOTS, G_SLOTS = 4, 2

    @property
    def supports_custom_loss(self):
        return self.variant not in ("be", "info")

    def _take_slot(self, kind):
        if not self.supports_custom_loss:
            raise GmError("per-call forwards with a backward are built for the discriminators with one score per image "
                          "(not %s)" % self.variant)
        gens = self._slot_gen[kind]
        self._calls[kind] += 1
        slot = (self._calls[kind] - 1) % len(gens)
        gens[slot] = self._calls[kind]
        return dict(kind=kind, slot=slot, gen=self._calls[kind])

    def _check_live(self, handle, what):
        if self._slot_gen[handle["kind"]][handle["slot"]] != handle["gen"]:
            raise RuntimeError("%s activations were overwritten: at most %d %s.forward results can await their backward"
                               % (what, len(self._slot_gen[handle["kind"]]), what))

    def custom_d_forward(self, images):
        """D(images) in training mode (batch statistics; the running statistics move per call, as nn.BatchNorm2d.train()):
        images [n, ch*64*64] (NCHW flattened) -> (scores [n, 1] fp32 = out_act(logits), the handle for custom_d_backward:
        slot, generation, saved activations sv).  The VAE's encoder returns ((mu, log_var) [n, z] fp32, handle), the
        autoencoder's (the code relu(h) [n, z] fp32, the bf16 values the decoder reads, handle), as encode does."""
        x = self._image_arg(images)
        n = x.shape[0]
        h = self._take_slot("d")
        tag = "cd%d" % h["slot"]
        rows = self.image_to_rows(x, dst=self._buf(tag + "x", n * 4096, self.ch))
        if self.variant in ("vae", "ae"):
            head = self._buf(tag + "head", n, self.mp, torch.float32)
            h.update(n=n, sv=self.d_forward(rows, n, head, tag), head=head)
            if self.variant == "ae":
                return self._ae_latent(head, n, tag)[:, :self.z].float(), h
            return (head[:, :self.z].clone(), head[:, self.z:2 * self.z].clone()), h
        logits = self._buf(tag + "logits", 16, n, torch.float32)
        h.update(n=n, sv=self.d_forward(rows, n, logits, tag), s=logits[0, :n])
        return self._out_act(h["s"].view(n, 1)), h

    def custom_d_backward(self, handle, dscore, need_dx):
        """dscore [n] = dL/d(score) of custom_d_forward's call -> ({"D.<name>": weight / BatchNorm gradient in torch's layout},
        dL/d(images) [n, ch*64*64] fp32 or None).  dL/dlogit = dscore act'(s) is formed on the n logits.  For the VAE's
        encoder dscore is (dL/dmu, dL/dlog_var), each [n, z], for the autoencoder's dL/dcode [n, z]; they have no dL/dx."""
        if self.variant in ("vae", "ae"):
            self._check_live(handle, "Encoder")
            if need_dx:
                raise GmError("the gradient with respect to the encoder's input is not computed")
            return self._torch_views({"D": self._encoder_backward(handle, dscore)}), None
        self._check_live(handle, "Discriminator")
        n, s = handle["n"], handle["s"]
        d = dscore.reshape(n).to(self.device, torch.float32)
        if self.d_out_act == "sigmoid":
            p = torch.sigmoid(s)
            d = d * (p * (1 - p))
        elif self.d_out_act == "relu":
            d = d * (s > 0).float()
        grads = torch.zeros(self.D.total, device=self.device)   # d_backward writes, never adds: one buffer per call
        dimg = self.d_backward(handle["sv"], d.contiguous(), grads, need_dimg=need_dx, tag="cdb", dimg_mode=C2I_NONE)
        return self._torch_views({"D": grads}), (self.rows_to_image(dimg, n) if need_dx else None)

    def _encoder_backward(self, handle, dhead):
        """the head's bf16 upstream rows [n, mp] (the VAE's [dmu | dlog_var | 0] by gm_cast_bf16 into zeroed padding, the
        autoencoder's dcode 1[h > 0] by gm_ae_dlatent_rows), then the trunk's backward -> flat D gradient"""
        n, z, mp = handle["n"], self.z, self.mp
        key = "cdhead%d" % handle["slot"]
        if key not in self._bufs or self._bufs[key].shape[0] < n:
            self._bufs[key] = torch.zeros(n, mp, device=self.device, dtype=torch.bfloat16)   # columns [2z, mp) stay zero
        up = self._bufs[key][:n]
        if self.variant == "ae":
            dz = dhead.to(self.device, torch.float32).contiguous()
            check(self.h, lib().gm_ae_dlatent_rows(self.h, _ptr(handle["head"]), mp, _ptr(dz), z, _ptr(up), mp, n, z, _stream()))
        else:
            for k, d in enumerate(dhead):
                d = d.to(self.device, torch.float32).contiguous()
                check(self.h, lib().gm_cast_bf16(self.h, _ptr(d), n, z, C.c_void_p(up.data_ptr() + 2 * k * z), mp, None, 0, _stream()))
        grads = torch.zeros(self.D.total, device=self.device)
        self.d_backward(handle["sv"], up, grads, tag="cdb")
        return grads

    def custom_g_forward(self, noise):
        """G(noise) in training mode: noise [n, z] -> (images [n, ch*64*64] fp32, NCHW flattened; the handle for
        custom_g_backward)"""
        n = noise.shape[0]
        z = noise.to(self.device, torch.float32).reshape(n, self.zin).contiguous()
        h = self._take_slot("g")
        img, sv = self.g_forward(n, z, tag="cg%d" % h["slot"])
        h.update(n=n, sv=sv)
        return self.rows_to_image(img, n), h

    def custom_g_backward(self, handle, dimages, need_dz=False):
        """dimages [n, ch*64*64] = dL/dG(z) of custom_g_forward's call -> {"G.<name>": gradient in torch's layout}, and with
        need_dz (the VAE's / autoencoder's decoder) also dL/dz [n, z] fp32.  The upstream of the pre-sigmoid output,
        dimages G(z) (1 - G(z)), is rounded to bf16 once (gm_image_to_rows)."""
        self._check_live(handle, "Decoder" if self.variant in ("vae", "ae") else "Generator")
        sv, n = handle["sv"], handle["n"]
        dpre = self.image_to_rows(dimages, sv["img"], self._buf("cgdpre", n * 4096, self.ch))
        grads = torch.zeros(self.G.total, device=self.device)
        if not need_dz:
            self.g_backward(sv, dpre, grads=grads)
            return self._torch_views({"G": grads})
        dz = self.g_backward(sv, dpre, grads=grads, need_dx=True, tag="cg", dx_dtype=torch.float32)
        return self._torch_views({"G": grads}), dz[:, :self.zin].clone()
