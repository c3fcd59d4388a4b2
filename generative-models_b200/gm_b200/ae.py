"""AeEngine — the standard autoencoder of src/ae.py (x -> relu(W1 x + b1) -> sigmoid(W2 h + b2), loss = sum (x - out)^2,
Adam with coupled weight decay; src/ae.py:28-49,97-105,147-158) on the wgmma GEMM of libgm_b200.so.

The AE is a strict subset of the VAE's kernels (SURVEY.md 2): both layers are gm_gemm_bf16 calls with fused epilogues —
bias + ReLU (+ ones column), bias + sigmoid + the SSE loss and its gradient -2 (x - out) out (1 - out) in the decoder's
epilogue — the two weight gradients are MN-major split-K GEMMs whose extra ones-column row / column carries the bias
gradient, the hidden gradient is one GEMM with the ReLU mask in its epilogue, Adam is gm_adam_step.  This module only
sequences those C-ABI calls (host language of the reference: Python).

Flat fp32 layout = the reference's state_dict order: [encoder.linear.weight (h, x) | .bias (h) | decoder.linear.weight (x, h) | .bias (x)]."""
import torch

from . import _lib
from ._lib import GmError, IMG_FMTS, check, lib, _ptr, _stream, gemm_bf16, adam_step

NAMES = ["encoder.linear.weight", "encoder.linear.bias", "decoder.linear.weight", "decoder.linear.bias"]


def _pad(v, m):
    return (v + m - 1) // m * m


class AeEngine:
    def __init__(self, image_size=784, hidden_dim=32, max_batch=64, device=None):
        if not torch.cuda.is_available():
            raise GmError("gm_b200 needs a CUDA (H100) device; there is no CPU fallback")
        if image_size % 16 or hidden_dim % 16:
            raise GmError("image_size and hidden_dim must be multiples of 16")
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        self.h = _lib.ctx(self.device.index)
        self.X, self.H, self.max_batch = image_size, hidden_dim, max_batch
        self.XP, self.HP = _pad(image_size + 1, 16), _pad(hidden_dim + 1, 16)
        X, H = image_size, hidden_dim
        self.shapes = [(H, X), (H,), (X, H), (X,)]
        self.offsets, off = [], 0
        for shp in self.shapes:
            n = shp[0] * (shp[1] if len(shp) > 1 else 1)
            self.offsets.append((off, n))
            off += n
        kw = dict(device=self.device, dtype=torch.float32)
        self.params, self.grads = torch.zeros(off, **kw), torch.zeros(off, **kw)
        self.exp_avg, self.exp_avg_sq = torch.zeros(off, **kw), torch.zeros(off, **kw)
        self.steps = 0
        bf = dict(device=self.device, dtype=torch.bfloat16)
        self.W1s = torch.zeros(H, _pad(X, 8), **bf)[:, :X]
        self.W2s = torch.zeros(X, _pad(H, 8), **bf)[:, :H]
        self.W2t = torch.zeros(H, _pad(X, 8), **bf)[:, :X]
        B = max_batch
        self.xb, self.e = torch.zeros(B, self.XP, **bf), torch.zeros(B, self.HP, **bf)
        self.da, self.de = torch.zeros(B, self.XP, **bf), torch.zeros(B, self.HP, **bf)
        self.nslots = 2 * ((X + 207) // 208)
        self.slots = torch.zeros(self.nslots, B, **kw)
        # fp32 GEMM outputs need 16-byte rows (float4 stores): leading dimensions padded past the extra bias column
        self.gw2, self.gw1 = torch.zeros(X, _pad(H + 1, 16), **kw), torch.zeros(H, _pad(X + 1, 16), **kw)
        self.loss_buf = torch.zeros(1, **kw)

    def views(self, flat=None):
        flat = self.params if flat is None else flat
        return {n: flat[o:o + c].view(s) for n, (o, c), s in zip(NAMES, self.offsets, self.shapes)}

    def load(self, tensors):
        v = self.views()
        for n, t in tensors.items():
            v[n].copy_(torch.as_tensor(t, dtype=torch.float32).reshape(v[n].shape))
        self.sync_shadows()

    def sync_shadows(self):
        v = self.views()
        w1, w2 = v[NAMES[0]], v[NAMES[2]]
        check(self.h, lib().gm_cast_bf16(self.h, _ptr(w1), w1.shape[0], w1.shape[1], _ptr(self.W1s), self.W1s.stride(0), None, 0, _stream()))
        check(self.h, lib().gm_cast_bf16(self.h, _ptr(w2), w2.shape[0], w2.shape[1], _ptr(self.W2s), self.W2s.stride(0),
                                         _ptr(self.W2t), self.W2t.stride(0), _stream()))

    sync_all = sync_shadows

    def reset_optimizer(self):
        self.exp_avg.zero_()
        self.exp_avg_sq.zero_()
        self.steps = 0

    def _stage(self, images, fmt):
        n = images.shape[0]
        if n > self.max_batch:
            raise GmError("batch (%d) exceeds max_batch (%d)" % (n, self.max_batch))
        check(self.h, lib().gm_stage_images(self.h, _ptr(images.contiguous()), IMG_FMTS[fmt], None, _ptr(self.xb), n, self.X, self.XP, _stream()))
        return n

    def _encode(self, n):
        v = self.views()
        gemm_bf16(self.xb[:n], self.W1s, self.e[:n], "nt", K=self.X, bias=v[NAMES[1]], act=1, pad_one=True, out_cols=self.HP)

    def grad(self, images, fmt="f32"):
        """compute_batch + backward (src/ae.py:147-158,119-120): writes the flat gradient; returns the device loss (0-dim)."""
        n = self._stage(images, fmt)
        v = self.views()
        X, H = self.X, self.H
        self._encode(n)
        # decoder: out = sigmoid(e W2^T + b2); the epilogue emits sum (x - out)^2 per row and -2 (x - out) out (1 - out)
        gemm_bf16(self.e[:n], self.W2s, self.da[:n], "nt", K=H, bias=v[NAMES[3]], act=2, aux=self.xb[:n], aux_mode=3,
                  dot_out=self.slots, out_cols=X)
        self.loss_buf[0].copy_(self.slots[:, :n].sum())
        gemm_bf16(self.da[:n], self.e[:n], self.gw2, "tn", M=X, N=H + 1)                     # [dW2 | db2] = da^T [e | 1]
        gemm_bf16(self.da[:n], self.W2t, self.de[:n], "nt", K=X, aux=self.e[:n], aux_mode=2)  # de = (da W2) * 1[e > 0]
        gemm_bf16(self.de[:n], self.xb[:n], self.gw1, "tn", M=H, N=X + 1)                    # [dW1 | db1] = de^T [x | 1]
        g = self.views(self.grads)
        g[NAMES[0]].copy_(self.gw1[:, :X]); g[NAMES[1]].copy_(self.gw1[:, X])
        g[NAMES[2]].copy_(self.gw2[:, :H]); g[NAMES[3]].copy_(self.gw2[:, H])
        return self.loss_buf[0]

    def apply(self, hp):
        self.steps += 1
        adam_step(self.params, self.grads, self.exp_avg, self.exp_avg_sq, hp, self.steps)
        self.sync_shadows()

    def forward(self, images, fmt="f32", want_loss=False):
        """Autoencoder.forward (src/ae.py:63-64) without gradients -> (reconstruction [n, x] fp32, loss or None)."""
        n = self._stage(images, fmt)
        v = self.views()
        self._encode(n)
        out = torch.empty(n, self.X, device=self.device, dtype=torch.bfloat16)
        gemm_bf16(self.e[:n], self.W2s, out, "nt", K=self.H, bias=v[NAMES[3]], act=2)
        out = out.float()
        loss = None
        if want_loss:
            loss = torch.sum((self.xb[:n, :self.X].float() - out) ** 2)
        return out, loss

    def encode(self, images, fmt="f32"):
        n = self._stage(images, fmt)
        self._encode(n)
        return self.e[:n, :self.H].float()

    # ------------------------------------------------------------------ per-call encoder / decoder (user-written losses)
    # SLOTS encoder and SLOTS decoder calls keep their activations in their own buffers (allocated on first use) until their
    # backward ran.  A backward only reads them, so a call may be back-propagated more than once (retain_graph); its scratch
    # (da, de, gw1, gw2) is the fused step's (calls on one stream never overlap).
    SLOTS = 2

    def _slot(self, kind, slot):
        bufs = getattr(self, "_slots_" + kind, None)
        if bufs is None:
            bf = dict(device=self.device, dtype=torch.bfloat16)
            B = self.max_batch
            if kind == "enc":       # [x | 1], [relu(h) | 1], the code relu(h) fp32
                bufs = [(torch.zeros(B, self.XP, **bf), torch.zeros(B, self.HP, **bf),
                         torch.zeros(B, self.H, device=self.device)) for _ in range(self.SLOTS)]
            else:                   # [code | 1], the sigmoid output (its upstream after the backward)
                bufs = [(torch.zeros(B, self.HP, **bf), torch.zeros(B, self.XP, **bf)) for _ in range(self.SLOTS)]
            setattr(self, "_slots_" + kind, bufs)
        return bufs[slot]

    def slot_bytes(self):
        """device bytes one encoder slot and one decoder slot hold"""
        B = self.max_batch
        return B * (2 * self.XP + 2 * self.HP + 4 * self.H), B * (2 * self.HP + 2 * self.XP)

    def encoder_forward(self, slot, images):
        """Encoder.forward (src/ae.py:36-38): images [n, x] fp32 -> the code relu(W1 x + b1) [n, h] fp32 (the bf16 values the
        decoder reads, as encode)"""
        n = images.shape[0]
        if n > self.max_batch:
            raise GmError("batch (%d) exceeds max_batch (%d)" % (n, self.max_batch))
        xb, e, code = self._slot("enc", slot)
        check(self.h, lib().gm_stage_images(self.h, _ptr(images.contiguous()), IMG_FMTS["f32"], None, _ptr(xb), n, self.X, self.XP, _stream()))
        gemm_bf16(xb[:n], self.W1s, e[:n], "nt", K=self.X, bias=self.views()[NAMES[1]], act=1, pad_one=True, out_cols=self.HP)
        code[:n].copy_(e[:n, :self.H])
        return code[:n].clone()

    def encoder_backward(self, slot, n, dcode):
        """dcode [n, h] fp32 = dL/dcode of encoder_forward's call -> {encoder parameter name: gradient}: dh = dcode 1[h > 0]
        (gm_ae_dlatent_rows), [dW1 | db1] = dh^T [x | 1]"""
        xb, _, code = self._slot("enc", slot)
        X, H = self.X, self.H
        check(self.h, lib().gm_ae_dlatent_rows(self.h, _ptr(code), H, _ptr(dcode.float().contiguous()), H, _ptr(self.de), self.HP, n, H,
                                               _stream()))
        gemm_bf16(self.de[:n], xb[:n], self.gw1, "tn", M=H, N=X + 1)
        return {NAMES[0]: self.gw1[:, :X].clone(), NAMES[1]: self.gw1[:, X].clone()}

    def decoder_forward(self, slot, codes):
        """Decoder.forward (src/ae.py:49-50): codes [n, h] fp32 -> images sigmoid(W2 code + b2) [n, x] fp32 (as decode)"""
        n = codes.shape[0]
        if n > self.max_batch:
            raise GmError("batch (%d) exceeds max_batch (%d)" % (n, self.max_batch))
        e, out = self._slot("dec", slot)
        check(self.h, lib().gm_noise_rows(self.h, _ptr(codes.float().contiguous()), _ptr(e), n, self.H, self.HP, 0, 0, _stream()))
        gemm_bf16(e[:n], self.W2s, out[:n], "nt", K=self.H, bias=self.views()[NAMES[3]], act=2, out_cols=self.X)
        return out[:n, :self.X].float()

    def decoder_backward(self, slot, n, dimages):
        """dimages [n, x] fp32 = dL/d(images) of decoder_forward's call -> ({decoder parameter name: gradient}, dL/dcode [n, h]
        fp32): the sigmoid upstream da = dimages out (1 - out) formed in scratch from the slot's out (gm_sigmoid_upstream_rows),
        [dW2 | db2] = da^T [code | 1], dcode = da W2"""
        e, out = self._slot("dec", slot)
        X, H = self.X, self.H
        da = self.da[:n]
        da.copy_(out[:n])
        check(self.h, lib().gm_sigmoid_upstream_rows(self.h, _ptr(dimages.float().contiguous()), _ptr(da), n, X, self.XP, _stream()))
        gemm_bf16(da, e[:n], self.gw2, "tn", M=X, N=H + 1)
        dcode = torch.empty(n, H, device=self.device)
        gemm_bf16(da, self.W2t, dcode, "nt", K=X)
        return {NAMES[2]: self.gw2[:, :H].clone(), NAMES[3]: self.gw2[:, H].clone()}, dcode

    def decode(self, codes):
        n = codes.shape[0]
        e = torch.zeros(n, self.HP, device=self.device, dtype=torch.bfloat16)
        e[:, :self.H] = codes.to(torch.bfloat16)
        out = torch.empty(n, self.X, device=self.device, dtype=torch.bfloat16)
        gemm_bf16(e, self.W2s, out, "nt", K=self.H, bias=self.views()[NAMES[3]], act=2)
        return out.float()
