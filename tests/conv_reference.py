"""Plain float64 references of the conv building blocks (conv_ops.cuh), written from the index arithmetic of the
operations rather than from torch's conv ops, so that tests/test_conv_reference_cpu.py can pin them against torch on the
CPU and tests/test_conv_conformance_gpu.py can judge the CUDA kernels with them.  Every function takes torch tensors on
any device and returns float64 (or, where the operation is a pure data movement, the input's dtype)."""
import numpy as np
import torch

from oracle import ref_math as R

U_BF16 = 2.0 ** -8       # unit roundoff of bf16 (8 significant bits): round-to-nearest moves v by at most 2^-8 |v|
U_F32 = 2.0 ** -24       # unit roundoff of fp32


def bf16_rn(x):
    """float64 / float32 -> the nearest bf16 (ties to even), as float64"""
    return x.float().to(torch.bfloat16).double()


def im2col(x):
    """x [B, H, W, C] -> col [B * H/2 * W/2, 16 C], columns ordered (kh, kw, c); kernel 4, stride 2, zero padding 1"""
    B, H, W, C = x.shape
    Ho, Wo = H // 2, W // 2
    xp = torch.zeros(B, H + 2, W + 2, C, dtype=x.dtype, device=x.device)
    xp[:, 1:H + 1, 1:W + 1] = x
    taps = [xp[:, kh:kh + 2 * Ho:2, kw:kw + 2 * Wo:2] for kh in range(4) for kw in range(4)]     # input row 2 ho - 1 + kh
    return torch.stack(taps, 3).reshape(B * Ho * Wo, 16 * C)


def col2im(col, B, Hi, Wi, C):
    """col [B * Hi * Wi, 16 C] (float64) -> (sum, sum of magnitudes), each [B, 2 Hi, 2 Wi, C]: output pixel (2 iy - 1 + kh,
    2 ix - 1 + kw) receives tap (kh, kw) of input pixel (iy, ix)"""
    c5 = col.reshape(B, Hi, Wi, 16, C)
    out = torch.zeros(2, B, 2 * Hi + 2, 2 * Wi + 2, C, dtype=torch.float64, device=col.device)
    for kh in range(4):
        for kw in range(4):
            t = c5[:, :, :, kh * 4 + kw]
            out[0, :, kh:kh + 2 * Hi:2, kw:kw + 2 * Wi:2] += t
            out[1, :, kh:kh + 2 * Hi:2, kw:kw + 2 * Wi:2] += t.abs()
    return out[0, :, 1:-1, 1:-1], out[1, :, 1:-1, 1:-1]


def border_class(B, Ho, Wo, device):
    """[B, Ho, Wo] int: 2 corner, 1 edge, 0 interior pixel of an Ho x Wo image"""
    ey = torch.zeros(Ho, dtype=torch.int64, device=device)
    ex = torch.zeros(Wo, dtype=torch.int64, device=device)
    ey[0] = ey[-1] = 1
    ex[0] = ex[-1] = 1
    return (ey[:, None] + ex[None, :]).expand(B, Ho, Wo)


def lrelu_mask(x, m, slope):
    """x * LeakyReLU'(m) as the kernels store it: x where m > 0, else bf16_rn(fp32(slope) * x in fp32)"""
    sl = torch.tensor(slope, dtype=torch.float32, device=x.device)
    return torch.where(m.float() > 0, x.double(), bf16_rn(sl * x.float()))


def act(pre, kind, slope):
    if kind == 1:
        return pre.clamp_min(0)
    if kind == 2:
        return torch.where(pre > 0, pre, slope * pre)
    return pre


def act_grad(pre, kind, slope):
    one = torch.ones_like(pre)
    if kind == 1:
        return (pre > 0).double()
    if kind == 2:
        return torch.where(pre > 0, one, slope * one)
    return one


def bn_stats(x):
    """column mean, biased variance and mean of squares of x [rows, C] in float64"""
    x = x.double()
    mean = x.mean(0)
    return mean, ((x - mean) ** 2).mean(0), (x * x).mean(0)


def bn_running(running, mean, var, rows, momentum):
    """torch's update of (running_mean, running_var): momentum, unbiased variance"""
    unb = var * rows / max(rows - 1, 1)
    return torch.stack([(1 - momentum) * running[0].double() + momentum * mean, (1 - momentum) * running[1].double() + momentum * unb])


def bn_forward(x, mean, invstd, gamma, beta, kind, slope):
    """-> (pre-activation, y) of y = act(gamma (x - mean) invstd + beta), all float64"""
    pre = gamma.double() * (x.double() - mean.double()) * invstd.double() + beta.double()
    return pre, act(pre, kind, slope)


def bn_backward(dy, x, mean, invstd, gamma, beta, kind, slope, dgb=None):
    """BatchNorm backward at given (mean, invstd): g = dy act'(pre), dbeta = sum g, dgamma = sum g xhat,
    dx = gamma invstd (g - (dbeta + xhat dgamma) / N), with dgb = (dbeta, dgamma) taken as given when passed.
    -> dict(pre, xhat, g, dbeta, dgamma, dx, mag) with mag = |gamma invstd| (|g| + (|dbeta| + |xhat| |dgamma|) / N)"""
    x, dy = x.double(), dy.double()
    n = x.shape[0]
    xh = (x - mean.double()) * invstd.double()
    pre = gamma.double() * xh + beta.double()
    g = dy * act_grad(pre, kind, slope)
    dbeta, dgamma = g.sum(0), (g * xh).sum(0)
    ub, ug = (dbeta, dgamma) if dgb is None else (dgb[0].double(), dgb[1].double())
    sc = gamma.double() * invstd.double()
    dx = sc * (g - (ub + xh * ug) / n)
    mag = sc.abs() * (g.abs() + (ub.abs() + xh.abs() * ug.abs()) / n)
    return dict(pre=pre, xhat=xh, g=g, dbeta=dbeta, dgamma=dgamma, dx=dx, mag=mag)


def noise_rows(noise, ld):
    """[rows, z] fp32 -> bf16 [rows, ld]: the noise rounded to nearest even, 1 at column z, zeros after"""
    rows, z = noise.shape
    out = torch.zeros(rows, ld, dtype=torch.bfloat16, device=noise.device)
    out[:, :z] = noise.to(torch.bfloat16)
    out[:, z] = 1
    return out


def stage_images(images, fmt, rows_idx, x, ld):
    """images in format fmt ("f32": [n, x] fp32; "u8": [n, x] uint8, non-zero -> 1; "bits": np.packbits of the flattened
    [n, x] bits, most significant bit first) -> bf16 [len(rows_idx), ld] with the ones column at x"""
    dev = images.device
    if fmt == "f32":
        v = images.to(torch.bfloat16)
    elif fmt == "u8":
        v = (images != 0).to(torch.bfloat16)
    else:
        bits = np.unpackbits(images.cpu().numpy().reshape(-1))
        n = bits.size // x
        v = torch.from_numpy(bits[:n * x].reshape(n, x).astype(np.float32)).to(dev).to(torch.bfloat16)
    out = torch.zeros(len(rows_idx), ld, dtype=torch.bfloat16, device=dev)
    out[:, :x] = v[rows_idx.to(dev).long()]
    out[:, x] = 1
    return out


ROW_VARIANTS = ["ns", "mm", "w", "ls", "f_total_variation", "f_forward_kl", "f_reverse_kl", "f_pearson", "f_hellinger", "f_jensen_shannon"]


def d_out(s, out_act):
    """D's output from the logit (float64 numpy)"""
    if out_act == "sigmoid":
        return R.sigmoid(s)
    return np.maximum(s, 0) if out_act == "relu" else s


def loss_rows(variant, out_act, s, d, batch, g_step):
    """The row-wise adversarial losses of oracle/ref_math.py at given logits s and outputs d (float64 numpy; D step: batch
    real rows then batch fake rows, G step: batch fake rows).  -> (loss, ds [rows])"""
    s, d = s.reshape(-1, 1), d.reshape(-1, 1)
    if g_step:
        L, dd = R.g_loss(variant, d)
        dd = dd * np.ones_like(d)
    else:
        L, gx, gg = R.d_loss(variant, d[:batch], d[batch:])
        dd = np.concatenate([gx * np.ones_like(d[:batch]), gg * np.ones_like(d[batch:])])
    ds = R.d_out_grad(dict(d=d, s=s), dd, out_act)
    return float(L), ds.reshape(-1)
