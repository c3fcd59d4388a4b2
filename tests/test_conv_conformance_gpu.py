"""Elementwise conformance of the conv building blocks shared by every DCGAN-path variant (conv_ops.cuh through the C ABI
of engine_conv.inl), against float64 references computed from the same bf16 inputs (tests/conv_reference.py) (GPU).

Layout of every case: inputs and outputs are views into larger buffers whose leading dimension is the logical width + 8 or
+ 16 (or + 0: contiguous).  Input padding holds bf16 NaN, outputs are prefilled with 0x4B4B; outside the logical block
every output byte must be unchanged and no NaN may reach an output or a statistic.

Bounds (u = 2^-24 fp32, U = 2^-8 bf16 unit roundoff; a bf16 store of a value f carrying an error m: |got - f| <= U (|f| + m) + m):
  im2col, masked im2col, lrelu_mask_rows, cast, pack_col0, noise rows of a caller tensor, stage_images: exact.
  col2im: s = fp32 sum of <= 4 taps in a fixed order, e = 3 u sum|taps|.  mode 0: f = s, m = e.  mode 1: f = sigmoid(s) by
      1 / (1 + __expf(-s)); __expf is off by at most 2 + |1.4427 s| ulp, d sigmoid / d E = -sigmoid^2, so
      m = e / 4 + sigmoid ((2 + 1.4427 |s|) 2 u (1 - sigmoid) + 2 u).  mode 2: f = s k, k = 1 (aux > 0) or slope, m = |k| e + u |f|.
      mode 3: f = s a (1 - a), m = |a (1 - a)| e + 3 u |f|.  Corner, edge and interior pixels are separate groups.
  BatchNorm statistics: a thread sums 64 rows in fp32 before it flushes into doubles, so sum x and sum x^2 are off by at
      most 64 u = 2^-18 of sum|x| and sum x^2: |mean - ref| <= 2^-18 mean|x| + u |ref|, dvar = 2^-18 (E[x^2] + 2 |mean| mean|x|),
      and invstd lies within the image of [var - dvar, var + dvar] (clamped at 0) under (v + eps)^-1/2, + 2 u.  The running
      statistics carry momentum times those + 4 u of the summed magnitudes.
  BatchNorm y, at the statistics the kernel stored: fma(x, sc, sh), sc = gamma invstd, sh = beta - mean sc:
      m = 4 u (|x sc| + |mean sc| + |beta|).  A unit within m of the kink moves by less than m: no exclusion needed.
  BatchNorm backward, at the stored statistics: g = dy act'(pre).  dbeta: 2^-18 sum|g| + u |dbeta|; dgamma: (2^-18 + 4 u)
      sum|g xhat| + u |dgamma|; both + the |g| (|g xhat|) of the units at the kink, |pre| <= 8 u (|gamma xhat| + |beta|), which may
      take either slope.  Those units are left out of the dx check, counted, and must stay below 0.1 % of the tensor.
      dx, at the stored (dbeta, dgamma): m = 8 u M, M = |gamma invstd| (|g| + (|dbeta| + |xhat| |dgamma|) / N) - the summed
      magnitudes, because the expression cancels (a dy that is constant per column must give dx = 0 within that m).
  gm_loss_rows: d against float64 act(s) (sigmoid by expf, a sum and a division: 8 u d); ds and the loss against oracle/ref_math.py evaluated at the stored d:
      |ds - ref| <= 16 u (|ref| + inv |act'| (1 + |d|)), |loss - ref| <= 8 u (|ref| + mean(1 + 2 |d| (+ e^|d| for f-GAN))).
With GM_PARITY_DIR set, the worst error-to-bound ratio of each group goes to $GM_PARITY_DIR/parity_conv_conformance.json."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import conv_reference as CR
import dcgan_harness as H

pytestmark = pytest.mark.gpu
_REPORT = H.Report("conv_conformance")

U, UB = CR.U_F32, CR.U_BF16
PAT16, PAT32 = 0x4B4B, 0x4B4B4B4B
SLOPE, EPS, MOM = 0.2, 1e-5, 0.1
SM_REF = 132                        # SM count of an H100 SXM: the case tables are sized for it (checked on the CPU)
UNROLL = dict(im2col=4, im2col_mask=4, col2im_vec=2, col2im_scalar=1, lrelu_rows=1, bn=4)
MAX_CASE_BYTES = 1 << 30
GM_ERR_ARG, GM_ERR_UNSUPPORTED = -1, -4
VARIANT_ID = {"ns": 0, "mm": 1, "w": 2, "wgp": 3, "ls": 4, "dra": 5, "ra": 6, "fisher": 7, "f_total_variation": 8,
              "f_forward_kl": 9, "f_reverse_kl": 10, "f_pearson": 11, "f_hellinger": 12, "f_jensen_shannon": 13, "info": 14, "began": 15}
OUT_ACT_ID = {"sigmoid": 0, "relu": 1, "none": 2}

# (B, H, W, C): H x W is the input grid of im2col (even) and of col2im (any).  C 1..7 takes col2im's scalar path, 12 only
# im2col's; 24, 40, 136 leave idle lanes in BatchNorm's thread mapping (256 % (C/8) != 0); 6x10 and 12x20 take FastDiv's
# division path; 2x2 and 4x4 make every output pixel a border pixel.  The last rows run more than two sweeps of the
# grid-stride loops on 132 SMs (sweep_items()) with a ragged tail.
SHAPES = [(1, 2, 2, 1), (3, 4, 4, 3), (5, 6, 10, 4), (3, 12, 20, 7), (1, 32, 32, 12), (1, 2, 2, 8), (3, 4, 4, 24), (5, 6, 10, 40),
          (3, 12, 20, 64), (1, 32, 32, 136), (3, 64, 64, 8), (1, 6, 10, 256), (3, 4, 4, 512), (1, 12, 20, 1024), (5, 2, 2, 2048),
          (5, 32, 32, 24), (1, 64, 64, 64)]
SWEEPS_IM2COL = [(67, 32, 32, 64), (9, 64, 64, 136)]
SWEEPS_COL2IM = [(35, 32, 32, 64), (3, 64, 64, 256), (37, 64, 64, 3)]
# BatchNorm (rows, C): the C % 8 == 0 rows of SHAPES as B H W rows, rows = 1 and 2, and three multi-sweep cases
BN_SHAPES = [(b * h * w, c) for b, h, w, c in SHAPES if c % 8 == 0] + [(1, 8), (2, 64), (1013, 24), (4133, 64)]
SWEEPS_BN = [(300037, 64), (40005, 512), (9001, 2048)]
SWEEPS_LRELU = [(140003, 64), (9001, 2048)]


def pad_of(i):
    """leading-dimension padding of case i: + 8, + 16, contiguous, in turn"""
    return (8, 16, 0)[i % 3]


def sweep_items(kernel, C=64, sms=SM_REF):
    """items one sweep of a kernel's grid-stride loop covers on `sms` SMs (BatchNorm: rows)"""
    if kernel == "bn":
        return sms * 8 * (256 // (C // 8)) * UNROLL["bn"]
    return sms * 8 * 256 * UNROLL[kernel]


def items_of(kernel, shape):
    """the item count of a multi-sweep case, as the entry points compute it"""
    if kernel == "bn" or kernel == "lrelu_rows":
        return shape[0] if kernel == "bn" else shape[0] * (shape[1] // 8)
    b, h, w, c = shape
    if kernel in ("im2col", "im2col_mask"):
        return b * (h // 2) * (w // 2) * 16 * (c // 8 if c % 8 == 0 else 1)
    return b * 4 * h * w * (c // 8 if c % 8 == 0 else 1)


def case_bytes(kind, shape, pad=16):
    """device bytes of the kernel's own buffers of a case (bf16 operands)"""
    if kind == "bn":
        return 3 * shape[0] * (shape[1] + pad) * 2
    b, h, w, c = shape
    if kind == "im2col":
        return 2 * (b * h * w * (c + pad) * 2 + b * (h // 2) * (w // 2) * (16 * c + pad))
    return 2 * (b * h * w * (16 * c + pad) + 2 * b * 4 * h * w * (c + pad))


# ------------------------------------------------------------------ library, buffers, bookkeeping
def _lib():
    from gm_b200 import _lib as M
    return M.lib(), M.ctx(), M._stream(), M


def _ok(rc):
    L, h, _, M = _lib()
    M.check(h, rc)


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, device="cuda", generator=g)


def _in(vals, ld, extra=3):
    """vals [rows, w] bf16 inside a NaN-filled [rows + extra, ld] buffer"""
    rows, w = vals.shape
    buf = torch.full((rows + extra, ld), float("nan"), device="cuda", dtype=torch.bfloat16)
    buf[:rows, :w] = vals
    return buf


def _out(rows, ld, extra=2):
    return torch.full((rows + extra, ld), PAT16, device="cuda", dtype=torch.int16).view(torch.bfloat16)


def _untouched(buf, rows, w):
    bits = buf.view(torch.int16)
    return bool((bits[rows:] == PAT16).all()) and bool((bits[:, w:] == PAT16).all())


def _f32(n, extra=3):
    return torch.full((n + extra,), PAT32, device="cuda", dtype=torch.int32).view(torch.float32)


def _f32_untouched(buf, n):
    return bool((buf.view(torch.int32)[n:] == PAT32).all())


def _ratio(err, tol):
    """worst err / tol; where tol is 0 only an exact match passes"""
    r = torch.where(tol > 0, err / tol.clamp_min(1e-300), torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max()) if r.numel() else 0.0


def _bf16_tol(f, m):
    return UB * (f.abs() + m) + m


_WORST = {}


def _record(group, name, ratio):
    if ratio >= _WORST.get(group, (-1.0, ""))[0]:
        _WORST[group] = (ratio, name)
        _REPORT.add(group, {"worst_ratio": ratio, "case": name})
    assert ratio <= 1, (group, name, ratio)


def _specials(t):
    """plant +0, -0, the smallest positive and negative bf16, +inf and -inf in the first values of a bf16 tensor"""
    bits = torch.tensor([0x0000, 0x8000, 0x0001, 0x8001, 0x7F80, 0xFF80], dtype=torch.int32).to(torch.int16).cuda()
    flat = t.view(torch.int16).view(-1)
    n = min(flat.numel(), 6)
    flat[:n] = bits[:n]
    return t


def _name(shape):
    return "x".join(str(v) for v in shape)


# ------------------------------------------------------------------ im2col
IM2COL_CASES = [(s, pad_of(i)) for i, s in enumerate(SHAPES + SWEEPS_IM2COL)]


def _run_im2col(shape, pad, seed=1):
    L, h, st, _ = _lib()
    B, Hh, W, Cc = shape
    g = _gen(seed)
    x = _randn(g, B * Hh * W, Cc).to(torch.bfloat16)
    xb = _in(x, Cc + pad)
    rows = B * (Hh // 2) * (W // 2)
    col = _out(rows, 16 * Cc + pad)
    _ok(L.gm_im2col_k4s2(h, _p(xb), B, Hh, W, Cc, Cc + pad, _p(col), 16 * Cc + pad, st))
    torch.cuda.synchronize()
    return x, col, rows


@pytest.mark.parametrize("shape,pad", IM2COL_CASES, ids=["%s_pad%d" % (_name(s), p) for s, p in IM2COL_CASES])
def test_im2col_is_bit_exact(shape, pad):
    B, Hh, W, Cc = shape
    x, col, rows = _run_im2col(shape, pad)
    ref = CR.im2col(x.view(B, Hh, W, Cc))
    assert torch.equal(col[:rows, :16 * Cc].view(torch.int16), ref.view(torch.int16)), shape      # zeros at the border are +0
    assert _untouched(col, rows, 16 * Cc), shape


MASK_SHAPES = [s for s in SHAPES if s[3] % 8 == 0] + SWEEPS_IM2COL[:2]
MASK_CASES = [(s, pad_of(i + 1)) for i, s in enumerate(MASK_SHAPES)]


@pytest.mark.parametrize("shape,pad", MASK_CASES, ids=["%s_pad%d" % (_name(s), p) for s, p in MASK_CASES])
def test_im2col_lrelu_mask_is_exact(shape, pad):
    L, h, st, _ = _lib()
    B, Hh, W, Cc = shape
    g = _gen(2)
    x = _randn(g, B * Hh * W, Cc).to(torch.bfloat16)
    m = _specials(_randn(g, B * Hh * W, Cc).to(torch.bfloat16))
    xb, mb = _in(x, Cc + pad), _in(m, Cc + 24 - pad)
    rows = B * (Hh // 2) * (W // 2)
    col = _out(rows, 16 * Cc + pad)
    _ok(L.gm_im2col_k4s2_lrelu_mask(h, _p(xb), B, Hh, W, Cc, Cc + pad, _p(mb), Cc + 24 - pad, SLOPE, _p(col), 16 * Cc + pad, st))
    torch.cuda.synchronize()
    ref = CR.im2col(CR.lrelu_mask(x, m, SLOPE).view(B, Hh, W, Cc))
    got = col[:rows, :16 * Cc]
    assert torch.equal(got.double(), ref), shape
    # where the mask is positive the value passes through bit for bit
    on = CR.im2col((m.float() > 0).view(B, Hh, W, Cc))
    assert torch.equal(got.view(torch.int16)[on], CR.im2col(x.view(B, Hh, W, Cc)).view(torch.int16)[on]), shape
    assert _untouched(col, rows, 16 * Cc), shape


LRELU_ROWS = [(r, c) for r, c in BN_SHAPES[:8]] + SWEEPS_LRELU
LRELU_CASES = [(s, pad_of(i), alias) for i, s in enumerate(LRELU_ROWS) for alias in ("none", "x", "m")]


@pytest.mark.parametrize("shape,pad,alias", LRELU_CASES, ids=["%s_pad%d_alias_%s" % (_name(s), p, a) for s, p, a in LRELU_CASES])
def test_lrelu_mask_rows_is_exact(shape, pad, alias):
    L, h, st, _ = _lib()
    rows, Cc = shape
    g = _gen(3)
    x = _randn(g, rows, Cc).to(torch.bfloat16)
    m = _specials(_randn(g, rows, Cc).to(torch.bfloat16))
    xb, mb = _in(x, Cc + pad), _in(m, Cc + 24 - pad)
    out = {"none": _out(rows, Cc + 8, extra=3), "x": xb, "m": mb}[alias]
    _ok(L.gm_lrelu_mask_rows(h, _p(xb), Cc + pad, _p(mb), Cc + 24 - pad, rows, Cc, SLOPE, _p(out), out.stride(0), st))
    torch.cuda.synchronize()
    ref = CR.lrelu_mask(x, m, SLOPE)
    got = out[:rows, :Cc]
    assert torch.equal(got.double(), ref), shape
    on = m.float() > 0
    assert torch.equal(got.view(torch.int16)[on], x.view(torch.int16)[on]), shape
    if alias == "none":
        assert _untouched(out, rows, Cc), shape
    else:       # the padding of the aliased operand still holds its NaN
        assert bool(torch.isnan(out[rows:]).all()) and bool(torch.isnan(out[:, Cc:]).all()), shape


# ------------------------------------------------------------------ col2im
COL2IM_SHAPES = [s for s in SHAPES if s[3] % 8 == 0 or s[3] < 8] + SWEEPS_COL2IM
COL2IM_CASES = [(s, mode, pad_of(i + mode)) for i, s in enumerate(COL2IM_SHAPES) for mode in range(4)]


def _run_col2im(shape, mode, pad, seed=4):
    L, h, st, _ = _lib()
    B, Hi, Wi, Cc = shape
    g = _gen(seed + mode)
    col = _randn(g, B * Hi * Wi, 16 * Cc).to(torch.bfloat16)
    rows = B * 4 * Hi * Wi
    aux = None
    if mode == 2:
        aux = _specials(_randn(g, rows, Cc).to(torch.bfloat16))
    elif mode == 3:
        aux = torch.rand(rows, Cc, device="cuda", generator=g).to(torch.bfloat16)
    vec = Cc % 8 == 0
    ldc, ldy, lda = 16 * Cc + pad, Cc + (24 - pad if vec else 5), Cc + (pad + 8 if vec else 3)
    cb = _in(col, ldc)
    ab = _in(aux, lda) if aux is not None else None
    y = _out(rows, ldy)
    _ok(L.gm_col2im_k4s2(h, _p(cb), ldc, B, Hi, Wi, Cc, _p(y), ldy, mode, _p(ab), lda if ab is not None else 0, SLOPE, st))
    torch.cuda.synchronize()
    return col, aux, y, rows


def _col2im_reference(shape, mode, col, aux):
    """-> (f, m) [rows, C]: the float64 value and the error it may carry before the bf16 store"""
    B, Hi, Wi, Cc = shape
    s, sabs = CR.col2im(col.double(), B, Hi, Wi, Cc)
    s, e = s.reshape(-1, Cc), 3 * U * sabs.reshape(-1, Cc)
    if mode == 0:
        return s, e
    if mode == 1:
        f = torch.sigmoid(s)
        return f, e / 4 + f * ((2 + 1.4427 * s.abs()) * 2 * U * (1 - f) + 2 * U)
    a = aux.double()
    if mode == 2:
        k = torch.where(a > 0, torch.ones_like(a), torch.full_like(a, float(np.float32(SLOPE))))
        return s * k, k * e + U * (s * k).abs()
    k = a * (1 - a)
    return s * k, k.abs() * e + 3 * U * (s * k).abs()


@pytest.mark.parametrize("shape,mode,pad", COL2IM_CASES, ids=["%s_mode%d_pad%d" % (_name(s), m, p) for s, m, p in COL2IM_CASES])
def test_col2im_matches_float64(shape, mode, pad):
    B, Hi, Wi, Cc = shape
    col, aux, y, rows = _run_col2im(shape, mode, pad)
    f, m = _col2im_reference(shape, mode, col, aux)
    got = y[:rows, :Cc]
    assert bool(torch.isfinite(got).all()), shape
    assert _untouched(y, rows, Cc), shape
    err, tol = (got.double() - f).abs(), _bf16_tol(f, m)
    cls = CR.border_class(B, 2 * Hi, 2 * Wi, "cuda").reshape(-1)
    for k, where in enumerate(("interior", "edge", "corner")):
        sel = cls == k
        if bool(sel.any()):
            _record("col2im_mode%d_%s" % (mode, where), _name(shape), _ratio(err[sel], tol[sel]))


# ------------------------------------------------------------------ BatchNorm
DATASETS = ("normal", "offset", "constant", "outlier")


def _bn_data(g, rows, Cc, data):
    x = _randn(g, rows, Cc) * 1.5 + 0.3
    if data == "offset":            # E[x^2] - mean^2 cancels 3600 : 1
        x = 30 + 0.5 * _randn(g, rows, Cc)
    elif data == "constant":        # even columns constant: variance 0, invstd = eps^-1/2
        x[:, 0::2] = 1.5
    elif data == "outlier":         # even columns zero but for one row
        x[:, 0::2] = 0
        x[rows // 2, 0::2] = 100
    return x.to(torch.bfloat16)


def _bn_params(g, Cc):
    return (1 + 0.1 * _randn(g, Cc)).float(), (0.1 * _randn(g, Cc)).float()


BN_FWD_CASES = [(s, (i + j) % 3, DATASETS[0], pad_of(i + j)) for i, s in enumerate(BN_SHAPES + SWEEPS_BN) for j in range(2)]
BN_FWD_CASES += [((1013, 24), k, d, pad_of(k)) for k in range(3) for d in DATASETS[1:]] + [((4133, 64), 2, d, 8) for d in DATASETS[1:]]
_bn_id = lambda c: "%s_act%d_%s_pad%d" % (_name(c[0]), c[1], c[2], c[3])


def _run_bn_forward(shape, act, data, pad, running=True, seed=5):
    L, h, st, _ = _lib()
    rows, Cc = shape
    g = _gen(seed)
    x = _bn_data(g, rows, Cc, data)
    gamma, beta = _bn_params(g, Cc)
    xb = _in(x, Cc + pad)
    y = _out(rows, Cc + 24 - pad)
    stats = _f32(2 * Cc)
    run0 = torch.stack([0.2 * _randn(g, Cc), 0.5 + torch.rand(Cc, device="cuda", generator=g)]).contiguous() if running else None
    run = run0.clone() if running else None
    _ok(L.gm_bn_forward(h, _p(xb), rows, Cc, Cc + pad, _p(gamma), _p(beta), EPS, act, SLOPE, _p(y), Cc + 24 - pad, _p(stats), _p(run), MOM, st))
    torch.cuda.synchronize()
    return dict(x=x, xb=xb, gamma=gamma, beta=beta, y=y, stats=stats, run0=run0, run=run)


def _check_bn_y(name, T, mean, invstd, act, group):
    rows, Cc = T["x"].shape
    _, f = CR.bn_forward(T["x"], mean, invstd, T["gamma"], T["beta"], act, SLOPE)
    sc = (T["gamma"].double() * invstd.double()).abs()
    m = 4 * U * (T["x"].double().abs() * sc + mean.double().abs() * sc + T["beta"].double().abs())
    got = T["y"][:rows, :Cc]
    assert bool(torch.isfinite(got).all()), name
    assert _untouched(T["y"], rows, Cc), name
    _record(group, name, _ratio((got.double() - f).abs(), _bf16_tol(f, m)))


@pytest.mark.parametrize("case", BN_FWD_CASES, ids=[_bn_id(c) for c in BN_FWD_CASES])
def test_bn_forward_matches_float64(case):
    shape, act, data, pad = case
    rows, Cc = shape
    name = _bn_id(case)
    T = _run_bn_forward(shape, act, data, pad, running=(pad != 16))      # a third of the cases pass running == NULL
    st = T["stats"][:2 * Cc].double().view(2, Cc)
    assert bool(torch.isfinite(st).all()) and _f32_untouched(T["stats"], 2 * Cc), name
    x64 = T["x"].double()
    mean, var, ex2 = CR.bn_stats(x64)
    mabs = x64.abs().mean(0)
    tol_mean = 2.0 ** -18 * mabs + U * mean.abs()
    _record("bn_mean_" + data, name, _ratio((st[0] - mean).abs(), tol_mean))
    dvar = 2.0 ** -18 * (ex2 + 2 * mean.abs() * mabs)
    inv = lambda v: (v + EPS) ** -0.5
    tol_inv = torch.maximum(inv((var - dvar).clamp_min(0)) - inv(var), inv(var) - inv(var + dvar)) + 2 * U * inv(var)
    _record("bn_invstd_" + data, name, _ratio((st[1] - inv(var)).abs(), tol_inv))
    if data == "constant":      # 1.5 and 2.25 sum exactly in fp32: the variance is exactly 0
        assert bool(((st[1, 0::2] - EPS ** -0.5).abs() <= 2 * U * EPS ** -0.5).all()), name
    if T["run"] is not None:
        ref = CR.bn_running(T["run0"], mean, var, rows, MOM)
        unb = rows / max(rows - 1, 1)
        tol = torch.stack([MOM * tol_mean + 4 * U * ((1 - MOM) * T["run0"][0].double().abs() + MOM * mean.abs()),
                           MOM * dvar * unb + 4 * U * ((1 - MOM) * T["run0"][1].double().abs() + MOM * var * unb)])
        _record("bn_running_" + data, name, _ratio((T["run"].double() - ref).abs(), tol))
    _check_bn_y(name, T, st[0], st[1], act, "bn_y_act%d" % act)


BN_EVAL_CASES = [(s, i % 3, pad_of(i)) for i, s in enumerate(BN_SHAPES[::2] + SWEEPS_BN[1:])]


@pytest.mark.parametrize("shape,act,pad", BN_EVAL_CASES, ids=["%s_act%d_pad%d" % (_name(s), a, p) for s, a, p in BN_EVAL_CASES])
def test_bn_forward_eval_matches_float64(shape, act, pad):
    L, h, st, _ = _lib()
    rows, Cc = shape
    g = _gen(6)
    x = _bn_data(g, rows, Cc, "normal")
    gamma, beta = _bn_params(g, Cc)
    run = torch.stack([0.3 * _randn(g, Cc), 0.5 + 2 * torch.rand(Cc, device="cuda", generator=g)]).contiguous()
    keep = run.clone()
    T = dict(x=x, gamma=gamma, beta=beta, y=_out(rows, Cc + 24 - pad))
    xb = _in(x, Cc + pad)
    _ok(L.gm_bn_forward_eval(h, _p(xb), rows, Cc, Cc + pad, _p(gamma), _p(beta), _p(run), EPS, act, SLOPE, _p(T["y"]), Cc + 24 - pad, st))
    torch.cuda.synchronize()
    assert torch.equal(run.view(torch.int32), keep.view(torch.int32)), shape
    _check_bn_y(_name(shape), T, run[0].double(), (run[1].double() + EPS) ** -0.5, act, "bn_eval_y")


BN_BWD_CASES = [(s, (i + 1) % 3, "normal", pad_of(i)) for i, s in enumerate(BN_SHAPES + SWEEPS_BN)]
BN_BWD_CASES += [((1013, 24), k, "offset", 16) for k in range(3)] + [((4133, 64), 0, "common_mode", 8), ((1013, 24), 0, "common_mode", 0),
                                                                       ((40005, 512), 0, "common_mode", 16)]


def _run_bn_backward(case, seed=7):
    L, h, st, _ = _lib()
    shape, act, data, pad = case
    rows, Cc = shape
    T = _run_bn_forward(shape, act, "normal" if data == "common_mode" else data, pad, running=False, seed=seed)
    g = _gen(seed + 1)
    dy = _randn(g, rows, Cc)
    if data == "common_mode":           # the same upstream gradient for every row of a column
        dy = _randn(g, 1, Cc).expand(rows, Cc)
    dy = dy.to(torch.bfloat16).contiguous()
    T["dy"] = dy
    dyb = _in(dy, Cc + pad)             # dy is read with x's leading dimension
    T["dx"] = _out(rows, Cc + 24 - pad)
    T["dgb"] = _f32(2 * Cc)
    _ok(L.gm_bn_backward(h, _p(dyb), _p(T["xb"]), rows, Cc, Cc + pad, _p(T["stats"]), _p(T["gamma"]), _p(T["beta"]), act, SLOPE, _p(T["dx"]),
                         Cc + 24 - pad, _p(T["dgb"]), st))
    torch.cuda.synchronize()
    return T


@pytest.mark.parametrize("case", BN_BWD_CASES, ids=[_bn_id(c) for c in BN_BWD_CASES])
def test_bn_backward_matches_float64(case):
    shape, act, data, pad = case
    rows, Cc = shape
    name = _bn_id(case)
    T = _run_bn_backward(case)
    st = T["stats"][:2 * Cc].view(2, Cc)
    dgb = T["dgb"][:2 * Cc].view(2, Cc)
    assert bool(torch.isfinite(dgb).all()) and _f32_untouched(T["dgb"], 2 * Cc), name
    r = CR.bn_backward(T["dy"], T["x"], st[0], st[1], T["gamma"], T["beta"], act, SLOPE)
    kink = torch.zeros_like(r["pre"], dtype=torch.bool)
    if act:
        kink = r["pre"].abs() <= 8 * U * ((T["gamma"].double() * r["xhat"]).abs() + T["beta"].double().abs())
    assert int(kink.sum()) <= 1e-3 * kink.numel() + 1, (name, int(kink.sum()))
    gk = T["dy"].double().abs() * kink
    tol_b = 2.0 ** -18 * r["g"].abs().sum(0) + U * r["dbeta"].abs() + gk.sum(0)
    tol_g = (2.0 ** -18 + 4 * U) * (r["g"] * r["xhat"]).abs().sum(0) + U * r["dgamma"].abs() + (gk * r["xhat"].abs()).sum(0)
    _record("bn_dbeta", name, _ratio((dgb[0].double() - r["dbeta"]).abs(), tol_b))
    _record("bn_dgamma", name, _ratio((dgb[1].double() - r["dgamma"]).abs(), tol_g))
    r = CR.bn_backward(T["dy"], T["x"], st[0], st[1], T["gamma"], T["beta"], act, SLOPE, dgb=dgb)
    got = T["dx"][:rows, :Cc]
    assert bool(torch.isfinite(got).all()) and _untouched(T["dx"], rows, Cc), name
    err, tol = (got.double() - r["dx"]).abs(), _bf16_tol(r["dx"], 8 * U * r["mag"])
    _record("bn_dx_common_mode" if data == "common_mode" else "bn_dx_act%d" % act, name, _ratio(err[~kink], tol[~kink]))
    if data == "common_mode":           # BatchNorm rejects the common mode: what is left is rounding of the summed magnitudes
        assert float((got.double().abs() / r["mag"].clamp_min(1e-300)).max()) <= 2.0 ** -9, name


# ------------------------------------------------------------------ cast, pack, noise, images
DIMS = (1, 3, 48, 1005, 2048)
CAST_CASES = [(r, c, which) for r in DIMS for c in DIMS for which in ("dst", "dst_t", "both")]


@pytest.mark.parametrize("R,Cc,which", CAST_CASES, ids=["%dx%d_%s" % c for c in CAST_CASES])
def test_cast_bf16_is_bit_exact(R, Cc, which):
    L, h, st, _ = _lib()
    g = _gen(8)
    src = _randn(g, R * Cc)
    # ties of the bf16 rounding (to even, both ways), an fp32 subnormal, infinities, NaN
    sp = torch.tensor([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -1 - 2.0 ** -8, 1e-40, -1e-40, math.inf, -math.inf, math.nan, 3.3895e38, 0.0],
                      device="cuda")
    src[:min(R * Cc, sp.numel())] = sp[:R * Cc]
    src = src.view(R, Cc)
    ld, ldt = Cc + (3, 8)[R % 2], R + (8, 5)[Cc % 2]
    dst = _out(R, ld) if which != "dst_t" else None
    dstt = _out(Cc, ldt) if which != "dst" else None
    _ok(L.gm_cast_bf16(h, _p(src), R, Cc, _p(dst), ld, _p(dstt), ldt, st))
    torch.cuda.synchronize()
    ref = src.to(torch.bfloat16)
    for out, want, rr, cc in ((dst, ref, R, Cc), (dstt, ref.t().contiguous(), Cc, R)):
        if out is None:
            continue
        got = out[:rr, :cc]
        nan = torch.isnan(want)
        assert torch.equal(torch.isnan(got), nan), (R, Cc)
        assert torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan]), (R, Cc)
        assert _untouched(out, rr, cc), (R, Cc)


@pytest.mark.parametrize("rows,ld", [(1, 8), (7, 16), (1000, 24), (4099, 16)])
def test_pack_col0_is_exact(rows, ld):
    L, h, st, _ = _lib()
    v = _randn(_gen(9), rows)
    out = _out(rows, ld)
    _ok(L.gm_pack_col0(h, _p(v), rows, _p(out), ld, st))
    torch.cuda.synchronize()
    ref = torch.zeros(rows, ld, device="cuda", dtype=torch.bfloat16)
    ref[:, 0] = v.to(torch.bfloat16)
    assert torch.equal(out[:rows].view(torch.int16), ref.view(torch.int16)) and _untouched(out, rows, ld)


NOISE_CASES = [(z, rows, pad_of(i)) for i, z in enumerate((1, 7, 8, 30, 100, 127)) for rows in (1, 300)]


@pytest.mark.parametrize("z,rows,pad", NOISE_CASES, ids=["z%d_rows%d_pad%d" % c for c in NOISE_CASES])
def test_noise_rows_of_a_caller_tensor_are_exact(z, rows, pad):
    L, h, st, _ = _lib()
    ld = (z + 8) // 8 * 8 + pad
    noise = _randn(_gen(10), rows, z)
    noise.view(-1)[0] = 1 + 2.0 ** -8
    out = _out(rows, ld)
    _ok(L.gm_noise_rows(h, _p(noise), _p(out), rows, z, ld, 0, 0, st))
    torch.cuda.synchronize()
    assert torch.equal(out[:rows].view(torch.int16), CR.noise_rows(noise, ld).view(torch.int16)) and _untouched(out, rows, ld)


def test_noise_rows_philox_is_repeatable_keyed_and_standard_normal():
    L, h, st, _ = _lib()
    rows, z, ld = 8192, 128, 144

    def draw(seed, stream_id):
        out = _out(rows, ld)
        _ok(L.gm_noise_rows(h, None, _p(out), rows, z, ld, seed, stream_id, st))
        torch.cuda.synchronize()
        assert _untouched(out, rows, ld)
        return out[:rows]

    a, b, c, d = draw(7, 3), draw(7, 3), draw(7, 4), draw(8, 3)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16))
    assert not torch.equal(a[:, :z], c[:, :z]) and not torch.equal(a[:, :z], d[:, :z])
    assert bool((a[:, z] == 1).all()) and bool((a[:, z + 1:] == 0).all())
    v = a[:, :z].double()
    n = v.numel()                                           # 2^20 draws: 5 standard errors of the mean and of the variance
    assert abs(float(v.mean())) < 5 / math.sqrt(n) and abs(float(v.var()) - 1) < 5 * math.sqrt(2 / n), (float(v.mean()), float(v.var()))
    _REPORT.add("noise_philox", {"mean": float(v.mean()), "var": float(v.var()), "draws": n})


IMG_CASES = [(fmt, x, gather, pad_of(i + j)) for i, fmt in enumerate(("f32", "u8", "bits")) for j, x in enumerate((8, 784, 12288, 100))
             for gather in (False, True)]


@pytest.mark.parametrize("fmt,x,gather,pad", IMG_CASES, ids=["%s_x%d_%s_pad%d" % (f, x, "gather" if g else "rows", p) for f, x, g, p in IMG_CASES])
def test_stage_images_is_exact(fmt, x, gather, pad):
    L, h, st, _ = _lib()
    n_src, rows = 7, 5
    g = _gen(11)
    ld = (x + 8) // 8 * 8 + pad
    if fmt == "f32":
        images = torch.rand(n_src, x, device="cuda", generator=g)
    else:       # u8 values other than 0 and 1: both packed formats binarise
        images = torch.tensor([0, 1, 2, 3, 128, 255, 0, 0], device="cuda", dtype=torch.uint8)[torch.randint(0, 8, (n_src, x), device="cuda", generator=g)]
    src = images
    if fmt == "bits":
        src = torch.from_numpy(np.packbits((images != 0).cpu().numpy().reshape(-1))).cuda()
    idx = torch.tensor([6, 0, 3, 3, 1], device="cuda", dtype=torch.int32) if gather else None
    out = _out(rows, ld)
    _ok(L.gm_stage_images(h, _p(src), {"f32": 0, "u8": 1, "bits": 2}[fmt], _p(idx), _p(out), rows, x, ld, st))
    torch.cuda.synchronize()
    ref = CR.stage_images(src, fmt, idx if gather else torch.arange(rows), x, ld)
    assert torch.equal(out[:rows].view(torch.int16), ref.view(torch.int16)) and _untouched(out, rows, ld)


# ------------------------------------------------------------------ gm_loss_rows
def _loss_acts(variant):
    return ("sigmoid",) if variant in ("ns", "mm") else ("sigmoid", "relu", "none")     # log(d), log(1 - d) need d in (0, 1)


LOSS_CASES = [(v, a, gs, B) for v in CR.ROW_VARIANTS for a in _loss_acts(v) for gs in (0, 1) for B in (1, 7, 256, 5000)]


def _run_loss(variant, out_act, g_step, B, seed=12):
    L, h, st, _ = _lib()
    rows = B if g_step else 2 * B
    s = 2 * _randn(_gen(seed), rows)
    sp = torch.tensor([0.0, 30.0, -30.0], device="cuda") if out_act == "sigmoid" and not variant.startswith("f_") else torch.tensor([0.0], device="cuda")
    if variant.startswith("f_") or out_act != "sigmoid":
        s = s.clamp(-3, 3)
    s[:min(rows, sp.numel())] = sp[:rows]
    ds, d, loss = _f32(rows), _f32(rows), _f32(3)
    _ok(L.gm_loss_rows(h, VARIANT_ID[variant], OUT_ACT_ID[out_act], _p(s), B, g_step, 1.0 / B, _p(ds), _p(d), _p(loss), st))
    torch.cuda.synchronize()
    return s, ds, d, loss, rows


@pytest.mark.parametrize("variant,out_act,g_step,B", LOSS_CASES, ids=["%s_%s_%s_B%d" % (v, a, "G" if gs else "D", B) for v, a, gs, B in LOSS_CASES])
def test_loss_rows_match_the_float64_oracle(variant, out_act, g_step, B):
    name = "%s_%s_%d_%d" % (variant, out_act, g_step, B)
    s, ds, d, loss, rows = _run_loss(variant, out_act, g_step, B)
    assert _f32_untouched(ds, rows) and _f32_untouched(d, rows), name
    s64, d_got, ds_got = s.double().cpu().numpy(), d[:rows].double().cpu().numpy(), ds[:rows].double().cpu().numpy()
    assert np.isfinite(d_got).all() and np.isfinite(ds_got).all() and bool(torch.isfinite(loss[:2]).all()), name
    d_ref = CR.d_out(s64, out_act)
    tol_d = 8 * U * np.abs(d_ref) if out_act == "sigmoid" else np.zeros_like(d_ref)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    _record("loss_d_" + out_act, name, _ratio(T(np.abs(d_got - d_ref)), T(tol_d)))
    L_ref, ds_ref = CR.loss_rows(variant, out_act, s64, d_got, B, g_step)
    ag = np.abs(CR.R.d_out_grad(dict(d=d_got, s=s64), np.ones_like(d_got), out_act))
    _record("loss_ds_" + variant, name, _ratio(T(np.abs(ds_got - ds_ref)), T(16 * U * (np.abs(ds_ref) + ag * (1 + np.abs(d_got)) / B))))
    mag = 1 + 2 * np.abs(d_got) + (np.exp(np.abs(d_got)) if variant.startswith("f_") else 0)
    scale = 1 if g_step else 2
    _record("loss_" + variant, name, abs(float(loss[0]) - L_ref) / (8 * U * (abs(L_ref) + scale * float(mag.mean()))))
    total = float(ds_got.sum())
    assert abs(float(loss[1]) - total) <= 2 * U * abs(total) + 1e-12 * float(np.abs(ds_got).sum()) + 1e-30, name


# ------------------------------------------------------------------ determinism, a chain, refusals
def test_repeated_calls_give_identical_bits():
    """BatchNorm's and the losses' two-stage reductions run in a fixed order; the data movements have no order at all"""
    bits = lambda t: t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)
    a, b = _run_im2col(SWEEPS_IM2COL[0], 8), _run_im2col(SWEEPS_IM2COL[0], 8)
    assert torch.equal(bits(a[1]), bits(b[1]))
    for mode in range(4):
        a, b = _run_col2im(SWEEPS_COL2IM[0], mode, 8), _run_col2im(SWEEPS_COL2IM[0], mode, 8)
        assert torch.equal(bits(a[2]), bits(b[2])), mode
    case = (SWEEPS_BN[0], 2, "normal", 8)
    a, b = _run_bn_backward(case), _run_bn_backward(case)
    for k in ("y", "stats", "dx", "dgb"):
        assert torch.equal(bits(a[k]), bits(b[k])), k
    a, b = _run_bn_forward((4133, 64), 1, "offset", 0), _run_bn_forward((4133, 64), 1, "offset", 0)
    for k in ("y", "stats", "run"):
        assert torch.equal(bits(a[k]), bits(b[k])), k
    for v, act, gs in (("ns", "sigmoid", 0), ("ls", "none", 1), ("f_pearson", "relu", 0)):
        a, b = _run_loss(v, act, gs, 5000), _run_loss(v, act, gs, 5000)
        for i in (1, 2, 3):
            assert torch.equal(bits(a[i]), bits(b[i])), (v, i)


def test_conv_chain_without_host_sync():
    """im2col -> GEMM -> BatchNorm forward -> BatchNorm backward -> GEMM -> col2im enqueued back to back on one stream, every
    intermediate prefilled with NaN (a read ahead of its producer shows): each stage against float64 of the stored output
    of the stage before, and the launches the calls are documented to make (1 + 1 + 3 + 3 + 1 + 1)"""
    import gm_b200
    L, h, st, _ = _lib()
    B, Hh, Ci, Co, C2 = 4, 16, 16, 32, 8
    g = _gen(13)
    nan = lambda r, c: torch.full((r, c), float("nan"), device="cuda", dtype=torch.bfloat16)
    x = _randn(g, B * Hh * Hh, Ci).to(torch.bfloat16)
    W1 = (_randn(g, Co, 16 * Ci) / 16).to(torch.bfloat16)
    W2 = (_randn(g, 16 * C2, Co) / 6).to(torch.bfloat16)
    gamma, beta = _bn_params(g, Co)
    rows = B * (Hh // 2) ** 2
    col, y1, y2, dx, col2, out = nan(rows, 16 * Ci), nan(rows, Co), nan(rows, Co), nan(rows, Co), nan(rows, 16 * C2), nan(4 * rows, C2)
    stats, dgb = torch.full((2, Co), float("nan"), device="cuda"), torch.full((2, Co), float("nan"), device="cuda")
    torch.cuda.synchronize()
    n0 = gm_b200.launch_count()
    _ok(L.gm_im2col_k4s2(h, _p(x), B, Hh, Hh, Ci, Ci, _p(col), 16 * Ci, st))
    gm_b200.gemm_bf16(col, W1, y1, "nt")
    _ok(L.gm_bn_forward(h, _p(y1), rows, Co, Co, _p(gamma), _p(beta), EPS, 2, SLOPE, _p(y2), Co, _p(stats), None, MOM, st))
    _ok(L.gm_bn_backward(h, _p(y2), _p(y1), rows, Co, Co, _p(stats), _p(gamma), _p(beta), 2, SLOPE, _p(dx), Co, _p(dgb), st))
    gm_b200.gemm_bf16(dx, W2, col2, "nt")
    _ok(L.gm_col2im_k4s2(h, _p(col2), 16 * C2, B, Hh // 2, Hh // 2, C2, _p(out), C2, 0, None, 0, SLOPE, st))
    torch.cuda.synchronize()
    assert gm_b200.launch_count() - n0 == 10
    assert torch.equal(col.view(torch.int16), CR.im2col(x.view(B, Hh, Hh, Ci)).view(torch.int16))

    def gemm(a, w, got, K):      # the bound of tests/test_gemm_conformance_gpu.py
        pre = a.double() @ w.double().t()
        e = 4 * math.ceil(K / 16) * 2.0 ** -23 * (a.double().abs() @ w.double().abs().t())
        return _ratio((got.double() - pre).abs(), 2.0 ** -8 * (pre.abs() + e) + e)

    worst = [gemm(col, W1, y1, 16 * Ci)]
    T = dict(x=y1, gamma=gamma, beta=beta, y=y2)
    _, f = CR.bn_forward(y1, stats[0], stats[1], gamma, beta, 2, SLOPE)
    sc = (gamma.double() * stats[1].double()).abs()
    m = 4 * U * (y1.double().abs() * sc + stats[0].double().abs() * sc + beta.double().abs())
    worst.append(_ratio((y2.double() - f).abs(), _bf16_tol(f, m)))
    mean, var, _ = CR.bn_stats(y1)
    assert float(((stats[0].double() - mean).abs() / (2.0 ** -18 * y1.double().abs().mean(0) + U * mean.abs())).max()) <= 1
    r = CR.bn_backward(y2, y1, stats[0], stats[1], gamma, beta, 2, SLOPE, dgb=dgb)
    kink = r["pre"].abs() <= 8 * U * ((gamma.double() * r["xhat"]).abs() + beta.double().abs())
    tol = _bf16_tol(r["dx"], 8 * U * r["mag"])
    worst.append(_ratio((dx.double() - r["dx"]).abs()[~kink], tol[~kink]))
    worst.append(gemm(dx, W2, col2, Co))
    f, sabs = CR.col2im(col2.double(), B, Hh // 2, Hh // 2, C2)
    f, e = f.reshape(-1, C2), 3 * U * sabs.reshape(-1, C2)
    worst.append(_ratio((out.double() - f).abs(), _bf16_tol(f, e)))
    _record("chain", "im2col_gemm_bn_bnbwd_gemm_col2im", max(worst))


def test_invalid_conv_arguments_are_refused_before_any_launch():
    """every refusal include/gm_b200.h documents for the conv building blocks: the GM_ERR_* code, a message, nothing launched"""
    L, h, st, _ = _lib()
    bf = lambda r, c: torch.zeros(r, c, device="cuda", dtype=torch.bfloat16)
    x, col, y, aux = bf(64 + 1, 16), bf(16 + 1, 256 + 8), bf(64 + 1, 16), bf(64 + 1, 16)
    f32 = torch.zeros(4096, device="cuda")
    idx = torch.zeros(8, device="cuda", dtype=torch.int32)
    u8 = torch.zeros(4096, device="cuda", dtype=torch.uint8)
    P, off = (lambda t: t.data_ptr()), 2         # one bf16 past a 16-byte boundary
    A, UNS = GM_ERR_ARG, GM_ERR_UNSUPPORTED

    def im2col(x_=P(x), B=1, Hh=8, W=8, Cc=16, ldx=16, col_=P(col), ldc=256):
        return L.gm_im2col_k4s2(h, x_, B, Hh, W, Cc, ldx, col_, ldc, st)

    def im2colm(x_=P(x), B=1, Hh=8, W=8, Cc=16, ldx=16, m_=P(aux), ldm=16, col_=P(col), ldc=256):
        return L.gm_im2col_k4s2_lrelu_mask(h, x_, B, Hh, W, Cc, ldx, m_, ldm, SLOPE, col_, ldc, st)

    def col2im(col_=P(col), ldc=256, B=1, Hi=4, Wi=4, Cc=16, y_=P(y), ldy=16, mode=0, aux_=None, lda=0):
        return L.gm_col2im_k4s2(h, col_, ldc, B, Hi, Wi, Cc, y_, ldy, mode, aux_, lda, SLOPE, st)

    def bnf(x_=P(x), rows=64, Cc=16, ld=16, act=0, y_=P(y), ldy=16):
        return L.gm_bn_forward(h, x_, rows, Cc, ld, P(f32), P(f32), EPS, act, SLOPE, y_, ldy, P(f32), None, MOM, st)

    def bne(x_=P(x), rows=64, Cc=16, ld=16, act=0, y_=P(y), ldy=16):
        return L.gm_bn_forward_eval(h, x_, rows, Cc, ld, P(f32), P(f32), P(f32), EPS, act, SLOPE, y_, ldy, st)

    def bnb(dy_=P(aux), x_=P(x), rows=64, Cc=16, ld=16, act=0, dx_=P(y), lddx=16):
        return L.gm_bn_backward(h, dy_, x_, rows, Cc, ld, P(f32), P(f32), P(f32), act, SLOPE, dx_, lddx, P(f32), st)

    def lrelu(x_=P(x), ldx=16, m_=P(aux), ldm=16, rows=64, Cc=16, out_=P(y), ldo=16):
        return L.gm_lrelu_mask_rows(h, x_, ldx, m_, ldm, rows, Cc, SLOPE, out_, ldo, st)

    def cast(R=4, Cc=16, dst=P(x), ld=16, dst_t=P(y), ld_t=16):
        return L.gm_cast_bf16(h, P(f32), R, Cc, dst, ld, dst_t, ld_t, st)

    def noise(out_=P(x), rows=4, z=8, ld=16, src=None):
        return L.gm_noise_rows(h, src, out_, rows, z, ld, 1, 1, st)

    def stage(fmt=0, out_=P(x), rows=4, xx=8, ld=16, img=P(f32), gi=None):
        return L.gm_stage_images(h, img, fmt, gi, out_, rows, xx, ld, st)

    def loss(variant=0, out_act=0, batch=8):
        return L.gm_loss_rows(h, variant, out_act, P(f32), batch, 0, 0.125, P(f32) + 1024, None, P(f32) + 2048, st)

    bad = [
        # gm_im2col_k4s2 / gm_im2col_k4s2_lrelu_mask
        ("im2col odd H", A, lambda: im2col(Hh=7)), ("im2col odd W", A, lambda: im2col(W=6 + 1)),
        ("im2col ldx < C", A, lambda: im2col(ldx=8)), ("im2col ldc < 16 C", A, lambda: im2col(ldc=248)),
        ("im2col ldx % 8", A, lambda: im2col(ldx=20)), ("im2col x misaligned", A, lambda: im2col(x_=P(x) + off)),
        ("im2col col misaligned", A, lambda: im2col(col_=P(col) + off)),
        ("im2col 2^31 items", UNS, lambda: im2col(B=32768, Hh=512, W=512, Cc=8, ldx=8, ldc=128)),
        ("mask im2col C % 8", A, lambda: im2colm(Cc=12, ldx=16, ldc=256)), ("mask im2col ldm < C", A, lambda: im2colm(ldm=8)),
        ("mask im2col odd H", A, lambda: im2colm(Hh=7)),
        ("mask im2col x misaligned", A, lambda: im2colm(x_=P(x) + off)), ("mask im2col m misaligned", A, lambda: im2colm(m_=P(aux) + off)),
        ("mask im2col col misaligned", A, lambda: im2colm(col_=P(col) + off)),
        ("mask im2col 2^31 items", UNS, lambda: im2colm(B=32768, Hh=512, W=512, Cc=8, ldx=8, ldm=8, ldc=128)),
        # gm_col2im_k4s2
        ("col2im mode 4", A, lambda: col2im(mode=4)), ("col2im mode -1", A, lambda: col2im(mode=-1)),
        ("col2im mode 2 without aux", A, lambda: col2im(mode=2)), ("col2im mode 3 without aux", A, lambda: col2im(mode=3)),
        ("col2im ld_aux < C", A, lambda: col2im(mode=2, aux_=P(aux), lda=8)), ("col2im ld_aux % 8", A, lambda: col2im(mode=3, aux_=P(aux), lda=20)),
        ("col2im ldy < C", A, lambda: col2im(ldy=8)), ("col2im ldc < 16 C", A, lambda: col2im(ldc=248)),
        ("col2im C = 12", UNS, lambda: col2im(Cc=12)),
        ("col2im col misaligned", A, lambda: col2im(col_=P(col) + off)), ("col2im y misaligned", A, lambda: col2im(y_=P(y) + off)),
        ("col2im aux misaligned", A, lambda: col2im(mode=2, aux_=P(aux) + off, lda=16)),
        ("col2im 2^31 items", UNS, lambda: col2im(B=32768, Hi=256, Wi=256, Cc=8, ldc=128, ldy=8)),
        # gm_bn_forward / gm_bn_forward_eval / gm_bn_backward
        ("bn_forward ld < C", A, lambda: bnf(ld=8)), ("bn_forward ldy < C", A, lambda: bnf(ldy=8)), ("bn_forward act 3", A, lambda: bnf(act=3)),
        ("bn_forward act -1", A, lambda: bnf(act=-1)), ("bn_forward C % 8", A, lambda: bnf(Cc=12)),
        ("bn_forward x misaligned", A, lambda: bnf(x_=P(x) + off)), ("bn_forward y misaligned", A, lambda: bnf(y_=P(y) + off)),
        ("bn_forward C > 2048", UNS, lambda: bnf(Cc=2056, ld=2056, ldy=2056, rows=1)),
        ("bn_eval ld < C", A, lambda: bne(ld=8)), ("bn_eval ldy < C", A, lambda: bne(ldy=8)), ("bn_eval act 3", A, lambda: bne(act=3)),
        ("bn_eval x misaligned", A, lambda: bne(x_=P(x) + off)), ("bn_eval y misaligned", A, lambda: bne(y_=P(y) + off)),
        ("bn_eval C > 2048", UNS, lambda: bne(Cc=2056, ld=2056, ldy=2056, rows=1)),
        ("bn_backward ld < C", A, lambda: bnb(ld=8)), ("bn_backward lddx < C", A, lambda: bnb(lddx=8)), ("bn_backward act 3", A, lambda: bnb(act=3)),
        ("bn_backward dy misaligned", A, lambda: bnb(dy_=P(aux) + off)), ("bn_backward x misaligned", A, lambda: bnb(x_=P(x) + off)),
        ("bn_backward dx misaligned", A, lambda: bnb(dx_=P(y) + off)),
        ("bn_backward C > 2048", UNS, lambda: bnb(Cc=2056, ld=2056, lddx=2056, rows=1)),
        # gm_lrelu_mask_rows
        ("lrelu ldx < C", A, lambda: lrelu(ldx=8)), ("lrelu C % 8", A, lambda: lrelu(Cc=12)), ("lrelu x misaligned", A, lambda: lrelu(x_=P(x) + off)),
        ("lrelu m misaligned", A, lambda: lrelu(m_=P(aux) + off)), ("lrelu out misaligned", A, lambda: lrelu(out_=P(y) + off)),
        ("lrelu 2^31 items", UNS, lambda: lrelu(rows=1 << 31, Cc=8, ldx=8, ldm=8, ldo=8)),
        # gm_cast_bf16 / gm_pack_col0
        ("cast ld < C", A, lambda: cast(ld=8)), ("cast ld_t < R", A, lambda: cast(ld_t=3)), ("cast no output", A, lambda: cast(dst=None, dst_t=None)),
        ("cast 2^32 values", UNS, lambda: cast(R=65536, Cc=65536, ld=65536, ld_t=65536)),
        ("pack_col0 2^31 values", UNS, lambda: L.gm_pack_col0(h, P(f32), 1 << 28, P(x), 8, st)),
        # gm_noise_rows
        ("noise ld <= z", A, lambda: noise(ld=8)), ("noise ld % 8", A, lambda: noise(ld=12)), ("noise out misaligned", A, lambda: noise(out_=P(x) + off)),
        ("noise 2^31 threads", UNS, lambda: noise(rows=(1 << 31) - 1)),
        # gm_stage_images
        ("stage img_fmt 3", A, lambda: stage(fmt=3)), ("stage img_fmt -1", A, lambda: stage(fmt=-1)), ("stage ld <= x", A, lambda: stage(ld=8)),
        ("stage out misaligned", A, lambda: stage(out_=P(x) + off)), ("stage fp32 images misaligned", A, lambda: stage(img=P(f32) + 2)),
        ("stage gather_idx misaligned", A, lambda: stage(gi=P(idx) + 2)),
        # gm_loss_rows
        ("loss variant 16", A, lambda: loss(variant=16)), ("loss variant -1", A, lambda: loss(variant=-1)), ("loss out_act 3", A, lambda: loss(out_act=3)),
        ("loss out_act -1", A, lambda: loss(out_act=-1)), ("loss batch 0", A, lambda: loss(batch=0)),
        ("loss RaNS", UNS, lambda: loss(variant=6)), ("loss WGAN-GP", UNS, lambda: loss(variant=3)), ("loss BEGAN", UNS, lambda: loss(variant=15)),
    ]
    torch.cuda.synchronize()
    n0 = L.gm_launch_count(h, 0)
    for what, code, call in bad:
        rc = call()
        assert rc == code and L.gm_last_error(h).decode(), (what, rc)
    assert L.gm_launch_count(h, 0) == n0
    # the valid neighbours of those calls run: 1 launch each, 3 per training-mode BatchNorm call, 2 in inference mode
    good = [im2col, im2colm, col2im, lambda: col2im(mode=2, aux_=P(aux), lda=16), bnf, lambda: bnf(act=2), bne, bnb, lrelu, cast, noise,
            lambda: noise(src=P(f32)), stage, lambda: stage(fmt=1, img=P(u8) + 1), lambda: stage(fmt=2, img=P(u8) + 1, gi=P(idx)), loss,
            lambda: loss(variant=13, out_act=2)]
    for call in good:
        _ok(call())
    torch.cuda.synchronize()
    assert L.gm_launch_count(h, 0) == n0 + len(good) + 3 * 2 + 1
