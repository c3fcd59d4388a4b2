"""The float64 references of tests/conv_reference.py against torch in float64 on the CPU, and the shape of the case tables
of tests/test_conv_conformance_gpu.py (leading dimensions, multi-sweep sizes for 132 SMs, memory per case)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import conv_reference as CR
import test_conv_conformance_gpu as T
from oracle import ref_math as R

SMALL = [(1, 2, 2, 1), (3, 4, 4, 3), (2, 6, 10, 8), (2, 12, 20, 24)]


@pytest.mark.parametrize("shape", SMALL, ids=[T._name(s) for s in SMALL])
def test_im2col_then_matmul_is_conv2d(shape):
    B, H, W, Cc = shape
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, H, W, Cc, generator=g, dtype=torch.float64)
    w = torch.randn(5, Cc, 4, 4, generator=g, dtype=torch.float64)                          # torch layout [Cout, Cin, kh, kw]
    y = CR.im2col(x) @ w.permute(0, 2, 3, 1).reshape(5, 16 * Cc).t()                        # columns (kh, kw, c)
    ref = F.conv2d(x.permute(0, 3, 1, 2), w, stride=2, padding=1).permute(0, 2, 3, 1).reshape(-1, 5)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("shape", SMALL + [(2, 3, 5, 7)], ids=[T._name(s) for s in SMALL + [(2, 3, 5, 7)]])
def test_matmul_then_col2im_is_conv_transpose2d(shape):
    B, Hi, Wi, Cc = shape
    g = torch.Generator().manual_seed(2)
    x = torch.randn(B * Hi * Wi, 6, generator=g, dtype=torch.float64)
    w = torch.randn(6, Cc, 4, 4, generator=g, dtype=torch.float64)                          # torch layout [Cin, Cout, kh, kw]
    col = x @ w.permute(2, 3, 1, 0).reshape(16 * Cc, 6).t()
    y, yabs = CR.col2im(col, B, Hi, Wi, Cc)
    ref = F.conv_transpose2d(x.view(B, Hi, Wi, 6).permute(0, 3, 1, 2), w, stride=2, padding=1).permute(0, 2, 3, 1)
    assert torch.allclose(y, ref, rtol=1e-12, atol=1e-12)
    assert torch.allclose(yabs, CR.col2im(col.abs(), B, Hi, Wi, Cc)[0]) and bool((yabs >= y.abs() - 1e-12).all())
    cls = CR.border_class(B, 2 * Hi, 2 * Wi, "cpu")
    assert int((cls == 2).sum()) == 4 * B and int((cls == 1).sum()) == B * (2 * (2 * Hi - 2) + 2 * (2 * Wi - 2))
    taps = CR.col2im(torch.ones_like(col), B, Hi, Wi, Cc)[0][..., 0]                         # taps that reach a pixel of a 2x+ grid
    if Hi > 1 and Wi > 1:
        assert bool((taps[cls == 2] == 1).all()) and bool((taps[cls == 1] == 2).all()) and bool((taps[cls == 0] == 4).all())


@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("rows,Cc", [(2, 8), (37, 24), (300, 64)])
def test_batchnorm_reference_is_torch_batch_norm_and_its_autograd(rows, Cc, act):
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(rows, Cc, generator=g, dtype=torch.float64) * 1.5 + 0.3).requires_grad_()
    gamma = (1 + 0.1 * torch.randn(Cc, generator=g, dtype=torch.float64)).requires_grad_()
    beta = (0.1 * torch.randn(Cc, generator=g, dtype=torch.float64)).requires_grad_()
    dy = torch.randn(rows, Cc, generator=g, dtype=torch.float64)
    rm, rv = 0.2 * torch.randn(Cc, generator=g, dtype=torch.float64), 0.5 + torch.rand(Cc, generator=g, dtype=torch.float64)
    run0 = torch.stack([rm, rv]).clone()
    fn = {0: lambda t: t, 1: torch.relu, 2: lambda t: F.leaky_relu(t, 0.2)}[act]
    yt = fn(F.batch_norm(x, rm, rv, gamma, beta, True, 0.1, 1e-5))
    yt.backward(dy)
    mean, var, ex2 = CR.bn_stats(x.detach())
    assert torch.allclose(ex2 - mean ** 2, var, atol=1e-12)
    invstd = (var + 1e-5) ** -0.5
    _, y = CR.bn_forward(x.detach(), mean, invstd, gamma.detach(), beta.detach(), act, 0.2)
    assert torch.allclose(y, yt.detach(), rtol=1e-11, atol=1e-12)
    assert torch.allclose(CR.bn_running(run0, mean, var, rows, 0.1), torch.stack([rm, rv]), rtol=1e-12, atol=1e-12)
    r = CR.bn_backward(dy, x.detach(), mean, invstd, gamma.detach(), beta.detach(), act, 0.2)
    assert torch.allclose(r["dbeta"], beta.grad, rtol=1e-10, atol=1e-11) and torch.allclose(r["dgamma"], gamma.grad, rtol=1e-10, atol=1e-11)
    assert torch.allclose(r["dx"], x.grad, rtol=1e-9, atol=1e-11)
    assert bool((r["mag"] >= r["dx"].abs() - 1e-12).all())
    r2 = CR.bn_backward(dy, x.detach(), mean, invstd, gamma.detach(), beta.detach(), act, 0.2, dgb=torch.stack([r["dbeta"], r["dgamma"]]))
    assert torch.equal(r2["dx"], r["dx"])
    # inference mode: the same formula on the running statistics
    ye = fn(F.batch_norm(x.detach(), run0[0], run0[1], gamma.detach(), beta.detach(), False, 0.1, 1e-5))
    assert torch.allclose(CR.bn_forward(x.detach(), run0[0], (run0[1] + 1e-5) ** -0.5, gamma.detach(), beta.detach(), act, 0.2)[1], ye, rtol=1e-11, atol=1e-12)


def test_lrelu_mask_noise_and_image_references():
    x = torch.tensor([1.0, -2.0, 3.0, 0.5, -0.75, 1.5]).to(torch.bfloat16)
    m = torch.tensor([0.0, -0.0, 1e-40, -1e-40, float("inf"), float("-inf")]).to(torch.bfloat16)
    want = torch.tensor([0.2 * 1.0, 0.2 * -2.0, 0.2 * 3.0, 0.2 * 0.5, -0.75, 0.2 * 1.5])
    m.view(torch.int16)[2:4] = torch.tensor([1, -32767], dtype=torch.int16)                 # the smallest bf16 of either sign
    want[2] = 3.0
    assert torch.equal(CR.lrelu_mask(x, m, 0.2), want.to(torch.bfloat16).double())
    nz = CR.noise_rows(torch.tensor([[1 + 2.0 ** -8, 2.0, 3.0]]), 8)
    assert nz.tolist() == [[1.0, 2.0, 3.0, 1.0, 0.0, 0.0, 0.0, 0.0]]
    img = torch.tensor([[0, 1, 2, 0, 255, 0, 0, 3, 0, 7], [9, 0, 0, 0, 0, 1, 0, 0, 0, 0]], dtype=torch.uint8)
    want = torch.zeros(2, 16)
    want[:, :10] = (img[[1, 0]] != 0).float()
    want[:, 10] = 1
    idx = torch.tensor([1, 0])
    assert torch.equal(CR.stage_images(img, "u8", idx, 10, 16).float(), want)
    packed = torch.from_numpy(np.packbits((img != 0).numpy().reshape(-1)))
    assert torch.equal(CR.stage_images(packed, "bits", idx, 10, 16).float(), want)
    assert torch.equal(CR.stage_images(img.float() / 255, "f32", idx, 10, 16)[:, :10], (img[[1, 0]].float() / 255).to(torch.bfloat16))


@pytest.mark.parametrize("variant,out_act", [(v, a) for v in CR.ROW_VARIANTS for a in T._loss_acts(v)])
def test_loss_reference_is_the_derivative_of_the_oracle_loss(variant, out_act):
    """ds of conv_reference.loss_rows (oracle/ref_math.py's closed forms) against central differences of the same loss value
    (NS and MM with a sigmoid output only: log(d) and log(1 - d) need d in (0, 1))"""
    B = 7
    s = np.random.default_rng(4).standard_normal(2 * B).clip(-3, 3)
    for g_step in (0, 1):
        rows = B if g_step else 2 * B
        d = CR.d_out(s[:rows], out_act)
        L, ds = CR.loss_rows(variant, out_act, s[:rows], d, B, g_step)
        num = np.zeros(rows)
        for i in range(rows):                                   # central differences of the loss value in the logits
            e = np.zeros(rows)
            e[i] = 1e-6
            lp = CR.loss_rows(variant, out_act, s[:rows] + e, CR.d_out(s[:rows] + e, out_act), B, g_step)[0]
            lm = CR.loss_rows(variant, out_act, s[:rows] - e, CR.d_out(s[:rows] - e, out_act), B, g_step)[0]
            num[i] = (lp - lm) / 2e-6
        assert np.allclose(ds, num, rtol=1e-5, atol=1e-8), (variant, out_act, g_step)
    assert L == pytest.approx(float(R.g_loss(variant, d.reshape(-1, 1))[0]))


def test_case_tables_are_well_formed():
    for (b, h, w, c) in T.SHAPES + T.SWEEPS_IM2COL:
        assert h % 2 == 0 and w % 2 == 0
    assert {c for _, _, _, c in T.SHAPES} == {1, 3, 4, 7, 12, 8, 24, 40, 64, 136, 256, 512, 1024, 2048}
    assert {(h, w) for _, h, w, _ in T.SHAPES} == {(2, 2), (4, 4), (6, 10), (12, 20), (32, 32), (64, 64)}
    assert {b for b, _, _, _ in T.SHAPES} == {1, 3, 5}
    assert all(T.pad_of(i) % 8 == 0 for i in range(3)) and {T.pad_of(i) for i in range(3)} == {0, 8, 16}
    # multi-sweep cases: more than two sweeps on 132 SMs, and a ragged tail
    multi = [("im2col", s) for s in T.SWEEPS_IM2COL] + [("col2im_vec" if s[3] % 8 == 0 else "col2im_scalar", s) for s in T.SWEEPS_COL2IM]
    multi += [("lrelu_rows", s) for s in T.SWEEPS_LRELU]
    for kernel, s in multi:
        n, sweep = T.items_of(kernel, s), T.sweep_items(kernel)
        assert n > 2 * sweep and n % (sweep // T.UNROLL[kernel]) != 0, (kernel, s, n, sweep)
    for s in T.SWEEPS_BN:
        sweep = T.sweep_items("bn", s[1])
        assert s[0] > 2 * sweep and s[0] % (sweep // T.UNROLL["bn"]) != 0, (s, sweep)
    assert sum(len(v) >= 2 for v in (T.SWEEPS_IM2COL, T.SWEEPS_COL2IM, T.SWEEPS_BN, T.SWEEPS_LRELU)) == 4
    for s in T.SHAPES + T.SWEEPS_IM2COL:
        assert T.case_bytes("im2col", s) < T.MAX_CASE_BYTES, s
    for s in T.COL2IM_SHAPES:
        assert T.case_bytes("col2im", s) < T.MAX_CASE_BYTES, s
    for s in T.BN_SHAPES + T.SWEEPS_BN + T.LRELU_ROWS:
        assert s[1] % 8 == 0 and T.case_bytes("bn", s) < T.MAX_CASE_BYTES, s
    assert all(s[3] % 8 == 0 or s[3] < 8 for s in T.COL2IM_SHAPES) and all(s[3] % 8 == 0 for s in T.MASK_SHAPES)
    ids = [T._bn_id(c) for c in T.BN_FWD_CASES]
    assert len(set(ids)) == len(ids)
