"""wgmma GEMM kernel at shapes with more tiles (or split-K work items) than SMs, so that every
persistent CTA runs several tiles and the operand ring's phase carries from one tile into the
next; ragged last k-blocks, M not a multiple of the 16-row epilogue slice, and the 16-column
last epilogue step of the 208-wide tile with padding columns beyond N (GPU)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _mk(rows, cols, ld=None, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = ld or cols
    t = torch.zeros(rows, ld, device="cuda", dtype=torch.bfloat16)
    t[:, :cols] = (torch.randn(rows, cols, device="cuda", generator=g) * scale).to(torch.bfloat16)
    return t


@pytest.mark.parametrize("M,N,K", [(128 * 300, 208, 784), (128 * 300, 400, 400), (1000, 400, 784),
                                   (2 * 128 * 133 + 7, 64, 400)])
def test_nt_plain_multitile(M, N, K):
    import gm_b200
    A, B = _mk(M, K, seed=11, scale=0.5), _mk(N, K, seed=12, scale=0.05)
    out = torch.full((M, N), 7.0, device="cuda", dtype=torch.bfloat16)
    gm_b200.gemm_bf16(A, B, out, "nt")
    torch.cuda.synchronize()
    ref = A.float() @ B.float().t()
    assert _rel(out.float(), ref) < 4e-3


@pytest.mark.parametrize("M", [128 * 300, 1000 + 5])
def test_nt_epilogues_multitile(M):
    import gm_b200
    N, K, ldo = 400, 784, 416
    A, B = _mk(M, K, 800, seed=13, scale=0.5), _mk(N, K, seed=14, scale=0.05)
    bias = torch.randn(N, device="cuda") * 0.1
    w = torch.randn(N, device="cuda")
    ref_pre = A[:, :K].float() @ B.float().t() + bias
    # relu + ones column in the 16-column last step of the second n-tile + fused row-dot
    out = torch.full((M, ldo), 7.0, device="cuda", dtype=torch.bfloat16)
    slots = torch.zeros(4, M, device="cuda")
    gm_b200.gemm_bf16(A, B, out, "nt", K=K, bias=bias, act=1, pad_one=True, out_cols=ldo, dot_w=w, dot_out=slots)
    torch.cuda.synchronize()
    ref = torch.relu(ref_pre)
    assert _rel(out[:, :N].float(), ref) < 4e-3
    assert torch.all(out[:, N] == 1) and torch.all(out[:, N + 1:] == 0)
    assert _rel(slots.sum(0), ref @ w) < 2e-3
    # sigmoid, padding columns zero
    out2 = torch.full((M, ldo), 7.0, device="cuda", dtype=torch.bfloat16)
    gm_b200.gemm_bf16(A, B, out2, "nt", K=K, bias=bias, act=2, out_cols=ldo)
    torch.cuda.synchronize()
    assert _rel(out2[:, :N].float(), torch.sigmoid(ref_pre)) < 4e-3
    assert torch.all(out2[:, N:] == 0)
    # aux modes (cp.async aux tiles, next-tile L2 prefetch)
    aux = torch.rand(M, ldo, device="cuda").to(torch.bfloat16)
    out3 = torch.zeros(M, ldo, device="cuda", dtype=torch.bfloat16)
    gm_b200.gemm_bf16(A, B, out3, "nt", K=K, aux=aux, aux_mode=1)
    torch.cuda.synchronize()
    a = aux[:, :N].float()
    assert _rel(out3[:, :N].float(), (ref_pre - bias) * a * (1 - a)) < 4e-3
    auxm = torch.randn(M, ldo, device="cuda").to(torch.bfloat16)
    out4 = torch.zeros(M, ldo, device="cuda", dtype=torch.bfloat16)
    gm_b200.gemm_bf16(A, B, out4, "nt", K=K, aux=auxm, aux_mode=2)
    torch.cuda.synchronize()
    assert _rel(out4[:, :N].float(), (ref_pre - bias) * (auxm[:, :N].float() > 0)) < 4e-3


@pytest.mark.parametrize("K,M,N,tr", [(256, 4096, 2048, False), (256, 4096, 1000, True)])
def test_tn_multitile(K, M, N, tr):
    import gm_b200
    lda, ldb = ((M + 15) // 16) * 16, ((N + 15) // 16) * 16
    A, B = _mk(K, M, lda, seed=15, scale=0.3), _mk(K, N, ldb, seed=16, scale=0.3)
    ldc = ((max(M, N) + 63) // 64) * 64
    out = torch.full((N if tr else M, ldc), 7.0, device="cuda", dtype=torch.float32)
    gm_b200.gemm_bf16(A, B, out, "tn", M=M, N=N, transpose=tr)
    torch.cuda.synchronize()
    ref = A[:, :M].float().t() @ B[:, :N].float()
    got = out[:N, :M].t() if tr else out[:M, :N]
    assert _rel(got, ref) < 1e-4
