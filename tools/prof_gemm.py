"""Launch the two characteristic K-major GEMMs of the step in isolation (for ncu):
  g1: [65536,32(64)] x [400,64]^T  -> relu, bias, ones column   (epilogue-bound)
  d1: [131072,784]   x [400,784]^T -> relu, bias, fused row-dot (mainloop + epilogue)
  dx: [65536,400]    x [784,400]^T -> * aux(1-aux)
and the two split-K weight gradients of the step (MN-major; the time is the GEMM kernel's alone, without the partials'
reduction that gm_gemm_bf16 runs after it):
  dw1d: [131072,785]^T x [131072,400] -> fp32, transposed partials (D's first layer + bias column)
  dw2g: [65536,784]^T  x [65536,401]  -> fp32 partials (G's output layer + bias row)
Prints CUDA-event times."""
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "generative-models_b200"))
import gm_b200  # noqa: E402

which = sys.argv[1:] or ["g1", "d1", "dx"]
dev = "cuda"
torch.manual_seed(0)


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3


B = 65536
if "g1" in which:
    A, W = bf(B, 64), bf(400, 64, scale=0.1)
    out = torch.zeros(B, 416, device=dev, dtype=torch.bfloat16)
    bias = torch.randn(400, device=dev)
    t = timeit(lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=32, bias=bias, act=1, pad_one=True, out_cols=416))
    print("g1 %.1f us" % t)
if "d1" in which:
    A, W = bf(2 * B, 800), bf(400, 784, scale=0.05)
    out = torch.zeros(2 * B, 416, device=dev, dtype=torch.bfloat16)
    bias, w2 = torch.randn(400, device=dev), torch.randn(400, device=dev)
    slots = torch.zeros(4, 2 * B, device=dev)
    t = timeit(lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=784, bias=bias, act=1, dot_w=w2, dot_out=slots))
    print("d1 %.1f us  %.0f TFLOP/s" % (t, 2 * 2 * B * 400 * 784 / t / 1e6))
if "dx" in which:
    A, W = bf(B, 416), bf(784, 400, scale=0.05)
    aux = torch.rand(B, 800, device=dev).to(torch.bfloat16)
    out = torch.zeros(B, 800, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=400, aux=aux, aux_mode=1))
    print("dx %.1f us  %.0f TFLOP/s" % (t, 2 * B * 400 * 784 / t / 1e6))
if "g2" in which:
    A, W = bf(B, 416), bf(784, 400, scale=0.05)
    out = torch.zeros(B, 832, device=dev, dtype=torch.bfloat16)
    bias = torch.randn(784, device=dev)
    t = timeit(lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=400, bias=bias, act=2, pad_one=True, out_cols=832))
    print("g2 %.1f us  %.0f TFLOP/s" % (t, 2 * B * 400 * 784 / t / 1e6))
if "dhg" in which:
    A, W = bf(B, 800), bf(400, 784, scale=0.05)
    aux = torch.randn(B, 416, device=dev).to(torch.bfloat16)
    out = torch.zeros(B, 416, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=784, aux=aux, aux_mode=2))
    print("dhg %.1f us  %.0f TFLOP/s" % (t, 2 * B * 400 * 784 / t / 1e6))


def gemm_only(fn, n=5):
    """mean time of the GEMM kernel alone (level-1 profile: events around each GEMM launch), us"""
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    gm_b200.prof_collect()
    gm_b200.prof_enable(1)
    for _ in range(n):
        fn()
    gm_b200.prof_enable(0)
    ms = sum(r[1] for r in gm_b200.prof_collect())
    return ms / n * 1e3


if "dw1d" in which:
    A, G = bf(2 * B, 800), bf(2 * B, 416, scale=0.1)
    out = torch.zeros(400, 788, device=dev)
    t = gemm_only(lambda: gm_b200.gemm_bf16(A, G, out, "tn", M=785, N=400, transpose=True))
    print("dw1d %.1f us  %.0f TFLOP/s" % (t, 2 * 2 * B * 785 * 400 / t / 1e6))
if "dw2g" in which:
    A, G = bf(B, 800), bf(B, 416, scale=0.1)
    out = torch.zeros(784, 448, device=dev)
    t = gemm_only(lambda: gm_b200.gemm_bf16(A, G, out, "tn", M=784, N=401))
    print("dw2g %.1f us  %.0f TFLOP/s" % (t, 2 * B * 784 * 401 / t / 1e6))
