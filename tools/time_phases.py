"""Per-tile phase timing of the GEMM kernel (CTA 0): first consumer warp's mainloop and epilogue.

The epilogue record splits the tile's epilogue into the fragment stores to the warp's scratch
tile (summed over its 64-column steps), the rest of the epilogue, and of that the row reads
from the scratch tile.  The clock reads are compiled out of the shipped library (they cost
registers next to the accumulators): build an instrumented copy and point GM_B200_LIB at it, e.g.
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fPIC -shared -I include \
       -DGM_PHASE_TIMING -o build_variants/lib_timing.so generative-models_b200/gm_b200/csrc/engine.cu
  GM_B200_LIB=$PWD/build_variants/lib_timing.so python tools/time_phases.py"""
import ctypes as C
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "generative-models_b200"))
import gm_b200  # noqa: E402
from gm_b200 import _lib  # noqa: E402

dev = "cuda"
torch.manual_seed(0)
B = 65536
dbg = torch.zeros(128, dtype=torch.int64, device=dev)
h = _lib.ctx()


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=dev) * scale).to(torch.bfloat16)


def run(name, fn):
    fn()
    torch.cuda.synchronize()
    dbg.zero_()
    _lib.lib().gm_debug_phase_buffer(h, C.c_void_p(dbg.data_ptr()))
    fn()
    torch.cuda.synchronize()
    _lib.lib().gm_debug_phase_buffer(h, None)
    d = dbg.cpu().view(2, 16, 4)
    print("==", name)
    print(" MMA  : tile | (unused) | mainloop | (unused) | start")
    t0 = int(d[0, 0, 3])
    for i in range(10):
        print("       %2d   %8d %8d %8d   @%d" % (i, d[0, i, 0], d[0, i, 1], d[0, i, 2], int(d[0, i, 3]) - t0))
    print(" EPI  : tile | fragment stores | rest of epilogue | of which scratch reads | start")
    for i in range(0, 10):
        print("       %2d   %8d %8d %8d   @%d" % (i, d[1, i, 0], d[1, i, 1], d[1, i, 2], int(d[1, i, 3]) - t0))


A, W = bf(B, 64), bf(400, 64, scale=0.1)
out = torch.zeros(B, 416, device=dev, dtype=torch.bfloat16)
bias = torch.randn(400, device=dev)
run("g1 (K=32)", lambda: gm_b200.gemm_bf16(A, W, out, "nt", K=32, bias=bias, act=1, pad_one=True, out_cols=416))
A2, W2 = bf(2 * B, 800), bf(400, 784, scale=0.05)
out2 = torch.zeros(2 * B, 416, device=dev, dtype=torch.bfloat16)
w2 = torch.randn(400, device=dev)
slots = torch.zeros(4, 2 * B, device=dev)
run("d1 (K=784)", lambda: gm_b200.gemm_bf16(A2, W2, out2, "nt", K=784, bias=bias, act=1, dot_w=w2, dot_out=slots))
A3, W3 = bf(B, 416), bf(784, 400, scale=0.05)
out3 = torch.zeros(B, 800, device=dev, dtype=torch.bfloat16)
bias3 = torch.randn(784, device=dev)
run("g2 (K=400, sigmoid+bias)", lambda: gm_b200.gemm_bf16(A3, W3, out3, "nt", K=400, bias=bias3, act=2, pad_one=True, out_cols=800))
aux3 = torch.rand(B, 800, device=dev).to(torch.bfloat16)
run("dx (K=400, aux sigmoid-grad)", lambda: gm_b200.gemm_bf16(A3, W3, out3, "nt", K=400, aux=aux3, aux_mode=1))
