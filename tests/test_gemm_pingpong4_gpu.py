"""The 128x208 K-major GEMM's ping-pong instances as 4-CTA clusters (GPU), for every epilogue gm_gemm_bf16 selects one for.

A cluster takes four adjacent m-tiles of one n-tile; each rank multicasts its 56- or 48-row share of the B tile into all
four CTAs, and a tile's second 64-row half is skipped in all four when rank 0's first row of it is past M.  The cases
cover m-tile counts of every residue mod 4 (M = 1, 64, 65, 128, 129, 257, 385 and 512 k + 64 / 512 k + 320, whose last
cluster has idle ranks or a skipped half), one k-block up to the step's longest K with a ragged last block (33, 400,
449, 784, 785), both n-tile counts of the step (N = 400, 784), item counts that do not divide over the clusters, and
repeatability.  The plain, bias + ReLU / sigmoid, row-dot (DOT_W), AUX_SIGMOID_GRAD, AUX_RELU_MASK and AUX_VAE_OUT
signatures are reached here; the G step's, WGAN-GP's and BEGAN's own signatures run in the engine tests against the
float64 oracle.  Operands, bounds and checks are those of test_gemm_conformance_gpu.py, element by element against
float64."""
import pytest
import torch

import test_gemm_conformance_gpu as C
from test_gemm_cluster_gpu import NT208, _case

pytestmark = pytest.mark.gpu

SIGS = {
    "plain": dict(),
    "relu": dict(bias=True, act=1, pad_one=True),
    "sigmoid": dict(bias=True, act=2, pad_one=True),
    "relu_dot": dict(bias=True, act=1, dot=True, pad_one=True),
    "aux1": dict(aux=1),
    "aux2": dict(aux=2),
    "vae_out": dict(bias=True, act=2, aux=3, sse=True),
}
M_VALUES = [1, 64, 65, 128, 129, 257, 385, 512 + 64, 512 + 320, 512 * 9 + 64, 512 * 9 + 320]
K_VALUES = [33, 400, 449, 784, 785]
N_VALUES = [400, 784]


def _out_cols(N, sig):
    return N + 16 if sig.get("pad_one") else N


# every signature at every M; K and N rotate with the M index so that each signature meets every K and both N
CASES = []
for si, (sname, sig) in enumerate(SIGS.items()):
    for mi, M in enumerate(M_VALUES):
        K = K_VALUES[(mi + si) % len(K_VALUES)]
        N = N_VALUES[(mi + si) % len(N_VALUES)]
        CASES.append(_case("%s_m%d_n%d_k%d" % (sname, M, N, K), M, N, K, out_cols=_out_cols(N, sig),
                           seed=100 + 16 * si + mi, **sig))
# the whole K x N grid for two ragged M, with the row-dot and the aux-mask epilogues
for sname in ("relu_dot", "aux2"):
    for M in (385, 512 * 3 + 320):
        for K in K_VALUES:
            for N in N_VALUES:
                CASES.append(_case("%s_grid_m%d_n%d_k%d" % (sname, M, N, K), M, N, K, out_cols=_out_cols(N, SIGS[sname]),
                                   seed=300 + K + N + M, **SIGS[sname]))


@pytest.mark.parametrize("c", CASES, ids=[c["name"] for c in CASES])
def test_pingpong4_gemm_matches_float64(c):
    T, counts, launches = C._run_counted(c)
    assert counts == [int(k == NT208) for k in range(4)] and launches == 1, (c["name"], counts, launches)
    C._check(c, T)


def test_pingpong4_gemm_repeats_bit_for_bit():
    for c in (CASES[len(M_VALUES) * 3 + 8], CASES[len(M_VALUES) * 6 + 7]):   # row-dot and VAE output at 512 + 320 / + 64
        T1, T2 = C._run(c), C._run(c)
        assert torch.equal(T1["out"].view(torch.int16), T2["out"].view(torch.int16)), c["name"]
        assert torch.equal(T1["slots"].view(torch.int32), T2["slots"].view(torch.int32)), c["name"]
