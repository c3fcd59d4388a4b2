"""The 128x208 K-major GEMM's ping-pong instances (GPU): bias + ReLU / sigmoid epilogues with at most 7 k-blocks.

Consumer warpgroup g runs rows [64 g, 64 g + 64) of every tile as its own half-item, and a tile's second half is skipped
in both CTAs of a cluster when rank 0's first row of it is past M.  These cases cover M around the 64-row halves (M = 1,
64, 65, 128, 129, 192 and 128 k + 64, whose last cluster skips a half), one k-block (K <= 64, like G's first layer), the
last ping-pong K (448) and the first cooperative one (449), an odd item count per cluster, G's two GEMMs at B = 65536,
and repeatability.  Operands, bounds and checks are those of test_gemm_conformance_gpu.py, element by element against
float64."""
import pytest
import torch

import test_gemm_conformance_gpu as C
from test_gemm_cluster_gpu import NT208, _case

pytestmark = pytest.mark.gpu

# (M, K): single and double halves, and 128 k + 64 with k even (skipped half in the last cluster) and odd
M_CASES = [(1, 400), (64, 400), (65, 32), (128, 448), (129, 400), (192, 56), (320, 400), (448, 120), (576, 449)]
SHAPES = [_case("m%d_k%d_relu" % (M, K), M, 400, K, out_cols=416, seed=30 + i, bias=True, act=1, pad_one=True)
          for i, (M, K) in enumerate(M_CASES)]
SHAPES += [_case("m%d_k%d_sigmoid" % (M, K), M, 784, K, out_cols=800, seed=50 + i, bias=True, act=2, pad_one=True)
           for i, (M, K) in enumerate(M_CASES[::2])]
# 51 m-tile pairs (the last one with a skipped half) x 4 n-tiles = 204 items: 3 or 4 per cluster
SHAPES += [_case("m12864_sigmoid_odd_items", 128 * 100 + 64, 784, 400, out_cols=800, seed=60, bias=True, act=2, pad_one=True)]

# G's two layers at B = 65536: [B, 32 (+ ones column)] x W1g^T with ReLU, [B, 416] x W2g^T with sigmoid
B = 65536
STEP = [
    _case("g1", B, 400, 32, out_cols=416, seed=70, bias=True, act=1, pad_one=True),
    _case("g2", B, 784, 400, out_cols=800, seed=71, bias=True, act=2, pad_one=True),
]


@pytest.mark.parametrize("c", SHAPES + STEP, ids=[c["name"] for c in SHAPES + STEP])
def test_pingpong_gemm_matches_float64(c):
    T, counts, launches = C._run_counted(c)
    assert counts == [int(k == NT208) for k in range(4)] and launches == 1, (c["name"], counts, launches)
    C._check(c, T)


def test_pingpong_gemm_repeats_bit_for_bit():
    for c in (SHAPES[0], SHAPES[6], SHAPES[-1], STEP[1]):
        T1, T2 = C._run(c), C._run(c)
        assert torch.equal(T1["out"].view(torch.int16), T2["out"].view(torch.int16)), c["name"]
