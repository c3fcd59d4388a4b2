"""The 128x208 K-major GEMM as 2-CTA clusters (GPU): shapes the conformance cases do not reach.

Each cluster takes two adjacent m-tiles of one n-tile and multicasts the shared B tile into both CTAs.  These cases cover an
odd m-tile count (the second CTA of the last cluster has no rows to store), item counts that do not divide evenly over
the clusters, the train step's own GEMM shapes and epilogues at B = 65536, split-K fp32 over an odd number of m-tile pairs,
and repeatability.  Operands, bounds and checks are those of test_gemm_conformance_gpu.py, element by element against
float64."""
import pytest
import torch

import test_gemm_conformance_gpu as C

pytestmark = pytest.mark.gpu
NT208 = C.KINDS["nt208"]


def _case(name, M, N, K, out_cols=None, seed=0, **epi):
    oc = out_cols or N
    k8 = (K + 7) // 8 * 8
    c = dict(name=name, mode="nt", M=M, N=N, K=K, out="bf16", out_cols=oc, ldc=oc, lda=k8, ldb=k8, bias=False, act=0, slope=0.2,
             aux=0, dot=False, sse=False, pad_one=False, transpose=False, tile="nt208", group="cluster", seed=500 + seed)
    c.update(epi)
    return c


# m-tiles: 3 and 131 (odd), 132, 138; items (m-tile pairs x n-tiles) 2 x 2, 66 x 2, 66 x 3, 69 x 2
RAGGED = [
    _case("m300_relu_dot", 300, 400, 784, out_cols=416, seed=1, bias=True, act=1, dot=True, pad_one=True),
    _case("m300_plain", 300, 208, 120, seed=2),
    _case("m16645_aux1", 128 * 130 + 5, 400, 400, out_cols=416, seed=3, aux=1),
    _case("m16773_sigmoid", 128 * 131 + 5, 624, 65, seed=4, bias=True, act=2),
    _case("m16773_aux2", 128 * 131 + 5, 400, 784, out_cols=416, seed=5, aux=2),
    _case("m17613_lrelu", 128 * 137 + 77, 256, 56, seed=6, act=3),
]

# the NSGAN step at B = 65536: G's output layer, D's hidden layer over real + fake rows, dL/dfake and dL/dHg
B = 65536
STEP = [
    _case("g2", B, 784, 400, out_cols=800, seed=10, bias=True, act=2, pad_one=True),
    _case("d1", 2 * B, 400, 784, out_cols=416, seed=11, bias=True, act=1, dot=True, pad_one=True),
    _case("dx", B, 784, 400, seed=12, aux=1),
    _case("dhg", B, 400, 784, out_cols=416, seed=13, aux=2),
]


@pytest.mark.parametrize("c", RAGGED + STEP, ids=[c["name"] for c in RAGGED + STEP])
def test_cluster_gemm_matches_float64(c):
    T, counts, launches = C._run_counted(c)
    assert counts == [int(k == NT208) for k in range(4)] and launches == 1, (c["name"], counts, launches)
    C._check(c, T)


# split-K fp32: 5 m-tiles (3 pairs, the last one half empty) x 2 n-tiles x 13 splits of one k-block each
SPLIT = dict(_case("f32_split_m600", 600, 400, 784, seed=20), out="f32", ldc=404, split=True, group="cluster_f32")


@pytest.mark.parametrize("transpose", [False, True])
def test_cluster_split_k_fp32_matches_float64(transpose):
    c = dict(SPLIT, transpose=transpose, ldc=608 if transpose else 404, name=SPLIT["name"] + ("_T" if transpose else ""))
    T, counts, launches = C._run_counted(c)
    assert counts == [int(k == NT208) for k in range(4)] and launches == 2, (c["name"], counts, launches)   # + the reduction
    C._check(c, T)


def test_cluster_gemm_repeats_bit_for_bit():
    for c in (RAGGED[0], STEP[1], SPLIT):
        T1, T2 = C._run(c), C._run(c)
        assert torch.equal(T1["out"].view(torch.int16), T2["out"].view(torch.int16)), c["name"]
        if "slots" in T1:
            assert torch.equal(T1["slots"].view(torch.int32), T2["slots"].view(torch.int32)), c["name"]
