"""The two-grid split of the 128x208 K-major ping-pong GEMMs (engine.cu: companion_groups, launch_pp208), on the CPU.

A train-step plan of two or more rounds of 4-CTA clusters runs m-tiles [0, 4 g) as a main grid of 4-CTA clusters and
m-tiles [4 g, m_tiles) in pairs as a companion grid of 2-CTA clusters on the SMs the main grid leaves free (30 clusters of
4 and 6 of 2 on an H100 SXM's 132 SMs).  For every K-major 208-wide plan shape of the NSGAN, WGAN-GP and VAE train steps
at their benchmark batches, and at ragged M, the model checks that the two grids together compute every (m-tile,
n-tile) exactly once, that no CTA of either grid computes a tile past the product's last m-tile except the idle rank of
the companion's last pair, and that the split finishes in fewer round-times than the single grid.  The companion's
2-CTA ping-pong barrier schedule is played to completion with the model of test_gemm_pingpong4_cpu.py."""
import os
import random
import re

import pytest

import test_gemm_pingpong4_cpu as P4

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BM = 128
MAIN_CLUSTERS, COMP_CLUSTERS = 30, 6      # cudaOccupancyMaxActiveClusters of the 4-CTA instance; (132 - 120) / 2


def cdiv(a, b):
    return -(-a // b)


def companion_rate():
    src = open(os.path.join(ROOT, "generative-models_b200", "gm_b200", "csrc", "engine.cu")).read()
    return float(re.search(r"constexpr double kCompanionRate = ([0-9.]+);", src).group(1))


RATE = companion_rate()


def companion_groups(m_tiles, n_tiles, main=MAIN_CLUSTERS, comp=COMP_CLUSTERS, rate=RATE):
    """engine.cu companion_groups: 4-CTA m-tile groups of the main grid, 0 for one grid"""
    if comp < 1 or main < 1:
        return 0
    single = cdiv(cdiv(m_tiles, 4) * n_tiles, main)
    if single < 2:
        return 0
    best, best_t = 0, float(single)
    g = 1
    while 4 * g < m_tiles:
        t_main = float(cdiv(g * n_tiles, main))
        t_comp = cdiv(cdiv(m_tiles - 4 * g, 2) * n_tiles, comp) / rate
        t = max(t_main, t_comp)
        if t < best_t or (best and t == best_t):
            best, best_t = g, t
        g += 1
    return best


def grid_tiles(m_tile0, m_tiles, n_tiles, cl, clusters):
    """(m-tile, n-tile) of every CTA's items: gemm_wgmma.cuh m0_of / n_tile_of with item stride = clusters launched"""
    items = cdiv(m_tiles, cl) * n_tiles
    launched = min(items, clusters)        # launch_inst: CL x min(items, clusters)
    out = []
    for c in range(launched):
        for item in range(c, items, launched):
            for rank in range(cl):
                out.append((m_tile0 + (item // n_tiles) * cl + rank, item % n_tiles))
    return out


def rounds(m_tiles, n_tiles, g):
    """round-times of the split: main rounds, companion rounds at its rate"""
    return (cdiv(g * n_tiles, MAIN_CLUSTERS), cdiv(cdiv(m_tiles - 4 * g, 2) * n_tiles, COMP_CLUSTERS) / RATE)


# K-major 208-wide plan shapes (M, n-tiles) of the train steps: n-tiles 2 for the 400-wide hidden layers (out_cols 400
# or 416), 4 for the 784-wide image layers (784 or 800).  NSGAN and WGAN-GP at B = 65536 (D's first layer on 2B rows as
# well), the VAE at B = 131072.
STEP_SHAPES = [(M, n) for B in (65536, 131072) for M in (B, 2 * B) for n in (2, 4)]
RAGGED = [(128 * 131 + 5, 2), (128 * 131 + 5, 3), (128 * 510 + 77, 2), (128 * 510 + 77, 4), (2 * (128 * 510 + 77), 2),
          (128 * 100 + 64, 4), (7681, 2), (7680, 2), (128 * 61 + 1, 2), (130000, 2), (99999, 4)]


@pytest.mark.parametrize("M,n_tiles", STEP_SHAPES + RAGGED)
def test_main_and_companion_cover_every_tile_once(M, n_tiles):
    m_tiles = cdiv(M, BM)
    g = companion_groups(m_tiles, n_tiles)
    if g == 0:
        tiles = grid_tiles(0, m_tiles, n_tiles, 4, MAIN_CLUSTERS)
        extra = [t for t in tiles if t[0] >= m_tiles]
        assert len(extra) <= 3 * n_tiles     # the idle ranks of the last 4-tile group
    else:
        assert 1 <= g and 4 * g < m_tiles
        main = grid_tiles(0, 4 * g, n_tiles, 4, MAIN_CLUSTERS)
        comp = grid_tiles(4 * g, m_tiles - 4 * g, n_tiles, 2, COMP_CLUSTERS)
        assert all(m < 4 * g for m, _ in main)                    # the main grid stays inside its range, all rows < M
        assert all(4 * g <= m for m, _ in comp)
        extra = [t for t in comp if t[0] >= m_tiles]
        assert len(extra) == ((m_tiles - 4 * g) % 2) * n_tiles   # only the idle rank of an odd last pair, storing nothing
        tiles = main + comp
        t_main, t_comp = rounds(m_tiles, n_tiles, g)
        assert max(t_main, t_comp) < cdiv(cdiv(m_tiles, 4) * n_tiles, MAIN_CLUSTERS)
    inside = sorted(t for t in tiles if t[0] < m_tiles)
    assert inside == sorted((m, n) for m in range(m_tiles) for n in range(n_tiles))


def test_the_step_shapes_split():
    # the GEMMs of the benchmark batches: the main grid runs 16 rounds of 30 4-CTA clusters instead of 18, 8 instead of 9
    # and 32 instead of 35, and the companion finishes within them
    for m_tiles, n_tiles, single, main in ((512, 4, 18, 16), (1024, 2, 18, 16), (512, 2, 9, 8), (2048, 2, 35, 32)):
        g = companion_groups(m_tiles, n_tiles)
        assert g > 0 and cdiv(cdiv(m_tiles, 4) * n_tiles, MAIN_CLUSTERS) == single
        t_main, t_comp = rounds(m_tiles, n_tiles, g)
        assert t_main == main and t_comp < single, (m_tiles, n_tiles, g, t_main, t_comp)


def test_one_round_plans_keep_one_grid():
    for M in (1, 64, 128, 1000, 4096, 7680):
        for n_tiles in (1, 2, 4):
            m_tiles = cdiv(M, BM)
            if cdiv(cdiv(m_tiles, 4) * n_tiles, MAIN_CLUSTERS) < 2:
                assert companion_groups(m_tiles, n_tiles) == 0
    assert companion_groups(512, 4, comp=0) == 0                   # a device whose SMs all hold 4-CTA clusters


# companion rows (M - 4 g * 128) around the 64-row halves, odd and even pair counts
COMP_M = [1, 63, 64, 65, 128, 129, 192, 257, 320, 385, 449, 577, 769, 1024 + 77]


@pytest.mark.parametrize("M", COMP_M)
def test_companion_cluster2_schedule_completes(M, monkeypatch):
    """The companion grid is the ping-pong kernel at CL = 2 over M - 4 g * 128 rows starting at an m-tile base: halves_of
    and m0_of shift by whole tiles, so its schedule is that of a 2-CTA ping-pong GEMM on those rows."""
    monkeypatch.setattr(P4, "CL", 2)
    assert [P4.b_share_rows(r) for r in range(2)] == [104, 104]
    assert [P4.b_share_row0(r) for r in range(2)] == [0, 104]
    geo = P4.Geometry(True)
    assert geo.empty_count == 8                                    # one warpgroup per CTA, locally and on the peer
    rng = random.Random(M)
    for n_tiles in (1, 2, 4):
        for kblocks in (1, 2, 7, 13):
            for clusters in (1, 2, 3, COMP_CLUSTERS):
                P4.play(P4.Gemm(geo, M, n_tiles, kblocks, 1), clusters, seed=rng.randrange(1 << 30))
