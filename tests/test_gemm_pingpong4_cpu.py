"""A CPU model of the 128x208 K-major GEMM's 4-CTA cluster schedule (gemm_wgmma.cuh, CL = 4), played to completion.

All four CTAs of a cluster are modelled with their TMA producer and their two consumer warpgroups, in ping-pong and in
the cooperative loop that the universal, split-operand and fp32-output instances keep.  The model follows the kernel's
item, half-item, skip and stage / phase rules: each rank multicasts its B share (56, 56, 48 and 48 rows, b_share_rows)
into all four CTAs, every full barrier expects the whole stage, and every consumer warp releases a stage it read on its
own empty barrier and, by remote arrive, on the three peers'.  A random scheduler interleaves the agents and the TMA
deliveries.  The model asserts that every wait is eventually satisfied (no deadlock), that each stage is read by exactly
the (half-)item the producers filled it for, that no delivery lands in a stage while it is being read, and that every
barrier is idle when the kernel ends."""
import random

import pytest

from test_gemm_pingpong_cpu import MBar, NamedBar

BM, BK, BN, CL = 128, 64, 208, 4
WG_THREADS = 128
BAR_WG0_ISSUED, BAR_WG1_ISSUED = 1, 2


def b_share_rows(r):    # gemm_wgmma.cuh b_share_rows(BN, CL, r)
    return 8 * (BN // 8 // CL + (r < BN // 8 % CL))


def b_share_row0(r):
    return 8 * (r * (BN // 8 // CL) + min(r, BN // 8 % CL))


def test_b_shares_tile_the_b_tile_on_swizzle_atoms():
    rows = [b_share_rows(r) for r in range(CL)]
    starts = [b_share_row0(r) for r in range(CL)]
    assert rows == [56, 56, 48, 48]
    assert [s * BK * 2 for s in starts] == [0, 7168, 14336, 20480]   # stage offsets: whole 1 KB atoms
    assert all(s + n == e for s, n, e in zip(starts, rows, starts[1:] + [BN]))
    # the feed per 128 rows and k-block: ping-pong loads A and the own B share once per 64-row half
    avg_share = BN * BK * 2 // CL
    assert 2 * (BM // 2 * BK * 2 + avg_share) == 29696


class Geometry:
    def __init__(self, pingpong):
        self.pingpong = pingpong
        self.a_rows = BM // 2 if pingpong else BM
        self.stages = 5 if pingpong else 4
        self.a_bytes = self.a_rows * BK * 2
        self.stage_bytes = self.a_bytes + BN * BK * 2
        # ping-pong: one warpgroup (4 warps) per CTA reads a stage; cooperative: both (8 warps).  Each arrives locally
        # and on every peer.
        self.empty_count = CL * (4 if pingpong else 8)


class Cta:
    def __init__(self, geo):
        self.full = [MBar(1) for _ in range(geo.stages)]
        self.empty = [MBar(geo.empty_count) for _ in range(geo.stages)]
        self.named = {BAR_WG0_ISSUED: NamedBar(2 * WG_THREADS), BAR_WG1_ISSUED: NamedBar(2 * WG_THREADS)}
        self.smem = [dict() for _ in range(geo.stages)]    # part -> tag of the data that landed
        self.readers = [set() for _ in range(geo.stages)]  # warpgroups whose wgmmas may still read the stage


class Gemm:
    """plan_gemm's split / k-block arithmetic for a K-major 208-wide plan"""

    def __init__(self, geo, M, n_tiles, kblocks, max_splits):
        self.geo, self.M, self.n_tiles = geo, M, n_tiles
        self.m_tiles = -(-M // BM)
        self.kblocks = kblocks
        splits = max(1, min(max_splits, self.kblocks))
        self.kb_per_split = -(-self.kblocks // splits)
        self.splits = -(-self.kblocks // self.kb_per_split)
        self.tiles = -(-self.m_tiles // CL) * n_tiles
        self.total = self.tiles * self.splits

    def halves_of(self, rem):
        if not self.geo.pingpong:
            return 1
        return 2 if (rem // self.n_tiles) * CL * BM + self.geo.a_rows < self.M else 1

    def item(self, item):
        split = item // self.tiles
        rem = item - split * self.tiles
        kb0 = split * self.kb_per_split
        return rem, kb0, min(kb0 + self.kb_per_split, self.kblocks), self.halves_of(rem)


def producer(g, ctas, rank, first, stride, deliveries):
    geo, me = g.geo, ctas[rank]
    it = 0
    for item in range(first, g.total, stride):
        rem, kb0, kb1, nh = g.item(item)
        for h in range(nh):
            for kb in range(kb0, kb1):
                stage, phase = it % geo.stages, (it // geo.stages) & 1
                yield lambda: me.empty[stage].done(phase ^ 1)
                me.full[stage].arrive_expect_tx(geo.stage_bytes)
                deliveries.append((rank, stage, "A", (item, rank, h, kb), geo.a_bytes))
                for dst in range(CL):   # multicast: this rank's share of the B rows into every CTA
                    deliveries.append((dst, stage, "B%d" % rank, (item, h, kb), b_share_rows(rank) * BK * 2))
                it += 1


def consumer(g, ctas, rank, wg, first, stride, log):
    geo, me = g.geo, ctas[rank]
    pp = geo.pingpong

    def named_sync(bar_id):
        gen = me.named[bar_id].add()
        yield lambda: me.named[bar_id].gen > gen

    def release(s):
        me.readers[s].discard(wg)
        for _ in range(4):      # every warp of the warpgroup, locally and by remote arrive on the 3 peers
            me.empty[s].arrive()
            for d in range(1, CL):
                ctas[rank ^ d].empty[s].arrive()

    it = 0
    stage, phase = 0, 0
    for item in range(first, g.total, stride):
        rem, kb0, kb1, nh = g.item(item)
        if pp:
            if wg == 1 or it != 0:
                yield from named_sync(BAR_WG0_ISSUED if wg == 1 else BAR_WG1_ISSUED)
            if wg == 1 and nh == 1:
                it += kb1 - kb0
                if item + stride < g.total:
                    me.named[BAR_WG1_ISSUED].add()
                continue
            it0 = it + (kb1 - kb0 if wg == 1 else 0)
            stage, phase = it0 % geo.stages, (it0 // geo.stages) & 1
            it += nh * (kb1 - kb0)
        prev = -1
        for kb in range(kb0, kb1):
            yield lambda s=stage, ph=phase: me.full[s].done(ph)
            h = wg if pp else 0
            want = {"A": (item, rank, h, kb)}
            want.update({"B%d" % r: (item, h, kb) for r in range(CL)})
            assert me.smem[stage] == want, (rank, wg, item, kb, me.smem[stage], want)
            me.readers[stage].add(wg)
            log.append((rank, wg, item, kb))
            if prev >= 0:
                release(prev)
            prev = stage
            stage += 1
            if stage == geo.stages:
                stage, phase = 0, phase ^ 1
        if pp and (wg == 0 or item + stride < g.total):
            me.named[BAR_WG0_ISSUED if wg == 0 else BAR_WG1_ISSUED].add()
        if prev >= 0:
            release(prev)
        yield lambda: True      # the epilogue: any other agent may run meanwhile


def play_cluster(g, first, stride, rng):
    ctas = [Cta(g.geo) for _ in range(CL)]
    deliveries, log = [], []
    agents = []
    for r in range(CL):
        agents.append(producer(g, ctas, r, first, stride, deliveries))
        agents += [consumer(g, ctas, r, wg, first, stride, log) for wg in range(2)]
    waits = [lambda: True] * len(agents)
    live = list(range(len(agents)))
    while live or deliveries:
        ready = [a for a in live if waits[a]()]
        choices = ready + (["tma"] if deliveries else [])
        assert choices, "deadlock: %d agents wait forever" % len(live)
        pick = rng.choice(choices)
        if pick == "tma":
            dst, s, part, tag, nbytes = deliveries.pop(rng.randrange(len(deliveries)))
            assert not ctas[dst].readers[s], "a TMA delivery landed in a stage that is being read"
            ctas[dst].smem[s][part] = tag
            ctas[dst].full[s].complete_tx(nbytes)
            continue
        try:
            waits[pick] = next(agents[pick])
        except StopIteration:
            live.remove(pick)
    for c in ctas:
        assert all(b.pending == b.count and b.tx == 0 for b in c.full + c.empty), "mbarrier not idle at exit"
        assert all(n.arrived == 0 for n in c.named.values()), "named barrier left with arrivals at exit"
        assert not any(c.readers), "stage still being read at exit"
    return log


def expected_reads(g, first, stride):
    want = []
    for item in range(first, g.total, stride):
        rem, kb0, kb1, nh = g.item(item)
        for r in range(CL):
            for wg in (range(nh) if g.geo.pingpong else range(2)):
                want += [(r, wg, item, kb) for kb in range(kb0, kb1)]
    return sorted(want)


def play(g, clusters_resident, seed):
    clusters = min(g.total, clusters_resident)   # launch_inst: CL x min(items, clusters resident at once)
    rng = random.Random(seed)
    for c in range(clusters):
        log = play_cluster(g, c, clusters, rng)
        assert sorted(log) == expected_reads(g, c, clusters)


# m-tile counts 1..8 (every residue mod 4) at and around each 64-row half boundary
M_VALUES = [1, 63, 64, 65, 128, 129, 192, 193, 257, 320, 385, 448, 449, 512, 513, 576, 577, 704, 769, 1024]


@pytest.mark.parametrize("pingpong", [True, False], ids=["pingpong", "cooperative"])
@pytest.mark.parametrize("M", M_VALUES)
def test_cluster4_schedule_completes(M, pingpong):
    geo = Geometry(pingpong)
    rng = random.Random(M * 2 + pingpong)
    for n_tiles in (1, 2, 3):
        for splits in (1, 3):
            for kblocks in (1, 2, 6, 7, 13):
                # 33 is what 132 SMs hold at most; fewer clusters than items leaves a ragged last round
                for clusters in (1, 2, 3, rng.randrange(4, 34), 33):
                    play(Gemm(geo, M, n_tiles, kblocks, splits), clusters, seed=rng.randrange(1 << 30))
