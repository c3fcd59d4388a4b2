"""A CPU model of the ping-pong schedule of the 128x208 K-major GEMM (gemm_wgmma.cuh, PINGPONG), played to completion.

Both CTAs of a cluster are modelled with their TMA producer and their two consumer warpgroups, following the kernel's
item, half-item, skip and stage / phase rules line for line: the full / empty mbarriers (arrival counts, transaction
bytes, phase parity), the multicast B shares landing in both CTAs, the release of each stage in the own and the peer
CTA, and the named-barrier handoff of the mainloops.  A random scheduler interleaves the agents and the TMA deliveries.
The model asserts that every wait is eventually satisfied (no deadlock), that each stage is read by exactly the half-item
the producers filled it for, that no delivery lands in a stage while it is being read, and that every barrier is idle
when the kernel ends."""
import random

import pytest

BM, BK, BN, CL = 128, 64, 208, 2
A_ROWS = BM // 2
STAGES = 5
A_BYTES, B_BYTES = A_ROWS * BK * 2, BN * BK * 2
STAGE_BYTES = A_BYTES + B_BYTES
WG_THREADS = 128
EMPTY_COUNT = CL * 4          # ping-pong: one warpgroup (4 warps) per CTA reads a stage, arriving locally and on the peer
BAR_WG0_ISSUED, BAR_WG1_ISSUED = 1, 2


class MBar:
    def __init__(self, count):
        self.count, self.pending, self.tx, self.phase = count, count, 0, 0

    def _check(self):
        if self.pending == 0 and self.tx == 0:
            self.phase += 1
            self.pending = self.count

    def arrive(self):
        assert self.pending > 0
        self.pending -= 1
        self._check()

    def arrive_expect_tx(self, nbytes):
        self.tx += nbytes
        self.arrive()

    def complete_tx(self, nbytes):
        self.tx -= nbytes
        self._check()

    def done(self, parity):   # mbarrier.try_wait.parity: the phase of this parity has completed
        return (self.phase & 1) != parity


class NamedBar:
    def __init__(self, threads):
        self.threads, self.arrived, self.gen = threads, 0, 0

    def add(self):
        self.arrived += WG_THREADS
        gen = self.gen
        if self.arrived == self.threads:
            self.arrived, self.gen = 0, self.gen + 1
        return gen


class Cta:
    def __init__(self):
        self.full = [MBar(1) for _ in range(STAGES)]
        self.empty = [MBar(EMPTY_COUNT) for _ in range(STAGES)]
        self.named = {BAR_WG0_ISSUED: NamedBar(2 * WG_THREADS), BAR_WG1_ISSUED: NamedBar(2 * WG_THREADS)}
        self.smem = [dict() for _ in range(STAGES)]    # part -> tag of the data that landed
        self.readers = [set() for _ in range(STAGES)]  # warpgroups whose wgmmas may still read the stage


class Gemm:
    """plan_gemm's split / k-block arithmetic for a K-major 208-wide plan"""

    def __init__(self, M, n_tiles, kblocks, max_splits):
        self.M, self.n_tiles = M, n_tiles
        self.m_tiles = -(-M // BM)
        self.kblocks = kblocks
        splits = max(1, min(max_splits, self.kblocks))
        self.kb_per_split = -(-self.kblocks // splits)
        self.splits = -(-self.kblocks // self.kb_per_split)
        self.tiles = -(-self.m_tiles // CL) * n_tiles
        self.total = self.tiles * self.splits

    def halves_of(self, rem):
        return 2 if (rem // self.n_tiles) * CL * BM + A_ROWS < self.M else 1

    def item(self, item):
        split = item // self.tiles
        rem = item - split * self.tiles
        kb0 = split * self.kb_per_split
        return rem, kb0, min(kb0 + self.kb_per_split, self.kblocks), self.halves_of(rem)


def producer(g, ctas, rank, first, stride, deliveries):
    me = ctas[rank]
    it = 0
    for item in range(first, g.total, stride):
        rem, kb0, kb1, nh = g.item(item)
        for h in range(nh):
            for kb in range(kb0, kb1):
                stage, phase = it % STAGES, (it // STAGES) & 1
                yield lambda: me.empty[stage].done(phase ^ 1)
                me.full[stage].arrive_expect_tx(STAGE_BYTES)
                deliveries.append((rank, stage, "A", (item, rank, h, kb), A_BYTES))
                for dst in range(CL):   # multicast: this CTA's share of the B rows into both CTAs
                    deliveries.append((dst, stage, "B%d" % rank, (item, h, kb), B_BYTES // CL))
                it += 1


def consumer(g, ctas, rank, wg, first, stride, log):
    me, peer = ctas[rank], ctas[rank ^ 1]

    def named_sync(bar_id):
        gen = me.named[bar_id].add()
        yield lambda: me.named[bar_id].gen > gen

    def release(s):
        me.readers[s].discard(wg)
        for _ in range(4):      # every warp of the warpgroup, locally and on the peer
            me.empty[s].arrive()
            peer.empty[s].arrive()

    it = 0
    for item in range(first, g.total, stride):
        rem, kb0, kb1, nh = g.item(item)
        if wg == 1 or it != 0:
            yield from named_sync(BAR_WG0_ISSUED if wg == 1 else BAR_WG1_ISSUED)
        if wg == 1 and nh == 1:
            it += kb1 - kb0
            if item + stride < g.total:
                me.named[BAR_WG1_ISSUED].add()
            continue
        prev = -1
        it0 = it + (kb1 - kb0 if wg == 1 else 0)
        stage, phase = it0 % STAGES, (it0 // STAGES) & 1
        it += nh * (kb1 - kb0)
        for kb in range(kb0, kb1):
            yield lambda s=stage, ph=phase: me.full[s].done(ph)
            want = {"A": (item, rank, wg, kb), "B0": (item, wg, kb), "B1": (item, wg, kb)}
            assert me.smem[stage] == want, (rank, wg, item, kb, me.smem[stage], want)
            me.readers[stage].add(wg)
            log.append((rank, wg, item, kb))
            if prev >= 0:
                release(prev)
            prev = stage
            stage += 1
            if stage == STAGES:
                stage, phase = 0, phase ^ 1
        if wg == 0 or item + stride < g.total:
            me.named[BAR_WG0_ISSUED if wg == 0 else BAR_WG1_ISSUED].add()
        if prev >= 0:
            release(prev)
        yield lambda: True      # the epilogue: any other agent may run meanwhile


def play_cluster(g, first, stride, rng):
    ctas = [Cta() for _ in range(CL)]
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
            for wg in range(nh):
                want += [(r, wg, item, kb) for kb in range(kb0, kb1)]
    return sorted(want)


def play(g, grid, seed):
    clusters = min(g.total, grid // CL)   # launch_inst: CL x min(items, clusters resident at once)
    rng = random.Random(seed)
    for c in range(clusters):
        log = play_cluster(g, c, clusters, rng)
        assert sorted(log) == expected_reads(g, c, clusters)


M_VALUES = [1, 63, 64, 65, 127, 128, 129, 191, 192, 193, 255, 256, 257, 319, 320, 321, 383, 384, 447, 448, 449, 575, 576,
            577, 640]


@pytest.mark.parametrize("M", M_VALUES)
def test_pingpong_schedule_completes(M):
    rng = random.Random(M)
    for n_tiles in range(1, 5):
        for splits in range(1, 4):
            for kblocks in (1, 2, 3, 5, 7, 13, 14):
                for grid in (2, 4, 6, rng.randrange(8, 133, 2), 132):
                    play(Gemm(M, n_tiles, kblocks, splits), grid, seed=rng.randrange(1 << 30))

