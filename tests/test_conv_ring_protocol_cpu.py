"""CPU model of the operand-ring protocol of the persistent conv kernel (csrc/conv_tc.cu `conv_tc_persistent_kernel`): one TMA
producer and eight consumer warps share a ring of full / empty mbarriers, and the ring position (stage, phase) carries over from
tile to tile.  The model runs the producer loop of `produce_kblocks` and the consumer loop of `consume_kblocks` plus the release
of a tile's last stage, under random interleavings, for tile counts that do not divide over the CTAs.  It checks that no wait
deadlocks, that every consumer reads each (tile, K-block) exactly once and in order, and that the producer never refills a stage
before all eight warps have released it."""
import random

import pytest

CONSUMER_WARPS = 8


class MBar:
    """mbarrier with an expected arrival count; try_wait.parity(P) succeeds once the phase of parity P has completed."""

    def __init__(self, count):
        self.count, self.pending, self.phase = count, count, 0

    def arrive(self):
        self.pending -= 1
        assert self.pending >= 0
        if self.pending == 0:
            self.phase ^= 1
            self.pending = self.count

    def try_wait(self, parity):
        return self.phase != parity


def producer(cta, grid, tiles, kblocks, stages, full, empty, ring, log):
    stage, phase = 0, 0
    for t in range(cta, tiles, grid):
        for kb in range(kblocks):
            while not empty[stage].try_wait(phase ^ 1):
                yield
            assert ring[stage] is None, f"stage {stage} refilled before all consumers released it"
            ring[stage] = (t, kb)  # TMA lands: expect_tx arrive + complete_tx in one step
            log.append(("load", t, kb))
            full[stage].arrive()
            stage += 1
            if stage == stages:
                stage, phase = 0, phase ^ 1
            yield


def consumer(warp, cta, grid, tiles, kblocks, stages, full, empty, ring, readers, seen):
    stage, phase = 0, 0
    for t in range(cta, tiles, grid):
        prev = -1
        for kb in range(kblocks):
            while not full[stage].try_wait(phase):
                yield
            assert ring[stage] == (t, kb), f"warp {warp} expected {(t, kb)}, stage {stage} holds {ring[stage]}"
            seen[warp].append((t, kb))
            yield  # wgmma in flight; wait_group 1 retires the previous stage's group
            if prev >= 0:
                release(prev, ring, readers, empty)
            prev = stage
            stage += 1
            if stage == stages:
                stage, phase = 0, phase ^ 1
        yield  # wait_group 0
        release(prev, ring, readers, empty)  # the tile's last stage, before the epilogue
        for _ in range(3):  # epilogue: the producer runs ahead meanwhile
            yield


def release(stage, ring, readers, empty):
    readers[stage] += 1
    if readers[stage] == CONSUMER_WARPS:
        readers[stage] = 0
        ring[stage] = None
    empty[stage].arrive()


def run_cta(cta, grid, tiles, kblocks, stages, seed):
    full = [MBar(1) for _ in range(stages)]
    empty = [MBar(CONSUMER_WARPS) for _ in range(stages)]
    ring, readers = [None] * stages, [0] * stages
    log, seen = [], [[] for _ in range(CONSUMER_WARPS)]
    agents = [producer(cta, grid, tiles, kblocks, stages, full, empty, ring, log)]
    agents += [consumer(w, cta, grid, tiles, kblocks, stages, full, empty, ring, readers, seen) for w in range(CONSUMER_WARPS)]
    rng = random.Random(seed)
    live, steps = list(agents), 0
    while live:
        a = rng.choice(live)
        try:
            next(a)
        except StopIteration:
            live.remove(a)
        steps += 1
        assert steps < 200000, "deadlock: no agent finished"
    want = [(t, kb) for t in range(cta, tiles, grid) for kb in range(kblocks)]
    assert [(t, kb) for _, t, kb in log] == want
    for w in range(CONSUMER_WARPS):
        assert seen[w] == want, f"warp {w} of CTA {cta}"
    assert all(r is None for r in ring)


@pytest.mark.parametrize("stages", [4, 6, 8])
@pytest.mark.parametrize("tiles,grid,kblocks", [(200, 132, 2), (512, 132, 9), (7, 3, 5), (5, 5, 1), (10, 4, 4), (3, 132, 3)])
def test_ring_carries_over_tiles(tiles, grid, kblocks, stages):
    for cta in sorted({0, min(grid, tiles) - 1, (tiles - 1) % grid, tiles % grid}):
        if cta < min(grid, tiles):
            run_cta(cta, min(grid, tiles), tiles, kblocks, stages, seed=cta * 7919 + tiles)
