"""CPU model of the staging-tile handshakes of the persistent conv kernel's TMA epilogue (csrc/conv_tc.cu
`conv_tc_persistent_kernel`), on top of the operand ring of tests/test_conv_ring_protocol_cpu.py.  Per tile the producer loads the
first ring-full of K-blocks, waits on `stg_free` (the previous tile's store has been read out of the staging tile), TMA-loads the
residual into the staging tile and signals `stg_full` (a plain arrive without a residual), then loads the remaining K-blocks.
The eight consumer warps run the K loop; consumer thread 0 (warp 0), after issuing a tile's first wgmma group, waits for the
previous store's read-out and arrives on `stg_free`.  After the K loop every warp waits on `stg_full`, reads its rows' residual,
writes its rows' output in place, and after a named barrier warp 0 issues the TMA store, which the store engine reads out of shared
memory later.  With the staging tile holding one column half at a time (BN 256), warp 0 waits for the first half's read-out, loads
the second half's residual (or merely arrives) on `stg_full`, and the consumers repeat the epilogue for that half.  Under random interleavings and tile counts that do not divide over the CTAs, with and without a residual, the model
checks: no deadlock; a residual never lands while a store still reads the staging tile or before every warp has finished the
previous tile; every warp reads its own tile's residual; every store reads exactly its tile's output; stores leave in tile order."""
import random

import pytest

from tests.test_conv_ring_protocol_cpu import CONSUMER_WARPS, MBar, release


class Staging:
    def __init__(self):
        self.rows = [None] * CONSUMER_WARPS  # per warp's rows: ("res" | "out", tile)
        self.stores = []                     # issued stores: [tile, read out, complete]
        self.bar_count, self.bar_gen = 0, 0  # named barrier over the consumer warps


def producer(tiles_of, kblocks, stages, res, halves, full, empty, ring, stg, stg_free, stg_full):
    stage, phase = 0, 0
    kres = min(stages, kblocks)

    def load(t, kb0, kb1):
        nonlocal stage, phase
        for kb in range(kb0, kb1):
            while not empty[stage].try_wait(phase ^ 1):
                yield
            assert ring[stage] is None
            ring[stage] = (t, kb)
            full[stage].arrive()
            stage += 1
            if stage == stages:
                stage, phase = 0, phase ^ 1
            yield

    for i, t in enumerate(tiles_of):
        yield from load(t, 0, kres)
        if i > 0:
            while not stg_free.try_wait((i - 1) & 1):
                yield
        assert all(s[1] for s in stg.stores), "residual load while a store still reads the staging tile"
        if res:
            assert all(r == ("out", (tiles_of[i - 1], halves - 1)) for r in stg.rows) if i > 0 else True, "residual load before the previous tile was written"
            yield  # the TMA load is in flight
            stg.rows = [("res", (t, 0))] * CONSUMER_WARPS
        stg_full.arrive()
        yield from load(t, kres, kblocks)


def consumer(warp, tiles_of, kblocks, stages, res, halves, full, empty, ring, readers, stg, stg_free, stg_full):
    stage, phase, sp = 0, 0, 0
    for i, t in enumerate(tiles_of):
        prev = -1
        for kb in range(kblocks):
            while not full[stage].try_wait(phase):
                yield
            assert ring[stage] == (t, kb)
            yield  # wgmma group issued
            if kb == 0 and warp == 0 and i > 0:
                while not stg.stores[-1][1]:  # cp.async.bulk.wait_group.read 0
                    yield
                stg_free.arrive()
            if prev >= 0:
                release(prev, ring, readers, empty)
            prev = stage
            stage += 1
            if stage == stages:
                stage, phase = 0, phase ^ 1
        yield  # wait_group 0
        release(prev, ring, readers, empty)
        for h in range(halves):
            if h > 0 and warp == 0:  # the previous half's store is read out, then this half's residual comes in
                while not stg.stores[-1][1]:
                    yield
                if res:
                    yield
                    stg.rows = [("res", (t, h))] * CONSUMER_WARPS
                stg_full.arrive()
            while not stg_full.try_wait(sp):
                yield
            sp ^= 1
            if res:
                assert stg.rows[warp] == ("res", (t, h)), f"warp {warp} tile {t} half {h} reads {stg.rows[warp]}"
            yield
            stg.rows[warp] = ("out", (t, h))
            gen = stg.bar_gen  # named barrier
            stg.bar_count += 1
            if stg.bar_count == CONSUMER_WARPS:
                stg.bar_count, stg.bar_gen = 0, gen + 1
            while stg.bar_gen == gen:
                yield
            if warp == 0:
                stg.stores.append([(t, h), False, False])
    if warp == 0:
        while not all(s[2] for s in stg.stores):  # drain before exit
            yield


def store_engine(stg, out, done):
    while not (done() and all(s[2] for s in stg.stores)):
        for s in stg.stores:
            if not s[1]:
                yield
                assert all(r == ("out", s[0]) for r in stg.rows), f"store of tile {s[0]} reads {stg.rows}"
                out.append(s[0])
                s[1] = True
            elif not s[2]:
                yield
                s[2] = True
        yield


def run_cta(cta, grid, tiles, kblocks, stages, res, halves, seed):
    tiles_of = list(range(cta, tiles, grid))
    full = [MBar(1) for _ in range(stages)]
    empty = [MBar(CONSUMER_WARPS) for _ in range(stages)]
    ring, readers = [None] * stages, [0] * stages
    stg, stg_free, stg_full, out = Staging(), MBar(1), MBar(1), []
    agents = [producer(tiles_of, kblocks, stages, res, halves, full, empty, ring, stg, stg_free, stg_full)]
    consumers = [consumer(w, tiles_of, kblocks, stages, res, halves, full, empty, ring, readers, stg, stg_free, stg_full)
                 for w in range(CONSUMER_WARPS)]
    agents += consumers
    live = list(agents)
    agents.append(store_engine(stg, out, lambda: not any(c in live for c in consumers)))
    live.append(agents[-1])
    rng = random.Random(seed)
    steps = 0
    while live:
        a = rng.choice(live)
        try:
            next(a)
        except StopIteration:
            live.remove(a)
        steps += 1
        assert steps < 400000, "deadlock: no agent finished"
    assert out == [(t, h) for t in tiles_of for h in range(halves)]
    assert all(r is None for r in ring)


@pytest.mark.parametrize("halves", [1, 2], ids=["whole_tile", "two_halves"])
@pytest.mark.parametrize("res", [True, False], ids=["residual", "no_residual"])
@pytest.mark.parametrize("stages", [3, 4, 8])
@pytest.mark.parametrize("tiles,grid,kblocks", [(200, 132, 2), (512, 132, 9), (7, 3, 5), (5, 5, 1), (10, 4, 4), (3, 132, 3), (1536, 132, 1)])
def test_staging_handshakes(tiles, grid, kblocks, stages, res, halves):
    for cta in sorted({0, min(grid, tiles) - 1, (tiles - 1) % grid, tiles % grid}):
        if cta < min(grid, tiles):
            run_cta(cta, min(grid, tiles), tiles, kblocks, stages, res, halves, seed=cta * 7919 + tiles + stages)
