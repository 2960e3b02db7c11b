"""CPU model of the loop kernel's row flags and launch counter (solver block: dcreg_b200.cu solver_block,
k1_stream.cuh publish_row / stream_rows_to_fin), run under adversarial interleavings.

The device code cannot run here, so the protocol is restated step by step and a random scheduler interleaves the
blocks' atomic steps:

  every block of a launch (after the previous launch completed) reads epoch E of the context
  tile block b:   writes its row, then stores flag[b] = E + 1 (release)
  solver warp w:  one poll round = acquire-load the flags of its next 32 rows (w + 8 k), take the ready prefix, add
                  those rows in order; when every row of the warp is in, the warp is done
  solver block:   once all warps are done, adds the 8 warp sums in order and stores epoch = E + 1
  a launch whose trial is done: every block returns at once (no row, no flag, no epoch change)

Checked: the result is bit-identical to the ticket path's flat order (k1s::reduce_to_fin) whatever the arrival order,
a row is never taken before its block published it in this launch (stale flags of earlier launches and runs, with
other grid sizes, are never accepted), and launches of a finished trial leave no skew between the counter and the
flags.  A model that polls for "flag != 0" instead of "flag == epoch + 1" does take stale rows under the same
schedules, and a different summation order does change the bits (so the test can see the failures it guards against).
"""
import random

import numpy as np
import pytest

WARPS = 8


def flat_order(rows):
    """k1s::reduce_to_fin: warp w adds rows w, w + 8, ... in order, then the 8 warp sums are added in order."""
    fin = np.zeros(rows.shape[1])
    for w in range(WARPS):
        s = np.zeros(rows.shape[1])
        for b in range(w, len(rows), WARPS):
            s = s + rows[b]
        fin = fin + s
    return fin


class Ctx:
    """Per-context device memory: the launch counter, the row flags (never reset) and the row buffer."""

    def __init__(self, cap, cols):
        self.epoch = 0
        self.flags = [0] * cap
        self.partials = np.full((cap, cols), np.nan)


def launch(ctx, rows, rng, done=False, accept_any=False):
    """One launch of the iteration kernel with len(rows) tile blocks.  Returns the solver's sum (None if done)."""
    if done:
        return None
    n = len(rows)
    want = ctx.epoch + 1                                  # every block reads the counter after pdl_wait
    published = set()
    pending = list(range(n))
    rng.shuffle(pending)
    k = [0] * WARPS                                       # next index j of warp w's sequence (row w + 8 j)
    sums = [np.zeros(rows.shape[1]) for _ in range(WARPS)]
    taken = []

    def warp_done(w):
        return w + WARPS * k[w] >= n

    while not all(warp_done(w) for w in range(WARPS)):
        movers = [("tile", b) for b in pending[:3]] + [("warp", w) for w in range(WARPS) if not warp_done(w)]
        kind, x = rng.choice(movers)
        if kind == "tile":
            pending.remove(x)
            ctx.partials[x] = rows[x]
            ctx.flags[x] = want
            published.add(x)
            continue
        w = x
        ready = []
        for lane in range(32):                            # one acquire load per lane, then the ballot
            r = w + WARPS * (k[w] + lane)
            ready.append(r >= n or (ctx.flags[r] != 0 if accept_any else ctx.flags[r] == want))
        prefix = ready.index(False) if False in ready else 32
        for j in range(prefix):
            r = w + WARPS * (k[w] + j)
            if r < n:
                taken.append((r, r in published))
                sums[w] = sums[w] + ctx.partials[r]
        k[w] += prefix
    fin = np.zeros(rows.shape[1])
    for w in range(WARPS):
        fin = fin + sums[w]
    ctx.epoch = want
    for b in pending:                                     # (a model that accepted a stale flag finished early)
        ctx.partials[b] = rows[b]
        ctx.flags[b] = want
    launch.stale = any(not fresh for _, fresh in taken)
    return fin


def wide_rows(rng, n, cols=32):
    """Rows whose sum depends on the order of the additions (magnitudes over 30 decades)."""
    return rng.standard_normal((n, cols)) * 10.0 ** rng.uniform(-15, 15, (n, cols))


@pytest.mark.parametrize("seed", range(40))
def test_streamed_sum_is_bit_identical_to_the_flat_order(seed):
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    sizes = [391, 237, 1, 9, 395, 391]                  # C2, the shipped cloud, tiny and ragged grids, C4
    ctx = Ctx(max(sizes), 32)
    for n in sizes:
        rows = wide_rows(nrng, n)
        fin = launch(ctx, rows, rng)
        assert not launch.stale
        assert fin.tobytes() == flat_order(rows).tobytes()


def test_the_order_matters_for_these_rows():
    nrng = np.random.default_rng(0)
    rows = wide_rows(nrng, 391)
    assert flat_order(rows).tobytes() != rows.sum(axis=0).tobytes()
    assert flat_order(rows).tobytes() != flat_order(rows[::-1]).tobytes()


@pytest.mark.parametrize("seed", range(20))
def test_stale_flags_of_earlier_launches_and_runs_are_never_accepted(seed):
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    ctx = Ctx(400, 32)
    # earlier runs with larger and smaller grids leave flags behind, with rows that must never be summed again
    for n in (395, 100, 391, 17, 391, 391):
        rows = wide_rows(nrng, n)
        fin = launch(ctx, rows, rng)
        assert not launch.stale
        assert fin.tobytes() == flat_order(rows).tobytes()
        assert all(f <= ctx.epoch for f in ctx.flags)  # no flag can match the next launch before it is written


@pytest.mark.parametrize("seed", range(20))
def test_a_flag_without_epoch_would_take_stale_rows(seed):
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    ctx = Ctx(400, 32)
    launch(ctx, wide_rows(nrng, 391), rng, accept_any=True)
    stale = False
    for _ in range(5):
        launch(ctx, wide_rows(nrng, 391), rng, accept_any=True)
        stale |= launch.stale
    assert stale


@pytest.mark.parametrize("seed", range(10))
def test_a_trial_that_finishes_early_leaves_no_epoch_skew(seed):
    rng = random.Random(seed)
    nrng = np.random.default_rng(seed)
    ctx = Ctx(400, 32)
    summed = 0
    # runs of a few iterations each; bodies past the end of a run (done) exit at once, as do whole chunks
    for run in range(6):
        iters = rng.randint(1, 5)
        for body in range(8):
            done = body >= iters
            rows = wide_rows(nrng, 391)
            fin = launch(ctx, rows, rng, done=done)
            if done:
                assert fin is None
            else:
                summed += 1
                assert not launch.stale
                assert fin.tobytes() == flat_order(rows).tobytes()
            assert ctx.epoch == summed                    # the counter moves exactly once per launch that summed
            assert max(ctx.flags) == ctx.epoch            # and every flag is at most the last launch's value
