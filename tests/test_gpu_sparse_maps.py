"""dcreg_set_sparse_maps: sparse row indexes for odometry's local maps and icp_run_pairs' targets too large for dense
grids.

With the setting on, a step or call that fits dense grids runs exactly as with it off (bytes and launches).  A step
whose maps are past the limits builds sparse indexes, whose searches give the dense grid's results bit for bit: a far
point that sorts after every other point changes nothing but the counts that include it, and every frame equals its own
single run on dcreg_set_target_sparse to the rounding of FP64 sums grouped differently.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o
from harness import ctx, log_bytes, params  # noqa: F401

pytestmark = pytest.mark.gpu

CELL = 0.5
FAR_CELL = 0.25          # the long-range scene's cell: rings = 2


@pytest.fixture(scope="module")
def odo():
    """12 frames (about 6 k points each) of one path with drifting odometry, as sequences of 5 and 7 frames"""
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(12, seed=71, n_scan=6_000, max_range=20.0)
    return [frames[:5], frames[5:]], T_true[[0, 5]], deltas


@pytest.fixture(scope="module")
def long_range():
    """2 x 8 frames of the long-range scene (sparse facades at 150 - 200 m, 20 m tall)"""
    from dcreg_b200.scenes import make_long_range_sequence
    frames, T_true, deltas = make_long_range_sequence(16, seed=81, n_scan=4_000, n_far=1_500)
    return [frames[:8], frames[8:]], T_true[[0, 8]], deltas


def assert_same(a, b, skip_counts=()):
    """a, b: flat lists of IcpResult; frames in skip_counts may differ in n_points and in their logs' fitness"""
    assert len(a) == len(b)
    for k, (x, y) in enumerate(zip(a, b)):
        assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged), k
        if k not in skip_counts:
            assert getattr(x, "n_points", None) == getattr(y, "n_points", None), k
        assert x.T.tobytes() == y.T.tobytes(), k
        assert x.T_prior.tobytes() == y.T_prior.tobytes(), k
        assert (x.cov is None) == (y.cov is None), k
        if x.cov is not None:
            assert x.cov.tobytes() == y.cov.tobytes(), k
        assert len(x.logs) == len(y.logs), k
        f = k not in skip_counts
        assert [log_bytes(r, f) for r in x.logs] == [log_bytes(r, f) for r in y.logs], k


def with_setting(ctx, enable, fn):
    """fn() with the setting at `enable`, and the launches it took"""
    ctx.set_sparse_maps(enable)
    try:
        n0 = ctx.launch_count
        out = fn()
        return out, ctx.launch_count - n0
    finally:
        ctx.set_sparse_maps(False)


def flat(seqs):
    return [r for s in seqs for r in s]


def assert_single_sparse(ctx, prm, frame, map_pts, b, cell):
    """frame's result b against set_target_sparse(map) + set_source(frame) + icp_run(b.T_prior)"""
    ctx.set_target_sparse(map_pts, cell)
    ctx.set_source(frame)
    single = ctx.icp_run(prm, b.T_prior)
    assert (b.status, b.iterations, b.converged) == (single.status, single.iterations, single.converged)
    assert o.se3_log_distance(single.T, b.T) < 1e-8
    assert len(b.logs) == len(single.logs)
    for x, y in zip(b.logs, single.logs):
        assert (x.n_corr_pt, x.n_effective, x.status) == (y.n_corr_pt, y.n_effective, y.status)
        assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)


def window_maps(seq, res, map_frames):
    from dcreg_b200.api import map_points
    return [None] + [np.concatenate([map_points(res[j].T, seq[j]) for j in range(max(0, k - map_frames), k)])
                     for k in range(1, len(seq))]


def box_cells(pts, cell):
    c = np.floor(np.asarray(pts, dtype=np.float64) * (1.0 / cell))
    return int(np.prod(c.max(0) - c.min(0) + 1))


# ---- 1. the setting on, nothing past the limits: the same bytes and launches ----------------------------------------

def test_under_limit_unchanged(ctx, odo):
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    prm = params()
    runs = {
        "window": lambda: flat([ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL,
                                                     want_log=True, want_cov=True)]),
        "voxel_map": lambda: ctx.icp_run_odometry_map(prm, seqs, T_init, deltas, map_voxel=0.25, max_distance=30.0,
                                                      map_max_points=4, cell_size=CELL, want_log=True, want_cov=True),
        "adaptive": lambda: ctx.icp_run_odometry(prm, seqs, T_init, None, motion="constant_velocity", map_frames=4,
                                                 cell_size=CELL, want_log=True, adaptive=api.AdaptiveThreshold()),
    }
    for name, fn in runs.items():
        off, n_off = with_setting(ctx, False, fn)
        on, n_on = with_setting(ctx, True, fn)
        assert n_on == n_off, name
        assert_same(off, on)

    def session():
        from dcreg_b200.scenes import make_parking_sweeps
        fr, ts, Tt, dl, _ = make_parking_sweeps(6, seed=73, n_scan=3_000)
        out = []
        for chunks in ((3, 3), (1, 5)):
            with ctx.odometry_session(prm, 1, Tt[:1], map_frames=3, cell_size=CELL) as s:
                at, res = 0, []
                for c in chunks:
                    res += s.push([fr[at:at + c]], dl[at:at + c], want_log=True, timestamps=[ts[at:at + c]])[0]
                    at += c
            out.append(res)
        assert_same(out[0], out[1])
        return out[0]
    off, n_off = with_setting(ctx, False, session)
    on, n_on = with_setting(ctx, True, session)
    assert n_on == n_off
    assert_same(off, on)

    def pairs():
        src = [f for s in seqs for f in s][1:7]
        tgt = [f for s in seqs for f in s][0:6]
        return ctx.icp_run_pairs(prm, src, tgt, np.tile(np.eye(4), (6, 1, 1)), want_log=True, metrics_threshold=0.5)
    off, n_off = with_setting(ctx, False, pairs)
    on, n_on = with_setting(ctx, True, pairs)
    assert n_on == n_off
    for x, y in zip(off, on):
        assert (x.status, x.iterations, x.converged, x.T.tobytes()) == (y.status, y.iterations, y.converged, y.T.tobytes())
        assert [log_bytes(r) for r in x.logs] == [log_bytes(r) for r in y.logs]
        assert x.metrics == y.metrics


# ---- 2. window odometry with a far point -----------------------------------------------------------------------------

def far_recording(odo):
    """5 frames; frame 2 carries a point 30 km away, above every other point (it sorts last in every order).  The
    frames without it have 3000 points, frame 2 2999 of its own, so the call's largest frame stays the same."""
    seqs, T_init, deltas = odo
    seq = [f[:3000] for f in seqs[0][:5]]
    plain = list(seq)
    plain[2] = seq[2][:2999]
    far = list(plain)
    far[2] = np.concatenate([plain[2], np.array([[3.0e4, 3.0e4, 50.0]], np.float32)])
    return plain, far, T_init[:1], deltas[:5]


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_far_point_window(ctx, odo, method):
    from dcreg_b200 import api
    plain, far, T0, D = far_recording(odo)
    prm = params(method)
    with pytest.raises(api.DcregError):                    # off: refused at frame 3's step, as before
        ctx.icp_run_odometry(prm, [far], T0, D, map_frames=3, cell_size=CELL)
    dense = ctx.icp_run_odometry(prm, [plain], T0, D, map_frames=3, cell_size=CELL, want_log=True, want_cov=True)
    sparse, _ = with_setting(ctx, True, lambda: ctx.icp_run_odometry(
        prm, [far], T0, D, map_frames=3, cell_size=CELL, want_log=True, want_cov=True))
    maps = window_maps(far, sparse, 3)
    assert all(box_cells(maps[k], CELL) > 2 ** 27 for k in (3, 4))      # frames 3 and 4 ran on sparse indexes
    assert sparse[2].n_points == dense[2].n_points + 1
    assert_same(dense, sparse, skip_counts={2})
    again, _ = with_setting(ctx, True, lambda: ctx.icp_run_odometry(
        prm, [far], T0, D, map_frames=3, cell_size=CELL, want_log=True, want_cov=True))
    assert_same(sparse, again)
    for k in range(1, 5):
        assert_single_sparse(ctx, prm, far[k], maps[k], sparse[k], CELL)


# ---- 3. the long-range scene: window and unpruned voxel map ---------------------------------------------------------

def test_long_range_window(ctx, long_range):
    seqs, T_init, deltas = long_range
    prm = params()
    run = lambda: ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=10, cell_size=FAR_CELL, want_log=True)
    res, _ = with_setting(ctx, True, run)
    again, _ = with_setting(ctx, True, run)
    assert_same(res, again)
    at = 0
    for seq in seqs:
        r = res[at:at + len(seq)]
        maps = window_maps(seq, r, 10)
        assert all(box_cells(maps[k], FAR_CELL) > 2 ** 27 for k in range(2, len(seq)))
        for k in range(1, len(seq)):
            assert_single_sparse(ctx, prm, seq[k], maps[k], r[k], FAR_CELL)
        at += len(seq)
    # a session in three chunkings gives the one call's bytes
    for chunks in ((8,), (3, 3, 2), (1, 4, 3)):
        ctx.set_sparse_maps(True)
        with ctx.odometry_session(prm, 2, T_init, map_frames=10, cell_size=FAR_CELL) as s:
            ctx.set_sparse_maps(False)                  # captured at open
            got, a = [[], []], 0
            for c in chunks:
                out = s.push([seqs[0][a:a + c], seqs[1][a:a + c]],
                             np.concatenate([deltas[a:a + c], deltas[8 + a:8 + a + c]]), want_log=True)
                got[0] += out[0]; got[1] += out[1]
                a += c
        assert_same(res, got[0] + got[1])


def test_long_range_voxel_map(ctx, long_range):
    from dcreg_b200 import api
    seqs, T_init, deltas = long_range
    prm = params()
    kw = dict(map_voxel=0.25, max_distance=float("inf"), map_max_points=4, cell_size=FAR_CELL, want_log=True)
    run = lambda: ctx.icp_run_odometry_map(prm, seqs, T_init, deltas, **kw)
    res, _ = with_setting(ctx, True, run)
    again, _ = with_setting(ctx, True, run)
    assert_same(res, again)
    at = 0
    for s, seq in enumerate(seqs):
        r = res[at:at + len(seq)]
        M = api.voxel_map_update(np.zeros((0, 3), np.float32), seq[0], T_init[s], 0.25, 4, float("inf"))
        for k in range(1, len(seq)):
            if k >= 2:
                assert box_cells(M, FAR_CELL) > 2 ** 27
            assert_single_sparse(ctx, prm, seq[k], M, r[k], FAR_CELL)
            M = api.voxel_map_update(M, seq[k], r[k].T, 0.25, 4, float("inf"))
        at += len(seq)
    for chunks in ((2, 6), (3, 3, 2)):
        ctx.set_sparse_maps(True)
        sess = ctx.odometry_map_session(prm, 2, T_init, map_voxel=0.25, max_distance=float("inf"), map_max_points=4,
                                        cell_size=FAR_CELL)
        ctx.set_sparse_maps(False)
        with sess as s:
            got, a = [[], []], 0
            for c in chunks:
                out = s.push([seqs[0][a:a + c], seqs[1][a:a + c]],
                             np.concatenate([deltas[a:a + c], deltas[8 + a:8 + a + c]]), want_log=True)
                got[0] += out[0]; got[1] += out[1]
                a += c
        assert_same(res, got[0] + got[1])


# ---- 4. sessions: the setting at open; a failing sparse push commits nothing ----------------------------------------

def test_session_captures_setting_and_failed_push(ctx, odo):
    from dcreg_b200 import api
    plain, far, T0, D = far_recording(odo)
    prm = params()
    with ctx.odometry_session(prm, 1, T0, map_frames=3, cell_size=CELL) as s:      # opened with the setting off
        ctx.set_sparse_maps(True)
        try:
            with pytest.raises(api.DcregError):
                s.push([far], D)
        finally:
            ctx.set_sparse_maps(False)
    one, _ = with_setting(ctx, True, lambda: ctx.icp_run_odometry(prm, [far], T0, D, map_frames=3, cell_size=CELL))
    ctx.set_sparse_maps(True)
    s = ctx.odometry_session(prm, 1, T0, map_frames=3, cell_size=CELL)
    ctx.set_sparse_maps(False)
    with s:
        first = s.push([far[:3]], D[:3])[0]
        # a sparse step that fails for another reason: a map coordinate beyond +-2^19 cells
        bad = far[3].copy()
        bad[0] = (1.0e6, 0.0, 0.0)
        with pytest.raises(api.DcregError) as e:
            s.push([[bad, far[4]]], D[3:5])
        assert "2^19" in str(e.value) or "2^19" in ctx.lib.dcreg_last_error(ctx._h).decode()
        rest = s.push([far[3:]], D[3:])[0]                 # nothing was committed: the retry continues the recording
    assert_same(one, first + rest)


# ---- 5. pairs --------------------------------------------------------------------------------------------------------

def test_pairs_far_target(ctx, cylinder, odo):
    from dcreg_b200 import api
    from dcreg_b200.scenes import g2_initial_pose
    prm = params()
    far = np.ascontiguousarray(np.concatenate([cylinder, cylinder + np.float32(4.0e4)]))
    T0 = g2_initial_pose()
    ctx.set_sparse_maps(True)
    try:
        got = ctx.icp_run_pairs(prm, [cylinder], [far], T0[None], want_log=True, cell_size=1.0)[0]
        frames = [f for s in odo[0] for f in s]
        src, tgt = [cylinder, frames[1], frames[3]], [far, frames[0], frames[2]]
        Ts = np.stack([T0, np.eye(4), np.eye(4)])
        mixed = ctx.icp_run_pairs(prm, src, tgt, Ts, want_log=True, cell_size=1.0)
        again = ctx.icp_run_pairs(prm, src, tgt, Ts, want_log=True, cell_size=1.0)
        for x, y in zip(mixed, again):
            assert (x.status, x.iterations, x.T.tobytes()) == (y.status, y.iterations, y.T.tobytes())
            assert [log_bytes(r) for r in x.logs] == [log_bytes(r) for r in y.logs]
        # metrics on a sparse pair: BAD_ARG after the poses, naming the pair
        with pytest.raises(api.DcregError) as e:
            ctx.icp_run_pairs(prm, src[1:] + src[:1], tgt[1:] + tgt[:1], np.stack([Ts[1], Ts[2], Ts[0]]), cell_size=1.0,
                              metrics_threshold=0.5)
        assert "pair 2" in str(e.value)
    finally:
        ctx.set_sparse_maps(False)
    for b, (s, t, T) in zip(mixed, zip(src, tgt, Ts)):
        ctx.set_target_sparse(t, 1.0)
        ctx.set_source(s)
        single = ctx.icp_run(prm, T)
        assert (b.status, b.iterations, b.converged) == (single.status, single.iterations, single.converged)
        assert o.se3_log_distance(single.T, b.T) < 1e-8
        for x, y in zip(b.logs, single.logs):
            assert (x.n_corr_pt, x.n_effective) == (y.n_corr_pt, y.n_effective)
    assert mixed[0].T.tobytes() == got.T.tobytes() or o.se3_log_distance(mixed[0].T, got.T) < 1e-8


# ---- 6. errors still refused with the setting on ---------------------------------------------------------------------

def test_errors_still_refused(ctx, cylinder, odo):
    from dcreg_b200 import api
    prm = params()
    ctx.set_sparse_maps(True)
    try:
        with pytest.raises(api.DcregError) as e:
            ctx.icp_run_pairs(prm, [cylinder, cylinder], [cylinder, cylinder + np.float32(1.0e6)],
                              np.tile(np.eye(4), (2, 1, 1)), cell_size=1.0)
        assert "2^19" in str(e.value) and "target 1" in str(e.value)
        plain, far, T0, D = far_recording(odo)
        bad = list(plain)
        bad[2] = np.concatenate([plain[2], np.array([[1.0e6, 0.0, 0.0]], np.float32)])
        with pytest.raises(api.DcregError) as e:
            ctx.icp_run_odometry(prm, [bad], T0, D, map_frames=3, cell_size=CELL)
        assert "2^19" in str(e.value) and "frame 3" in str(e.value)
        assert ctx.icp_run_odometry(prm, [plain], T0, D, map_frames=3, cell_size=CELL)[4].status == api.OK
    finally:
        ctx.set_sparse_maps(False)
    assert ctx.lib.dcreg_set_sparse_maps(ctx._h, 2) == api.BAD_ARG
