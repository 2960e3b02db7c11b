"""The odometry session (dcreg_odometry_open / _push / _close): scan-to-map odometry fed as the frames arrive.

Every comparison is byte for byte against one icp_run_odometry call over the same frames with the session's settings:
T_out, T_prior, status, iterations, converged, n_points, cov, and every log record with iter_time_ms zeroed.
"""
import numpy as np
import pytest

from harness import RADIUS, ctx, log_bytes, params  # noqa: F401
from odom_harness import CELL, RAGGED, assert_same, odo, one_per_push, pushed, raw_push, split  # noqa: F401

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)


def chunkings(lens):
    return {"all_at_once": [list(lens)], "one_per_push": one_per_push(lens), "ragged": RAGGED}


def one_call(ctx, prm, seqs, T_init, deltas=None, **kw):
    return split(ctx.icp_run_odometry(prm, seqs, T_init, deltas, cell_size=CELL, **kw), seqs)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
@pytest.mark.parametrize("chunking", ["all_at_once", "one_per_push", "ragged"])
def test_chunkings_equal_one_call(ctx, odo, method, chunking):
    """Any chunking, with and without logs and covariances, gives the one call's bytes"""
    seqs, T_init, deltas = odo
    prm = params(method)
    for extra in (dict(), dict(want_log=True, want_cov=True)):
        ref = one_call(ctx, prm, seqs, T_init, deltas, map_frames=3, **extra)
        got = pushed(ctx, prm, seqs, T_init, chunkings(LENS)[chunking], deltas, map_frames=3, **extra)
        assert_same(got, ref)


@pytest.mark.parametrize("map_frames", [1, 3, 100])
def test_constant_velocity_across_pushes(ctx, odo, map_frames):
    """The first push of every sequence ends right after its anchor, so the next frames' previous two results are
    retained frames (with map_frames = 1 the older one is kept as a pose alone)"""
    seqs, T_init, _ = odo
    prm = params()
    chunks = [[1, 1, 1]] + one_per_push([0, 6, 11])
    ref = one_call(ctx, prm, seqs, T_init, None, motion="constant_velocity", map_frames=map_frames, want_log=True)
    got = pushed(ctx, prm, seqs, T_init, chunks, None, motion="constant_velocity", map_frames=map_frames, want_log=True)
    assert_same(got, ref)
    ragged = pushed(ctx, prm, seqs, T_init, RAGGED, None, motion="constant_velocity", map_frames=map_frames)
    assert_same(ragged, one_call(ctx, prm, seqs, T_init, None, motion="constant_velocity", map_frames=map_frames))


@pytest.mark.parametrize("filters", [dict(source_voxel=0.25), dict(map_voxel=0.25),
                                     dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)])
def test_filters(ctx, odo, filters):
    seqs, T_init, deltas = odo
    prm = params()
    ref = one_call(ctx, prm, seqs, T_init, deltas, map_frames=3, want_cov=True, **filters)
    for chunks in (one_per_push(LENS), RAGGED):
        got = pushed(ctx, prm, seqs, T_init, chunks, deltas, map_frames=3, want_cov=True, **filters)
        assert_same(got, ref)
    if "source_voxel" in filters:
        assert all(r.n_points < 20_000 for rs in ref for r in rs)


def test_aborted_frame_enters_later_maps(ctx, odo):
    """A 5-point frame pushed alone mid-session aborts with NOT_ENOUGH_POINTS and enters the later maps at its pose"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    seq = list(seqs[2][:7])
    seq[2] = seq[2][:5]
    prm = params()
    ref = one_call(ctx, prm, [seq], T_init[2:3], deltas[8:15], map_frames=3, want_log=True)
    assert ref[0][2].status == api.NOT_ENOUGH_POINTS
    got = pushed(ctx, prm, [seq], T_init[2:3], [[2], [1], [1], [3]], deltas[8:15], map_frames=3, want_log=True)
    assert_same(got, ref)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_fixed_iterations(ctx, odo, method):
    seqs, T_init, deltas = odo
    prm = params(method, fixed_iterations=1, max_iterations=5)
    ref = one_call(ctx, prm, seqs, T_init, deltas, map_frames=3)
    assert all(r.iterations == 5 for rs in ref for r in rs[1:])
    assert_same(pushed(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, map_frames=3), ref)


def test_other_calls_between_pushes(ctx, odo):
    """Scans, one-shot odometry, set_target + icp_run and voxel_downsample between pushes change nothing, and icp_run
    returns the same bytes before, during and after the session"""
    seqs, T_init, deltas = odo
    prm = params()
    tgt = np.concatenate(seqs[2][:3])
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(seqs[2][1])
    before = ctx.icp_run(prm, T_init[2])
    ref = one_call(ctx, prm, seqs, T_init, deltas, map_frames=3, want_log=True)
    seen = []

    def between(i):
        kind = i % 4
        if kind == 0:
            ctx.icp_run_scans(prm, [seqs[2][1], seqs[2][2]], np.stack([T_init[2]] * 2))
        elif kind == 1:
            ctx.icp_run_odometry(prm, [seqs[1][:3]], T_init[1:2], deltas[1:4], map_frames=2, cell_size=CELL)
        elif kind == 2:
            ctx.set_target(tgt, RADIUS)
            ctx.set_source(seqs[2][1])
            seen.append(ctx.icp_run(prm, T_init[2]))
        else:
            ctx.voxel_downsample([seqs[2][3], seqs[1][2]], 0.3, 2)

    got = pushed(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, map_frames=3, want_log=True, between=between)
    assert_same(got, ref)
    after = ctx.icp_run(prm, T_init[2])
    for r in seen + [after]:
        assert (r.status, r.iterations, r.converged) == (before.status, before.iterations, before.converged)
        assert r.T.tobytes() == before.T.tobytes()
        assert [log_bytes(x) for x in r.logs] == [log_bytes(y) for y in before.logs]


def test_failed_map_push_changes_nothing(ctx, odo):
    """A push whose step map has no dense grid (a point 30 km away in a frame the next frame's map holds) fails naming
    the sequence and its frame since open; the session then continues as if it had never seen that push"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    seq = [f[:6000] for f in seqs[2][:6]]
    far = np.concatenate([seq[2], np.array([[3.0e4, 3.0e4, 0.0]], np.float32)])
    prm = params()
    ref = one_call(ctx, prm, [seq], T_init[2:3], deltas[8:14], map_frames=3, want_log=True, want_cov=True)
    with ctx.odometry_session(prm, 1, T_init[2:3], map_frames=3, cell_size=CELL) as sess:
        got = sess.push([seq[:2]], deltas[8:10], want_log=True, want_cov=True)[0]
        with pytest.raises(api.DcregError) as e:
            sess.push([[far, seq[3]]], deltas[10:12])
        assert e.value.status == api.BAD_ARG
        msg = ctx.lib.dcreg_last_error(ctx._h).decode()
        assert "sequence 0" in msg and "frame 3 of the sequence since open" in msg, msg
        got += sess.push([seq[2:]], deltas[10:14], want_log=True, want_cov=True)[0]
    assert_same([got], ref)


def test_pre_launch_errors_change_nothing(ctx, odo):
    """Bad tables, a frame the source filter leaves empty, constant velocity with deltas, push or close without a session
    and a second open are BAD_ARG; a session that met them continues as if it had not"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    prm = params()
    lib, h = ctx.lib, ctx._h
    short = [s[:4] for s in seqs]
    dl = np.concatenate([deltas[0:1], deltas[1:5], deltas[8:12]])
    ref = one_call(ctx, prm, short, T_init, dl, map_frames=3, source_voxel=0.25, want_log=True)
    assert api._odometry_call(lib, h, "dcreg_odometry_push", n_frames=1, stride=3, log_cap=0) == api.BAD_ARG
    assert "no session" in lib.dcreg_last_error(h).decode()
    assert lib.dcreg_odometry_close(h) == api.BAD_ARG
    nan = np.full((50, 3), np.nan, np.float32)
    with ctx.odometry_session(prm, 3, T_init, map_frames=3, cell_size=CELL, source_voxel=0.25) as sess:
        got = [list(r) for r in sess.push([s[:2] for s in short], np.concatenate([dl[0:1], dl[1:3], dl[5:7]]),
                                          want_log=True)]
        f = [short[1][2], short[2][2]]
        launches = ctx.launch_count
        bad = [raw_push(ctx, [0, 1, 0, 2], f),                                      # a decreasing table
               raw_push(ctx, [0, 0, 1, 1], f, n=2),                                 # does not end at n_frames
               raw_push(ctx, [0, 0, 1, 2], f, offsets=[0, 10, 10]),                 # an empty frame
               raw_push(ctx, [0, 0, 1, 2], f, stride=2)]
        assert all(rc == api.BAD_ARG for rc in bad), bad
        assert ctx.launch_count == launches                                         # nothing launched
        with pytest.raises(api.DcregError):                                         # the filter leaves nothing
            sess.push([[], [nan], []])
        assert "frame 2 of the sequence since open" in lib.dcreg_last_error(h).decode()
        with pytest.raises(api.DcregError):                                         # a second session
            ctx.odometry_session(prm, 3, T_init, cell_size=CELL)
        for s, r in enumerate(sess.push([s[2:] for s in short], np.concatenate([dl[3:5], dl[7:9]]), want_log=True)):
            got[s] += r
    assert_same(got, ref)
    with ctx.odometry_session(prm, 1, T_init[:1], motion="constant_velocity", cell_size=CELL):
        assert raw_push(ctx, [0, 1], [short[1][0]], deltas=deltas[:1]) == api.BAD_ARG
        assert "no deltas" in lib.dcreg_last_error(h).decode()


def test_sharded_context_has_no_session(odo):
    from dcreg_b200 import api, Context
    _, T_init, _ = odo
    with Context(0) as fresh:
        try:
            fresh.comm_init(fresh.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        with pytest.raises(api.DcregError):
            fresh.odometry_session(params(), 1, T_init[:1], cell_size=CELL)
        assert "rank" in fresh.lib.dcreg_last_error(fresh._h).decode()


def test_launches_per_push_are_steady(ctx, odo):
    """Once the window is full, every push of one frame per sequence launches the same number of kernels, however many
    frames the session has seen (fixed iterations: every frame runs the same loop)"""
    seqs, T_init, deltas = odo
    prm = params(fixed_iterations=1, max_iterations=4)
    two = [seqs[1], seqs[2][:7]]
    counts = []
    with ctx.odometry_session(prm, 2, T_init[1:], map_frames=3, cell_size=CELL, map_voxel=0.25) as sess:
        for k in range(7):
            before = ctx.launch_count
            sess.push([[s[k]] for s in two])
            counts.append(ctx.launch_count - before)
    assert len(set(counts[3:])) == 1, counts
