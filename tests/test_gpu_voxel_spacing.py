"""The minimum point spacing on the device: dcreg_voxel_downsample_spaced against its NumPy twin, and
dcreg_set_map_spacing, which gives scan-to-map odometry's window and voxel maps KISS-ICP's AddPoints spacing.

Every registered frame of a spaced call is checked against its reconstruction with the twin: its map is
voxel_downsample(window, map_voxel, map_max_points, s) for the window, and the chain of voxel_map_update(..., s) for the
voxel map."""
import contextlib
import math

import numpy as np
import pytest

from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, RAGGED, assert_anchor, assert_priors, assert_same, assert_same_flat,  # noqa: F401
                          crowded_clouds, map_call, odo, one_per_push, pushed, raw_downsample, raw_odometry,
                          seq_results, source_points, split, sweeps, twin_maps, window_call, window_map)

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)
SV, MV = 0.3, 0.25            # source and map voxel sizes
DIST = 10.0                   # the voxel map's prune distance
CAP = 4
S = MV / math.sqrt(CAP)          # KISS-ICP's spacing for the map filter of the tests
SPACED = "dcreg_voxel_downsample_spaced"
MAP = "dcreg_icp_run_odometry_map"
RAW_MAP = dict(source_voxel=SV, map_voxel=MV, source_max_points=1, map_max_points=4, max_distance=DIST)


@contextlib.contextmanager
def spacing(ctx, s):
    ctx.set_map_spacing(s)
    try:
        yield
    finally:
        ctx.set_map_spacing(0.0)


def assert_equals_twin(pts, kept, idx, clouds, voxel, max_points, s):
    from dcreg_b200.api import voxel_downsample
    at = 0
    for b, c in enumerate(clouds):
        tp, ti = voxel_downsample(c, voxel, max_points, s)
        assert kept[b] == at, b
        at += len(ti)
        assert pts[kept[b]:kept[b + 1]].tobytes() == tp.tobytes() and np.array_equal(idx[kept[b]:kept[b + 1]], ti), b
    assert kept[-1] == at


@pytest.fixture(scope="module")
def raw_frames():
    """Four unfiltered frames of about 50 k points: 0.5 m voxels then hold up to about 1 500 points"""
    from dcreg_b200.scenes import make_parking_sequence
    frames = make_parking_sequence(4, seed=47, n_scan=50_000, max_range=20.0)[0]
    return list(frames)


@pytest.mark.parametrize("max_points", [2, 4, 20])
@pytest.mark.parametrize("voxel", [0.25, 1.0])
def test_spaced_downsample_equals_twin(ctx, voxel, max_points):
    clouds = crowded_clouds()
    rng = np.random.default_rng(41)
    c4 = [np.concatenate([c, rng.uniform(0, 1, (len(c), 1)).astype(np.float32)], axis=1) for c in clouds]
    for s in (voxel / math.sqrt(max_points), 0.2 * voxel, 0.01 * voxel):
        for stride in (3, 4):
            rc, pts, kept, idx = raw_downsample(ctx, SPACED, c4, voxel, stride=stride, max_points=max_points,
                                                min_spacing=s)
            assert rc == 0
            assert_equals_twin(pts, kept, idx, clouds, voxel, max_points, s)
        got = ctx.voxel_downsample(clouds, voxel, max_points, s)
        assert [p.tobytes() for p, _ in got] == [pts[a:b].tobytes() for a, b in zip(kept[:-1], kept[1:])]
    rc, pts2, kept2, _ = raw_downsample(ctx, SPACED, c4, voxel, stride=4, want_index=False, max_points=max_points,
                                        min_spacing=S)
    rc3, pts3, kept3, _ = raw_downsample(ctx, SPACED, c4, voxel, stride=4, max_points=max_points, min_spacing=S)
    assert rc == rc3 == 0 and np.array_equal(kept2, kept3) and pts2[:kept3[-1]].tobytes() == pts3[:kept3[-1]].tobytes()


@pytest.mark.parametrize("max_points", [4, 20, 1 << 20])
def test_crowded_voxel_and_raw_frames(ctx, raw_frames, max_points):
    """One voxel of 6000 points, and unfiltered 50 k-point frames at 0.5 m (runs of up to about 1 500 points)"""
    from dcreg_b200.api import voxel_downsample
    clouds = crowded_clouds()[-1:]
    for s in (0.25 / math.sqrt(min(max_points, 20)), 0.004):
        rc, pts, kept, idx = raw_downsample(ctx, SPACED, clouds, 0.25, max_points=max_points, min_spacing=s)
        assert rc == 0
        assert_equals_twin(pts, kept, idx, clouds, 0.25, max_points, s)
    for voxel in (0.5, 0.25):
        s = voxel / math.sqrt(min(max_points, 20))
        rc, pts, kept, idx = raw_downsample(ctx, SPACED, raw_frames, voxel, max_points=max_points, min_spacing=s)
        assert rc == 0
        assert_equals_twin(pts, kept, idx, raw_frames, voxel, max_points, s)
        assert kept[-1] < sum(len(voxel_downsample(f, voxel, max_points)[1]) for f in raw_frames)


def test_zero_spacing_and_one_point_caps_are_the_n_call(ctx, raw_frames):
    clouds = crowded_clouds() + raw_frames[:1]
    for voxel, cap, s in ((0.25, 4, 0.0), (0.5, 20, 0.0), (0.25, 1, 0.1), (0.5, 1, 10.0)):
        a0 = ctx.launch_count
        a = raw_downsample(ctx, "dcreg_voxel_downsample_n", clouds, voxel, max_points=cap)
        a1 = ctx.launch_count
        b = raw_downsample(ctx, SPACED, clouds, voxel, max_points=cap, min_spacing=s)
        assert ctx.launch_count - a1 == a1 - a0
        assert a[0] == b[0] == 0
        kept = a[2]
        assert kept.tobytes() == b[2].tobytes()
        for x, y in ((a[1], b[1]), (a[3], b[3])):
            assert x[:kept[-1]].tobytes() == y[:kept[-1]].tobytes()


def test_spaced_launches_do_not_grow_with_clouds(ctx):
    clouds = crowded_clouds()
    a = ctx.launch_count
    ctx.voxel_downsample(clouds[:1], 0.5, 4, 0.25)
    b = ctx.launch_count
    ctx.voxel_downsample(clouds * 8, 0.5, 4, 0.25)
    c = ctx.launch_count
    ctx.voxel_downsample(clouds * 8, 0.5, 4)
    assert ctx.launch_count - c == c - b == b - a == 7


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_window_frames_equal_their_reconstruction(ctx, odo, method, motion):
    from dcreg_b200.api import voxel_downsample
    seqs, T_init, deltas = odo
    prm = params(method)
    D = deltas if motion == "increments" else None
    with spacing(ctx, S):
        res = ctx.icp_run_odometry(prm, seqs, T_init, D, motion=motion, map_frames=3, cell_size=CELL, want_log=True,
                                   want_cov=True, source_voxel=SV, map_voxel=MV, map_max_points=CAP)
    plain = ctx.icp_run_odometry(prm, seqs, T_init, D, motion=motion, map_frames=3, cell_size=CELL, source_voxel=SV,
                                 map_voxel=MV, map_max_points=CAP)
    assert any(a.T.tobytes() != b.T.tobytes() for a, b in zip(res, plain))      # the spacing changes the maps
    if D is not None:
        assert_priors(res, seqs, T_init, D)
    thinner = 0
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        for k in range(1, len(seq)):
            M = window_map(seq, rs, k, 3, SV, MV, (1, CAP), S)
            thinner += len(window_map(seq, rs, k, 3, SV, MV, (1, CAP), 0.0)) - len(M)
            ctx.set_target(M, CELL)
            ctx.set_source(source_points(seq[k], SV))
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))
    assert thinner > 0


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_voxel_map_frames_equal_their_reconstruction(ctx, odo, method, motion):
    from dcreg_b200.api import voxel_downsample
    seqs, T_init, deltas = odo
    prm = params(method)
    D = deltas if motion == "increments" else None
    with spacing(ctx, S):
        res = map_call(ctx, prm, seqs, T_init, D, DIST, motion=motion, source_voxel=SV, map_voxel=MV,
                       map_max_points=CAP)
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        twin = twin_maps(seq, rs, SV, MV, CAP, DIST, S)
        for k in range(1, len(seq)):
            ctx.set_target(twin[k], CELL)
            ctx.set_source(source_points(seq[k], SV))
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_deskewed_frames_with_spacing(ctx, sweeps, method):
    """With timestamps: the window and the voxel map, each frame against its twin map of deskewed kept points"""
    from dcreg_b200.api import map_points, voxel_downsample
    sw = sweeps
    prm = params(method)
    kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=CAP, timestamps=sw["stamps"], want_deskewed=True)
    with spacing(ctx, S):
        res_w = ctx.icp_run_odometry(prm, sw["skewed"], sw["T_init"], sw["deltas"], map_frames=3, cell_size=CELL,
                                     want_log=True, want_cov=True, **kw)
        res_m = map_call(ctx, prm, sw["skewed"], sw["T_init"], sw["deltas"], DIST, **kw)
    for seq, rw, rm in zip(sw["skewed"], split(res_w, sw["skewed"]), split(res_m, sw["skewed"])):
        twin = twin_maps(seq, rm, SV, MV, CAP, DIST, S, frames=[r.deskewed for r in rm])
        for k in range(1, len(seq)):
            M = np.concatenate([map_points(rw[j].T, rw[j].deskewed) for j in range(max(0, k - 3), k)])
            ctx.set_target(voxel_downsample(M, MV, CAP, S)[0], CELL)
            ctx.set_source(rw[k].deskewed)
            assert_same_run(rw[k], ctx.icp_run(prm, rw[k].T_prior))
            ctx.set_target(twin[k], CELL)
            ctx.set_source(rm[k].deskewed)
            assert_same_run(rm[k], ctx.icp_run(prm, rm[k].T_prior))


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
def test_infinite_distance_is_the_long_window(ctx, odo, sweeps, motion):
    seqs, T_init, deltas = odo
    prm = params()
    D = deltas if motion == "increments" else None
    kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=CAP, motion=motion)
    with spacing(ctx, S):
        assert_same_flat(map_call(ctx, prm, seqs, T_init, D, math.inf, **kw), window_call(ctx, prm, seqs, T_init, D, **kw))
        sw = sweeps
        D = sw["deltas"] if motion == "increments" else None
        kw.update(timestamps=sw["stamps"], want_deskewed=True)
        assert_same_flat(map_call(ctx, prm, sw["skewed"], sw["T_init"], D, math.inf, **kw),
                         window_call(ctx, prm, sw["skewed"], sw["T_init"], D, **kw))


def test_local_map_equals_twin_after_every_push(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    with spacing(ctx, S):
        maps = []
        res = pushed(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, voxel_map=True, maps=maps, want_log=True,
                     want_cov=True, source_voxel=SV, map_voxel=MV, map_max_points=CAP, max_distance=DIST)
    for s, (seq, rs) in enumerate(zip(seqs, res)):
        twin = twin_maps(seq, rs, SV, MV, CAP, DIST, S)
        for i in range(len(maps)):
            assert maps[i][s].tobytes() == twin[min(i + 1, len(seq))].tobytes(), (s, i)


CHUNKS = {"one_per_push": one_per_push(LENS), "ragged": RAGGED, "all_at_once": [list(LENS)]}


@pytest.mark.parametrize("chunking", sorted(CHUNKS))
def test_session_chunkings_equal_one_call(ctx, odo, chunking):
    """Sessions record the spacing at open: a change between pushes does not reach them"""
    seqs, T_init, deltas = odo
    prm = params()
    kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=CAP)
    with spacing(ctx, S):
        ref = map_call(ctx, prm, seqs, T_init, deltas, DIST, **kw)
        wref = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True,
                                    want_cov=True, **kw)
        toggle = lambda i: ctx.set_map_spacing([0.0, 0.3, S][i % 3])           # noqa: E731
        maps = []
        got = pushed(ctx, prm, seqs, T_init, CHUNKS[chunking], deltas, voxel_map=True, maps=maps, between=toggle,
                     want_log=True, want_cov=True, max_distance=DIST, **kw)
        ctx.set_map_spacing(S)
        assert_same(got, seq_results(ref, seqs))
        for s, (seq, rs) in enumerate(zip(seqs, got)):
            assert maps[-1][s].tobytes() == twin_maps(seq, rs, SV, MV, CAP, DIST, S)[-1].tobytes()
        # the window session too
        out = pushed(ctx, prm, seqs, T_init, CHUNKS[chunking], deltas, between=toggle, want_log=True, want_cov=True,
                     map_frames=3, **kw)
        ctx.set_map_spacing(S)
        assert_same(out, seq_results(wref, seqs))


def test_reproducible_and_context_intact(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    frames = [f for s in seqs for f in s]
    ctx.set_target(np.concatenate(frames[:3]), CELL)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_init[1])
    with spacing(ctx, S):
        rc_a, a = raw_odometry(ctx, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
        rc_b, b = raw_odometry(ctx, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
    rc_0, z = raw_odometry(ctx, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)     # the setting is back at 0
    assert rc_a == rc_b == rc_0 == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    assert a["npts"].tobytes() == z["npts"].tobytes() and a["T_out"].tobytes() != z["T_out"].tobytes()
    again = ctx.icp_run(prm, T_init[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    from dcreg_b200 import Context
    with Context(0) as fresh, spacing(fresh, S):
        rc, c = raw_odometry(fresh, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
        assert rc == 0
        for k in a:
            assert a[k].tobytes() == c[k].tobytes(), k


def test_launches_per_step_do_not_depend_on_sequences(ctx, odo):
    """With fixed iteration counts a spaced call launches what the unspaced call launches, for one sequence or three"""
    seqs, T_init, _ = odo
    prm = params(fixed_iterations=1, max_iterations=3)
    one = [seqs[2][:6]]
    three = [seqs[1][:6], seqs[2][:6], seqs[2][6:12]]
    T3 = np.stack([T_init[1], T_init[2], T_init[2]])
    counts = {}
    for name, ss, T0 in (("one", one, T_init[2:3]), ("three", three, T3)):
        for s in (0.0, S):
            with spacing(ctx, s):
                a = ctx.launch_count
                rc, _ = raw_odometry(ctx, MAP, prm, ss, T0, None, **RAW_MAP)
                b = ctx.launch_count
                ctx.icp_run_odometry(prm, ss, T0, None, map_frames=3, cell_size=CELL, source_voxel=SV, map_voxel=MV,
                                     map_max_points=CAP)
                counts[name, s] = (b - a, ctx.launch_count - b)
            assert rc == 0
    assert len(set(counts.values())) == 1, counts


def test_untouched_calls_and_maps(ctx, odo):
    """The spacing leaves plain odometry, a one-point map cap and an unfiltered map as they were"""
    seqs, T_init, deltas = odo
    prm = params()
    cases = [dict(), dict(source_voxel=SV, map_voxel=MV), dict(source_voxel=SV, source_max_points=4, map_max_points=4),
             dict(source_voxel=SV, source_max_points=4, map_voxel=MV, map_max_points=1)]
    for kw in cases:
        ref = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, **kw)
        a = ctx.launch_count
        ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, **kw)
        n_ref = ctx.launch_count - a
        with spacing(ctx, S):
            a = ctx.launch_count
            got = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, **kw)
            assert ctx.launch_count - a == n_ref
        assert_same([got], [ref])


def test_bad_arguments(ctx, odo):
    from dcreg_b200 import api
    good = [np.zeros((3, 3), np.float32), np.ones((2, 3), np.float32)]
    launches = ctx.launch_count
    for bad in (math.nan, -1e-9, -1.0, math.inf, -math.inf):
        assert raw_downsample(ctx, SPACED, good, 0.5, max_points=4, min_spacing=bad)[0] == api.BAD_ARG, bad
        assert "min_spacing" in ctx.lib.dcreg_last_error(ctx._h).decode()
        assert ctx.lib.dcreg_set_map_spacing(ctx._h, bad) == api.BAD_ARG, bad
        assert "min_spacing" in ctx.lib.dcreg_last_error(ctx._h).decode()
        with pytest.raises(api.DcregError):
            ctx.set_map_spacing(bad)
    assert ctx.launch_count == launches                                        # nothing launched
    # a refused setting leaves the last good one: 0 here, so a call is the unspaced call
    seqs, T_init, deltas = odo
    prm = params()
    a = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, source_voxel=SV, map_voxel=MV,
                             map_max_points=CAP)
    ctx.set_map_spacing(S)
    assert ctx.lib.dcreg_set_map_spacing(ctx._h, math.nan) == api.BAD_ARG
    b = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, source_voxel=SV, map_voxel=MV,
                             map_max_points=CAP)
    ctx.set_map_spacing(0.0)
    c = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, source_voxel=SV, map_voxel=MV,
                             map_max_points=CAP)
    assert [r.T.tobytes() for r in a] == [r.T.tobytes() for r in c] != [r.T.tobytes() for r in b]
    assert ctx.voxel_downsample(good, 0.5, 2, 0.1)[1][1].tolist() == [0]     # the context stays usable
