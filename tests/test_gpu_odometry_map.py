"""Scan-to-map odometry with a persistent voxel map per sequence (dcreg_icp_run_odometry_map, dcreg_odometry_open_map,
dcreg_odometry_local_map), KISS-ICP's VoxelHashMap: M_{k+1} = voxel_map_update(M_k, F_s(frame k), T_out[k]).

The device's maps are checked bit for bit against the NumPy twin (api.voxel_map_update) after every push; every registered
frame against its reconstruction set_target(twin M_k) + set_source + icp_run(T_prior[k]); and at max_distance = inf every
output against the window call with a window as long as the longest sequence, byte for byte."""
import ctypes as C
import math

import numpy as np
import pytest

from harness import RADIUS, assert_same_run, ctx, log_bytes, params  # noqa: F401
from odom_harness import (CELL, RAGGED, assert_anchor, assert_priors, assert_same, assert_same_flat,  # noqa: F401
                          map_call, odo, one_per_push, pushed, raw_odometry, raw_push, seq_results, split, sweeps,
                          twin_maps, window_call)

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)
SV, MV = 0.3, 0.25            # source and map voxel sizes
DIST = 10.0                   # a prune distance well inside the scenes' 20 m sensor range
dp = C.POINTER(C.c_double)
MAP = "dcreg_icp_run_odometry_map"
RAW_MAP = dict(source_voxel=SV, map_voxel=MV, source_max_points=1, map_max_points=4, max_distance=DIST)


def map_session(ctx, prm, seqs, T_init, chunks, deltas=None, **kw):
    """The recording pushed in `chunks` into a voxel-map session, with logs and covariances: (results per sequence,
    [local maps of every sequence after each push])"""
    maps = []
    out = pushed(ctx, prm, seqs, T_init, chunks, deltas, voxel_map=True, maps=maps, want_log=True, want_cov=True, **kw)
    return out, maps


@pytest.mark.parametrize("cap", [1, 4])
@pytest.mark.parametrize("sv", [SV, 0.0], ids=["filtered", "unfiltered"])
def test_local_map_equals_twin_after_every_push(ctx, odo, cap, sv):
    from dcreg_b200.api import map_points, voxel_downsample
    seqs, T_init, deltas = odo
    prm = params()
    res, maps = map_session(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, source_voxel=sv, map_voxel=MV,
                            map_max_points=cap, max_distance=DIST)
    pruned = 0
    for s, (seq, rs) in enumerate(zip(seqs, res)):
        twin = twin_maps(seq, rs, sv, MV, cap, DIST)
        for i in range(len(maps)):
            k = min(i + 1, len(seq))                    # frames of sequence s pushed after push i
            assert maps[i][s].tobytes() == twin[k].tobytes(), (s, i)
        every = np.concatenate([map_points(r.T, voxel_downsample(f, sv, 1)[0] if sv else f) for f, r in zip(seq, rs)])
        pruned += len(voxel_downsample(every, MV, cap)[0]) - len(twin[-1])
    assert pruned > 0


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_infinite_distance_is_the_long_window(ctx, odo, method, motion):
    """max_distance = inf: the _voxel_n call with map_frames >= the longest sequence, byte for byte"""
    seqs, T_init, deltas = odo
    prm = params(method)
    D = deltas if motion == "increments" else None
    for kw in (dict(source_voxel=SV, map_voxel=MV, map_max_points=4), dict(map_voxel=MV)):
        ref = window_call(ctx, prm, seqs, T_init, D, motion=motion, **kw)
        got = map_call(ctx, prm, seqs, T_init, D, math.inf, motion=motion, **kw)
        assert_same_flat(got, ref)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_infinite_distance_with_timestamps_is_the_long_window(ctx, sweeps, method):
    """... and with timestamps the _deskew call, deskewed points included"""
    sw = sweeps
    prm = params(method)
    for motion in ("increments", "constant_velocity"):
        D = sw["deltas"] if motion == "increments" else None
        kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=4, motion=motion, timestamps=sw["stamps"],
                  want_deskewed=True)
        ref = window_call(ctx, prm, sw["skewed"], sw["T_init"], D, **kw)
        got = map_call(ctx, prm, sw["skewed"], sw["T_init"], D, math.inf, **kw)
        assert_same_flat(got, ref)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_frames_equal_their_reconstruction(ctx, odo, method):
    """At a finite distance every registered frame is the single run against the twin's M_k, from compose_prior"""
    from dcreg_b200.api import voxel_downsample
    seqs, T_init, deltas = odo
    prm = params(method)
    res = map_call(ctx, prm, seqs, T_init, deltas, DIST, source_voxel=SV, map_voxel=MV, map_max_points=4)
    assert [r.n_points for r in res] == [len(voxel_downsample(f, SV, 1)[1]) for s in seqs for f in s]
    assert_priors(res, seqs, T_init, deltas)
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        twin = twin_maps(seq, rs, SV, MV, 4, DIST)
        for k in range(1, len(seq)):
            ctx.set_target(twin[k], CELL)
            ctx.set_source(voxel_downsample(seq[k], SV, 1)[0])
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))


def test_deskewed_frames_enter_the_map(ctx, sweeps):
    """With timestamps a frame enters the map as its deskewed kept points"""
    from dcreg_b200.api import voxel_downsample
    sw = sweeps
    prm = params()
    res = map_call(ctx, prm, sw["skewed"], sw["T_init"], sw["deltas"], DIST, source_voxel=SV, map_voxel=MV,
                   map_max_points=4, timestamps=sw["stamps"], want_deskewed=True)
    for seq, rs in zip(sw["skewed"], split(res, sw["skewed"])):
        twin = twin_maps(seq, rs, SV, MV, 4, DIST, frames=[r.deskewed for r in rs])
        for k in range(1, len(seq)):
            ctx.set_target(twin[k], CELL)
            ctx.set_source(rs[k].deskewed)
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))
        assert len(voxel_downsample(seq[0], SV, 1)[0]) == rs[0].n_points


CHUNKS = {"one_per_push": one_per_push(LENS), "ragged": RAGGED, "all_at_once": [list(LENS)]}


@pytest.mark.parametrize("chunking", sorted(CHUNKS))
def test_session_chunkings_equal_one_call(ctx, odo, chunking):
    seqs, T_init, deltas = odo
    prm = params()
    kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=4)
    ref = map_call(ctx, prm, seqs, T_init, deltas, DIST, **kw)
    got, maps = map_session(ctx, prm, seqs, T_init, CHUNKS[chunking], deltas, max_distance=DIST, **kw)
    assert_same(got, seq_results(ref, seqs))
    for s, (seq, rs) in enumerate(zip(seqs, got)):                 # the last maps hold every frame
        assert maps[-1][s].tobytes() == twin_maps(seq, rs, SV, MV, 4, DIST)[-1].tobytes()


def test_session_constant_velocity_across_pushes(ctx, odo):
    seqs, T_init, _ = odo
    prm = params()
    kw = dict(map_voxel=MV, map_max_points=4, motion="constant_velocity")
    ref = seq_results(map_call(ctx, prm, seqs, T_init, None, DIST, **kw), seqs)
    for chunks in ([[1, 1, 1]] + one_per_push([0, 6, 11]), RAGGED):
        got, _ = map_session(ctx, prm, seqs, T_init, chunks, None, max_distance=DIST, **kw)
        assert_same(got, ref)


def test_session_mixed_deskew_and_plain_pushes(ctx, sweeps):
    """A push without timestamps is a call whose frames have every tau = 0.5"""
    sw = sweeps
    prm = params()
    seqs = sw["skewed"]
    chunks = one_per_push([len(s) for s in seqs])
    plain = lambda i: i % 2 == 1                                                  # noqa: E731
    stamps = [[t if not plain(j) else np.full_like(t, 0.5) for j, t in enumerate(ts)] for ts in sw["stamps"]]
    kw = dict(source_voxel=SV, map_voxel=MV, map_max_points=4)
    ref = seq_results(map_call(ctx, prm, seqs, sw["T_init"], sw["deltas"], DIST, timestamps=stamps, **kw), seqs)
    got, _ = map_session(ctx, prm, seqs, sw["T_init"], chunks, sw["deltas"], stamps=sw["stamps"],
                         ts_push=lambda i: not plain(i), max_distance=DIST, **kw)
    assert_same(got, ref)


def test_session_other_calls_between_pushes(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    tgt = np.concatenate(seqs[2][:3])
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(seqs[2][1])
    before = ctx.icp_run(prm, T_init[2])
    kw = dict(map_voxel=MV, map_max_points=4)
    ref = seq_results(map_call(ctx, prm, seqs, T_init, deltas, DIST, **kw), seqs)
    seen = []

    def between(i):
        kind = i % 4
        if kind == 0:
            ctx.icp_run_odometry_map(prm, [seqs[1][:3]], T_init[1:2], deltas[1:4], map_voxel=MV, max_distance=3.0,
                                     cell_size=CELL)
        elif kind == 1:
            ctx.icp_run_odometry(prm, [seqs[1][:3]], T_init[1:2], deltas[1:4], map_frames=2, cell_size=CELL,
                                 map_voxel=0.5)
        elif kind == 2:
            ctx.set_target(tgt, RADIUS)
            ctx.set_source(seqs[2][1])
            seen.append(ctx.icp_run(prm, T_init[2]))
        else:
            ctx.voxel_downsample([seqs[2][3], seqs[1][2]], 0.3, 2)

    got, _ = map_session(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, between=between, max_distance=DIST, **kw)
    assert_same(got, ref)
    for r in seen + [ctx.icp_run(prm, T_init[2])]:
        assert (r.status, r.iterations, r.converged) == (before.status, before.iterations, before.converged)
        assert r.T.tobytes() == before.T.tobytes()
        assert [log_bytes(x) for x in r.logs] == [log_bytes(y) for y in before.logs]


def test_failed_pushes_change_nothing(ctx, odo):
    """Pre-launch errors (bad tables, a timestamp outside [0, 1]) launch nothing; a frame whose points leave the map
    filter's voxel range (an increment of 10^6 m before it) fails its push at the push's final update, naming the
    sequence and its frame since open.  After each, the session's map is as it was and the session continues as if it
    had never seen the push."""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    seq = [f[:6000] for f in seqs[2][:6]]
    D = deltas[8:14]
    prm = params()
    kw = dict(map_voxel=MV, map_max_points=4)
    ref = seq_results(map_call(ctx, prm, [seq], T_init[2:3], D, DIST, **kw), [seq])
    D_far = D.copy()
    D_far[3, 0, 3] += 1.0e6                                                    # frame 4's prior, 10^6 m away
    lib, h = ctx.lib, ctx._h
    with ctx.odometry_map_session(prm, 1, T_init[2:3], cell_size=CELL, max_distance=DIST, **kw) as sess:
        got = sess.push([seq[:3]], D[:3], want_log=True, want_cov=True)[0]
        before = sess.local_map(0)
        launches = ctx.launch_count
        assert raw_push(ctx, [0, 2], seq[3:5], stride=2) == api.BAD_ARG
        assert raw_push(ctx, [0, 2], seq[3:5], offsets=[0, 10, 10]) == api.BAD_ARG
        with pytest.raises(api.DcregError):
            sess.push([[seq[3]]], None, timestamps=[[np.full(len(seq[3]), 2.0, np.float32)]])
        assert ctx.launch_count == launches
        assert sess.local_map(0).tobytes() == before.tobytes()
        with pytest.raises(api.DcregError) as e:
            sess.push([seq[3:5]], D_far[3:5])
        msg = lib.dcreg_last_error(h).decode()
        assert e.value.status == api.BAD_ARG
        assert "sequence 0" in msg and "frame 4 of the sequence since open" in msg and "voxel" in msg, msg
        assert sess.local_map(0).tobytes() == before.tobytes()
        got += sess.push([seq[3:]], D[3:], want_log=True, want_cov=True)[0]
        final = sess.local_map(0)
    assert_same([got], ref)
    assert final.tobytes() == twin_maps(seq, got, 0.0, MV, 4, DIST)[-1].tobytes()


def test_empty_map_fails_at_its_step(ctx, odo):
    """A max_distance below every voxel's distance leaves the map empty: BAD_ARG at the first registered frame, the anchor
    returned, the context usable"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    prm = params()
    seq = [f[:3000] for f in seqs[2][:3]]
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_odometry_map(prm, [seq], T_init[2:3], deltas[8:11], map_voxel=MV, max_distance=1e-3, cell_size=CELL)
    assert e.value.status == api.BAD_ARG and "empty" in str(e.value) and "frame 1" in str(e.value)
    assert len(ctx.icp_run_odometry_map(prm, [seq], T_init[2:3], deltas[8:11], map_voxel=MV, max_distance=DIST,
                                        cell_size=CELL)) == 3


def test_more_sequences_than_map_points(ctx, odo):
    """300 sequences, the first push one 100-point anchor: the push's final update has one segment per sequence, more
    segments than points, and every sequence's map comes back right.  Then anchors for sequences 255 .. 299 and a second
    frame of sequence 0."""
    from dcreg_b200.api import voxel_map_update
    seqs, T_init, _ = odo
    S = 300
    frames = [np.ascontiguousarray(f[:100]) for f in seqs[2][:2]]
    T0 = np.repeat(T_init[2:3], S, axis=0)
    empty = np.zeros((0, 3), np.float32)
    want = [empty] * S
    with ctx.odometry_map_session(params(), S, T0, cell_size=CELL, map_voxel=MV, map_max_points=4,
                                  max_distance=DIST) as sess:
        push = [[] for _ in range(S)]
        push[0] = [frames[0]]
        sess.push(push)
        want[0] = voxel_map_update(empty, frames[0], T0[0], MV, 4, DIST)
        assert [sess.local_map(s).tobytes() for s in range(S)] == [w.tobytes() for w in want]
        push = [[] for _ in range(S)]
        push[0] = [frames[1]]
        for s in range(255, S):
            push[s] = [frames[s % 2]]
        res = sess.push(push)
        want[0] = voxel_map_update(want[0], frames[1], res[0][0].T, MV, 4, DIST)
        for s in range(255, S):
            want[s] = voxel_map_update(empty, frames[s % 2], T0[s], MV, 4, DIST)
        assert [sess.local_map(s).tobytes() for s in range(S)] == [w.tobytes() for w in want]


def test_reproducible_and_context_intact(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    frames = [f for s in seqs for f in s]
    ctx.set_target(np.concatenate(frames[:3]), CELL)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_init[1])
    rc_a, a = raw_odometry(ctx, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
    rc_b, b = raw_odometry(ctx, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    again = ctx.icp_run(prm, T_init[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [log_bytes(x) for x in again.logs] == [log_bytes(y) for y in one.logs]
    from dcreg_b200 import Context
    with Context(0) as fresh:
        rc, c = raw_odometry(fresh, MAP, prm, seqs, T_init, deltas, log_cap=30, **RAW_MAP)
        assert rc == 0
        for k in a:
            assert a[k].tobytes() == c[k].tobytes(), k


def test_launches_per_step_do_not_depend_on_sequences(ctx, odo):
    """Fixed iteration counts make every step's loop the same: a call of one sequence launches what a call of three
    launches, and once every map is past its first frames, equal-shaped pushes launch the same"""
    seqs, T_init, _ = odo
    prm = params(fixed_iterations=1, max_iterations=3)
    one = [seqs[2][:6]]
    three = [seqs[1][:6], seqs[2][:6], seqs[2][6:12]]
    counts = []
    for ss, T0 in ((one, T_init[2:3]), (three, np.stack([T_init[1], T_init[2], T_init[2]]))):
        a = ctx.launch_count
        rc, _ = raw_odometry(ctx, MAP, prm, ss, T0, None, **RAW_MAP)
        assert rc == 0
        counts.append(ctx.launch_count - a)
    assert counts[0] == counts[1], counts
    pushes = {}
    for name, ss, T0 in (("one", one, T_init[2:3]), ("three", three, np.stack([T_init[1], T_init[2], T_init[2]]))):
        pushes[name] = []
        with ctx.odometry_map_session(prm, len(ss), T0, cell_size=CELL, map_voxel=MV, map_max_points=4,
                                      max_distance=DIST) as sess:
            for k in range(6):
                before = ctx.launch_count
                sess.push([[s[k]] for s in ss])
                pushes[name].append(ctx.launch_count - before)
    assert len(set(pushes["one"][1:])) == 1 and pushes["one"] == pushes["three"], pushes


def test_bad_arguments(ctx, odo):
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    prm = params()
    lib, h = ctx.lib, ctx._h
    seq = [f[:3000] for f in seqs[2][:4]]
    launches = ctx.launch_count
    for mv, cap, dist, what in ((0.0, 4, DIST, "map_voxel"), (math.inf, 4, DIST, "map_voxel"),
                                (math.nan, 4, DIST, "map_voxel"), (MV, 0, DIST, "max_points"),
                                (MV, 4, 0.0, "max_distance"), (MV, 4, -1.0, "max_distance"),
                                (MV, 4, math.nan, "max_distance")):
        rc, out = raw_odometry(ctx, MAP, prm, [seq], T_init[2:3], deltas[8:12], log_cap=30,
                               **(RAW_MAP | dict(map_voxel=mv, map_max_points=cap, max_distance=dist)))
        assert rc == api.BAD_ARG, (mv, cap, dist)
        assert what in lib.dcreg_last_error(h).decode(), (mv, cap, dist)
        assert np.all(out["n_it"] == -1)
        T0 = np.ascontiguousarray(T_init[2:3])
        assert lib.dcreg_odometry_open_map(h, C.byref(prm), 1, CELL, 0, 0.0, float(mv), 1, int(cap), float(dist),
                                           T0.ctypes.data_as(dp)) == api.BAD_ARG
    assert ctx.launch_count == launches
    n = C.c_int64(-1)
    xyz = np.zeros((4, 3), np.float32)
    fp = xyz.ctypes.data_as(C.POINTER(C.c_float))
    assert lib.dcreg_odometry_local_map(h, 0, fp, 4, C.byref(n)) == api.BAD_ARG                # no session
    assert "no session" in lib.dcreg_last_error(h).decode()
    with ctx.odometry_session(prm, 1, T_init[2:3], map_frames=3, cell_size=CELL):              # a window session
        assert lib.dcreg_odometry_local_map(h, 0, fp, 4, C.byref(n)) == api.BAD_ARG
        assert "window" in lib.dcreg_last_error(h).decode()
    with ctx.odometry_map_session(prm, 2, T_init[1:3], cell_size=CELL, map_voxel=MV, max_distance=math.inf) as sess:
        assert lib.dcreg_odometry_local_map(h, 0, None, 0, C.byref(n)) == api.OK and n.value == 0  # before any frame
        assert sess.local_map(1).shape == (0, 3)
        for bad in (-1, 2):
            assert lib.dcreg_odometry_local_map(h, bad, fp, 4, C.byref(n)) == api.BAD_ARG
        sess.push([[seq[0]], seq[:2]])
        m = sess.local_map(1)
        assert len(m) > 4
        n.value = -1
        short = np.full((len(m) - 1, 3), 7.0, np.float32)
        assert lib.dcreg_odometry_local_map(h, 1, short.ctypes.data_as(C.POINTER(C.c_float)), len(m) - 1,
                                            C.byref(n)) == api.BAD_ARG
        assert n.value == len(m) and np.all(short == 7.0)                                        # nothing else written
        assert lib.dcreg_odometry_local_map(h, 1, None, len(m), None) == api.BAD_ARG
