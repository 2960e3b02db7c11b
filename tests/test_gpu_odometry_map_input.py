"""The map-input filter of scan-to-map odometry (dcreg_set_map_input_voxel, KISS-ICP's Voxelize): the frames enter the
local maps as F_in(frame) = voxel_downsample(frame, VIN) and register with F_s(F_in(frame)).

What is held: 0 is every call as before (bytes and launches of a fresh context); with source_voxel = 0 the source is
F_in itself, the call at source_voxel = VIN byte for byte; every registered frame of a split call equals its single run
against the twin's map of F_in points, window and voxel map, with and without deskewing; sessions under any chunking
equal the one call and keep the value they had at open; the errors name the sequence and frame."""
import contextlib
import math

import numpy as np
import pytest

from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, RAGGED, assert_anchor, assert_same, assert_same_flat, map_call, odo,  # noqa: F401
                          one_per_push, pushed, raw_odometry, raw_push, seq_results, split, sweeps, twin_maps,
                          window_map)

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)
VIN, SV, MV = 0.1, 0.3, 0.25          # map-input, source and map voxel sizes
CAP, DIST = 4, 10.0
MAPS = ["window", "voxel_map"]
FILTERS = dict(source_voxel=SV, map_voxel=MV, map_max_points=CAP)
RAW = dict(source_voxel=SV, map_voxel=MV, source_max_points=1, map_max_points=CAP, max_distance=DIST)
ENTRIES = ["dcreg_icp_run_odometry_voxel", "dcreg_icp_run_odometry_voxel_n", "dcreg_icp_run_odometry_deskew",
           "dcreg_icp_run_odometry_map", "dcreg_icp_run_odometry_adaptive", "dcreg_icp_run_odometry_gyro"]


@contextlib.contextmanager
def map_input(ctx, v):
    ctx.set_map_input_voxel(v)
    try:
        yield
    finally:
        ctx.set_map_input_voxel(0.0)


def run(ctx, which, prm, seqs, T_init, deltas, **kw):
    """The window call (map_frames 3) or the voxel map pruned at DIST, with logs and covariances"""
    if which == "voxel_map":
        return map_call(ctx, prm, seqs, T_init, deltas, DIST, **kw)
    return ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, want_cov=True,
                                **kw)


def f_in(P, stamps=None):
    """F_in(P) and, with stamps, its points' timestamps"""
    from dcreg_b200.api import voxel_downsample
    pts, idx = voxel_downsample(P, VIN)
    return pts if stamps is None else (pts, np.asarray(stamps, np.float32)[idx])


def within_contract(got, ref):
    ulp = np.spacing(np.abs(ref)).astype(np.float64)
    return bool((np.abs(got.astype(np.float64) - ref.astype(np.float64)) <= np.maximum(ulp, 1e-12)).all())


def twin_map(which, seq, rs, k, frames):
    """M_k of the twin from the frames as they enter the maps"""
    if which == "voxel_map":
        return twin_maps(seq, rs, SV, MV, CAP, DIST, frames=frames)[k]
    return window_map(seq, rs, k, 3, mv=MV, caps=(1, CAP), frames=frames)


def test_off_means_off(ctx, odo):
    """After set_map_input_voxel(0) every affected entry point and a session give a fresh context's bytes and launches"""
    from dcreg_b200 import Context
    seqs, T_init, deltas = odo
    prm = params()
    ref, counts = {}, {}
    with Context(0) as fresh:
        for e in ENTRIES:
            raw_odometry(fresh, e, prm, seqs, T_init, deltas, **RAW)
            a = fresh.launch_count
            ref[e] = raw_odometry(fresh, e, prm, seqs, T_init, deltas, log_cap=30, **RAW)
            counts[e] = fresh.launch_count - a
        sess_ref = pushed(fresh, prm, seqs, T_init, RAGGED, deltas, voxel_map=True, want_log=True, want_cov=True,
                          max_distance=DIST, **FILTERS)
    ctx.set_map_input_voxel(VIN)
    ctx.set_map_input_voxel(0.0)
    for e in ENTRIES:
        raw_odometry(ctx, e, prm, seqs, T_init, deltas, **RAW)
        a = ctx.launch_count
        rc, got = raw_odometry(ctx, e, prm, seqs, T_init, deltas, log_cap=30, **RAW)
        assert ctx.launch_count - a == counts[e], e
        assert rc == ref[e][0] == 0, e
        for k in got:
            assert got[k].tobytes() == ref[e][1][k].tobytes(), (e, k)
    assert_same(pushed(ctx, prm, seqs, T_init, RAGGED, deltas, voxel_map=True, want_log=True, want_cov=True,
                       max_distance=DIST, **FILTERS), sess_ref)


@pytest.mark.parametrize("stamped", [False, True])
@pytest.mark.parametrize("which", MAPS)
def test_no_source_filter_is_the_source_filter_at_the_map_input_voxel(ctx, sweeps, which, stamped):
    """map_input_voxel = VIN, source_voxel = 0 is the call at source_voxel = VIN, source_max_points = 1 without it"""
    sw = sweeps
    prm = params()
    kw = dict(map_voxel=MV, map_max_points=CAP, want_deskewed=stamped, timestamps=sw["stamps"] if stamped else None)
    ref = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], source_voxel=VIN, **kw)
    with map_input(ctx, VIN):
        got = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], source_voxel=0.0, **kw)
    assert_same_flat(got, ref)


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
@pytest.mark.parametrize("which", MAPS)
def test_frames_equal_their_twin(ctx, odo, which, method, motion):
    """Every registered frame is set_target(twin M_k of F_in points) + set_source(F_s(F_in(frame k))) + icp_run"""
    from dcreg_b200.api import voxel_downsample
    seqs, T_init, deltas = odo
    prm = params(method)
    D = deltas if motion == "increments" else None
    with map_input(ctx, VIN):
        res = run(ctx, which, prm, seqs, T_init, D, motion=motion, **FILTERS)
    denser = 0
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        fin = [f_in(P) for P in seq]
        src = [voxel_downsample(F, SV)[0] for F in fin]
        for k in range(len(seq)):
            assert rs[k].n_points == len(src[k]), (s, k)
        for k in range(1, len(seq)):
            M = twin_map(which, seq, rs, k, fin)
            denser += len(M) - len(twin_map(which, seq, rs, k, src))
            ctx.set_target(M, CELL)
            ctx.set_source(src[k])
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))
    assert denser > 0                   # the maps hold more than the sources would give them


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
@pytest.mark.parametrize("which", MAPS)
def test_deskewed_frames_equal_their_twin(ctx, sweeps, which, method):
    """With timestamps: F_in's points deskewed by the call's increments enter the maps, and the source is the deskewed
    copies of its own F_in points.  With increments the deskew does not depend on the poses, so the call at
    source_voxel = 0 returns the deskewed F_in points the split call put in its maps."""
    from dcreg_b200.api import deskew_points, voxel_downsample
    sw = sweeps
    prm = params(method)
    kw = dict(timestamps=sw["stamps"], want_deskewed=True, map_voxel=MV, map_max_points=CAP)
    with map_input(ctx, VIN):
        res = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], source_voxel=SV, **kw)
        fin_run = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], source_voxel=0.0, **kw)
    k0, moved = 0, 0
    for seq, stamps, rs, fs in zip(sw["skewed"], sw["stamps"], split(res, sw["skewed"]), split(fin_run, sw["skewed"])):
        dfin = []
        for k in range(len(seq)):
            F, ts = f_in(seq[k], stamps[k])
            src, sidx = voxel_downsample(F, SV)
            assert rs[k].n_points == len(src) and fs[k].n_points == len(F)
            assert rs[k].deskewed.tobytes() == fs[k].deskewed[sidx].tobytes(), k
            if k == 0:
                assert fs[k].deskewed.tobytes() == F.tobytes()
            else:
                D = sw["deltas"][k0 + k - 1]
                assert within_contract(fs[k].deskewed, deskew_points(F, ts, D))
                assert within_contract(rs[k].deskewed, deskew_points(src, ts[sidx], D))
                moved += int((rs[k].deskewed != src).any(axis=1).sum())
            dfin.append(fs[k].deskewed)
        for k in range(1, len(seq)):
            ctx.set_target(twin_map(which, seq, rs, k, dfin), CELL)
            ctx.set_source(rs[k].deskewed)
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))
        k0 += len(seq)
    assert moved > 0


CHUNKS = {"one_per_push": one_per_push(LENS), "ragged": RAGGED, "all_at_once": [list(LENS)]}


@pytest.mark.parametrize("chunking", sorted(CHUNKS))
def test_sessions_equal_one_call(ctx, odo, chunking):
    """Any chunking gives the one call's bytes and the twin's local maps; a session keeps the value it had at open"""
    seqs, T_init, deltas = odo
    prm = params()
    toggle = lambda i: ctx.set_map_input_voxel([0.0, 0.2, VIN][i % 3])       # noqa: E731
    with map_input(ctx, VIN):
        ref = run(ctx, "voxel_map", prm, seqs, T_init, deltas, **FILTERS)
        wref = run(ctx, "window", prm, seqs, T_init, deltas, **FILTERS)
        maps = []
        got = pushed(ctx, prm, seqs, T_init, CHUNKS[chunking], deltas, voxel_map=True, maps=maps, between=toggle,
                     want_log=True, want_cov=True, max_distance=DIST, **FILTERS)
        ctx.set_map_input_voxel(VIN)
        assert_same(got, seq_results(ref, seqs))
        for s, (seq, rs) in enumerate(zip(seqs, got)):
            assert maps[-1][s].tobytes() == twin_maps(seq, rs, SV, MV, CAP, DIST, frames=[f_in(P) for P in seq])[-1].tobytes()
        out = pushed(ctx, prm, seqs, T_init, CHUNKS[chunking], deltas, between=toggle, want_log=True, want_cov=True,
                     map_frames=3, **FILTERS)
        ctx.set_map_input_voxel(VIN)
        assert_same(out, seq_results(wref, seqs))


@pytest.mark.parametrize("which", MAPS)
def test_deskewed_sessions_equal_one_call(ctx, sweeps, which):
    sw = sweeps
    prm = params()
    lens = [len(s) for s in sw["skewed"]]
    kw = dict(want_deskewed=True, **FILTERS)
    with map_input(ctx, VIN):
        ref = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], timestamps=sw["stamps"], **kw)
        extra = dict(voxel_map=True, max_distance=DIST) if which == "voxel_map" else dict(map_frames=3)
        got = pushed(ctx, prm, sw["skewed"], sw["T_init"], one_per_push(lens), sw["deltas"], stamps=sw["stamps"],
                     want_log=True, want_cov=True, **extra, **kw)
    assert_same_flat([r for s in got for r in s], ref)


def test_local_map_after_every_push(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    maps = []
    with map_input(ctx, VIN):
        res = pushed(ctx, prm, seqs, T_init, one_per_push(LENS), deltas, voxel_map=True, maps=maps, max_distance=DIST,
                     **FILTERS)
    for s, (seq, rs) in enumerate(zip(seqs, res)):
        twin = twin_maps(seq, rs, SV, MV, CAP, DIST, frames=[f_in(P) for P in seq])
        for i in range(len(maps)):
            assert maps[i][s].tobytes() == twin[min(i + 1, len(seq))].tobytes(), (s, i)


def test_reproducible_and_context_intact(ctx, odo):
    seqs, T_init, deltas = odo
    prm = params()
    frames = [f for s in seqs for f in s]
    ctx.set_target(np.concatenate(frames[:3]), CELL)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_init[1])
    with map_input(ctx, VIN):
        rc_a, a = raw_odometry(ctx, "dcreg_icp_run_odometry_map", prm, seqs, T_init, deltas, log_cap=30, **RAW)
        rc_b, b = raw_odometry(ctx, "dcreg_icp_run_odometry_map", prm, seqs, T_init, deltas, log_cap=30, **RAW)
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    again = ctx.icp_run(prm, T_init[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    from dcreg_b200 import Context
    with Context(0) as fresh, map_input(fresh, VIN):
        rc, c = raw_odometry(fresh, "dcreg_icp_run_odometry_map", prm, seqs, T_init, deltas, log_cap=30, **RAW)
        assert rc == 0
        for k in a:
            assert a[k].tobytes() == c[k].tobytes(), k


def test_launches_do_not_depend_on_sequences(ctx, odo):
    seqs, T_init, _ = odo
    prm = params(fixed_iterations=1, max_iterations=3)
    one = [seqs[2][:6]]
    three = [seqs[1][:6], seqs[2][:6], seqs[2][6:12]]
    T3 = np.stack([T_init[1], T_init[2], T_init[2]])
    counts = {}
    with map_input(ctx, VIN):
        for name, ss, T0 in (("one", one, T_init[2:3]), ("three", three, T3)):
            for e in ("dcreg_icp_run_odometry_map", "dcreg_icp_run_odometry_voxel_n"):
                a = ctx.launch_count
                rc, _ = raw_odometry(ctx, e, prm, ss, T0, None, **RAW)
                assert rc == 0
                counts.setdefault(e, set()).add(ctx.launch_count - a)
    assert all(len(v) == 1 for v in counts.values()), counts


def test_bad_arguments(ctx, odo):
    from dcreg_b200 import api
    launches = ctx.launch_count
    for bad in (math.nan, -1e-9, -1.0, math.inf, -math.inf):
        assert ctx.lib.dcreg_set_map_input_voxel(ctx._h, bad) == api.BAD_ARG, bad
        assert "set_map_input_voxel" in ctx.lib.dcreg_last_error(ctx._h).decode()
        with pytest.raises(api.DcregError):
            ctx.set_map_input_voxel(bad)
    assert ctx.launch_count == launches
    seqs, T_init, deltas = odo
    prm = params()
    empty = np.full((50, 3), np.nan, np.float32)
    far = np.full((50, 3), 1.0e6, np.float32)
    bad_seqs = [seqs[0], seqs[1][:3] + [empty], seqs[2][:4]]
    far_seqs = [seqs[0], seqs[1][:2], seqs[2][:2] + [far]]
    with map_input(ctx, VIN):
        for sv in (SV, 0.0):
            for entry in ("dcreg_icp_run_odometry_voxel_n", "dcreg_icp_run_odometry_map"):
                raw = RAW | dict(source_voxel=sv)
                rc, out = raw_odometry(ctx, entry, prm, bad_seqs, T_init, None, **raw)
                msg = ctx.lib.dcreg_last_error(ctx._h).decode()
                assert rc == api.BAD_ARG
                assert "sequence 1, frame 4 (frame 3 of the sequence)" in msg
                assert "no point is left by the map-input filter" in msg, msg
                assert (out["T_out"] == -1.0).all()                  # before any loop launch
                rc, _ = raw_odometry(ctx, entry, prm, far_seqs, T_init, None, **raw)
                msg = ctx.lib.dcreg_last_error(ctx._h).decode()
                assert rc == api.BAD_ARG
                assert "sequence 2, frame 5 (frame 2 of the sequence)" in msg
                assert "a voxel coordinate of the map-input filter lies outside [-2^20, 2^20)" in msg, msg
        # a push that fails commits nothing
        ref = pushed(ctx, prm, seqs, T_init, [list(LENS)], voxel_map=True, max_distance=DIST, **FILTERS)
        with ctx.odometry_map_session(prm, 3, T_init, cell_size=CELL, max_distance=DIST, **FILTERS) as sess:
            first = sess.push([seqs[0], seqs[1][:3], seqs[2][:5]])
            assert raw_push(ctx, [0, 0, 1, 1], [empty]) == api.BAD_ARG
            assert "frame 3 of the sequence since open" in ctx.lib.dcreg_last_error(ctx._h).decode()
            rest = sess.push([[], seqs[1][3:], seqs[2][5:]])
        got = [first[s] + rest[s] for s in range(3)]
        assert_same(got, ref)
