"""dcreg_icp_run_odometry: scan-to-map odometry, frame k registering against a local map the device builds from the
registered frames before it.

The reconstruction used throughout: take the call's own T_out for the frames before k, build frame k's map with
map_points in the documented order, and run set_target(map_k, cell) + set_source(frame k) + icp_run(T_prior[k]).  Every
registered frame equals that run to the rounding of FP64 sums grouped differently (the tolerances of
tests/test_gpu_sequences.py), every prior is compose_prior of the previous result byte for byte, and a call reproduces
bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o

from harness import RADIUS, assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, assert_anchor, assert_priors, parking, raw_odometry, reconstruct, split,  # noqa: F401
                          window_map)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def odo():
    """20 dense frames (about 20 k points, 16 points / m^2 of ground) of one path with drifting odometry, split into
    sequences of 1, 7 and 12 frames; T_init = the true pose of each sequence's first frame."""
    seqs, T_init, deltas, frames, T_true = parking()
    return seqs, frames, T_init, deltas, T_true


@pytest.mark.parametrize("method,cell", [pytest.param(m, c, id=m if c == CELL else f"{m}-cell{c}")
                                         for c in (CELL, CELL / 2) for m in ("Ours", "ME-TSVD")])
def test_frames_equal_their_reconstruction(ctx, odo, method, cell):
    """Ours runs the frame's last step in the loop kernel's folded step; ME-TSVD in the separate solve kernel.
    cell = CELL / 2: the local maps searched over 2 rings of cells."""
    seqs, frames, T_init, deltas, T_true = odo
    prm = params(method)
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=cell, want_log=True, want_cov=True)
    assert len(res) == len(frames) == 20
    assert_priors(res, seqs, T_init, deltas)
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        for k in range(1, len(seq)):
            assert_same_run(rs[k], reconstruct(ctx, prm, seq, rs, k, 3, cell=cell))
    assert sum(r.converged for r in res) >= 15
    assert max(o.se3_log_distance(r.T, T) for r, T in zip(res, T_true)) < 0.05


@pytest.mark.parametrize("map_frames", [1, 100])
def test_window_rule(ctx, odo, map_frames):
    """map_frames = 1: the previous frame alone; map_frames past the sequence: every frame before k."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    seq = seqs[2][:6]
    res = ctx.icp_run_odometry(prm, [seq], T_init[2:3], deltas[8:14], map_frames=map_frames, cell_size=CELL, want_log=True)
    assert_anchor(res[0], T_init[2])
    for k in range(1, len(seq)):
        assert_same_run(res[k], reconstruct(ctx, prm, seq, res, k, map_frames))


def test_constant_velocity_and_identity_priors(ctx, odo):
    seqs, _, T_init, _, _ = odo
    prm = params()
    short = [s[:5] for s in seqs]
    cv = ctx.icp_run_odometry(prm, short, T_init, motion="constant_velocity", map_frames=4, cell_size=CELL)
    assert_priors(cv, short, T_init, None, motion="constant_velocity")
    rs = split(cv, short)[2]
    for k in (1, 2, 4):
        assert_same_run(rs[k], reconstruct(ctx, prm, short[2], rs, k, 4), logs=False)
    ident = ctx.icp_run_odometry(prm, short, T_init, map_frames=4, cell_size=CELL)
    assert_priors(ident, short, T_init, None)


def test_side_by_side_equal_own_calls(ctx, odo):
    """Sequences of 1, 7 and 12 frames in one call: each matches the same sequence in a call of its own."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL)
    k = 0
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        alone = ctx.icp_run_odometry(prm, [seq], T_init[s:s + 1], deltas[k:k + len(seq)], map_frames=3, cell_size=CELL)
        for a, b in zip(rs, alone):
            assert (a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged)
            assert o.se3_log_distance(a.T, b.T) < 1e-8
        k += len(seq)


def test_abort_enters_later_maps(ctx, odo):
    """A 5-point frame aborts with NOT_ENOUGH_POINTS and returns its prior; it enters the later maps at that pose, and the
    frames after it still match their reconstructions."""
    from dcreg_b200 import api
    seqs, _, T_init, deltas, _ = odo
    seq = list(seqs[2][:6])
    seq[2] = seq[2][:5]
    prm = params()
    res = ctx.icp_run_odometry(prm, [seq], T_init[2:3], deltas[8:14], map_frames=3, cell_size=CELL, want_log=True)
    assert res[2].status == api.NOT_ENOUGH_POINTS and not res[2].converged
    assert res[2].T.tobytes() == res[2].T_prior.tobytes()
    assert_priors(res, [seq], T_init[2:3], deltas[8:14])
    for k in range(1, len(seq)):
        assert_same_run(res[k], reconstruct(ctx, prm, seq, res, k, 3))


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_fixed_iterations_run_every_frame_to_the_cap(ctx, odo, method):
    seqs, _, T_init, deltas, _ = odo
    prm = params(method, fixed_iterations=1, max_iterations=5)
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL)
    for s, rs in enumerate(split(res, seqs)):
        assert_anchor(rs[0], T_init[s])
        assert all(r.iterations == 5 and r.status == 0 and not r.converged for r in rs[1:])
    assert_priors(res, seqs, T_init, deltas)


def test_reproducible_and_context_intact(ctx, odo):
    from dcreg_b200.scenes import make_parking_sequence
    seqs, frames, T_init, deltas, T_true = odo
    prm = params()
    tgt = np.concatenate(frames[:3])
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_true[1])
    sq1 = ctx.icp_run_sequences(prm, [frames[:3]], T_true[:1], deltas[:3], want_log=True)
    a = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    b = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    for x, y in zip(a, b):
        assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
        assert x.T.tobytes() == y.T.tobytes() and x.T_prior.tobytes() == y.T_prior.tobytes()
        assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]
    again = ctx.icp_run(prm, T_true[1])                      # the context's source and target are untouched
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]
    sq2 = ctx.icp_run_sequences(prm, [frames[:3]], T_true[:1], deltas[:3], want_log=True)
    for x, y in zip(sq1, sq2):
        assert x.T.tobytes() == y.T.tobytes() and x.iterations == y.iterations
        assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]


def test_first_frames_match_oracle(ctx, odo):
    import dcreg_oracle_c as oc
    seqs, _, T_init, deltas, _ = odo
    seq = seqs[2][:4]
    res = ctx.icp_run_odometry(params(), [seq], T_init[2:3], deltas[8:12], map_frames=3, cell_size=CELL, want_log=True)
    cp = oc.make_params(search_radius=RADIUS, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    for k in (1, 2, 3):
        b = res[k]
        sc = oc.Scene(seq[k], window_map(seq, res, k, 3))
        st, conv, n_it, Tc, clogs = sc.icp_run(cp, b.T_prior)
        sc.close()
        assert (b.status, b.converged, b.iterations) == (st, conv, n_it), k
        for Cl, G in zip(clogs, b.logs):
            assert G.n_effective == Cl.n_eff and G.n_corr_pt == Cl.n_pt
            assert list(G.analysis.degenerate_mask) == list(Cl.mask)
        assert o.se3_log_distance(Tc, b.T) < 1e-6, k


def test_odometry_bad_arguments(ctx, odo):
    from dcreg_b200 import api, Context
    seqs, frames, T_init, deltas, _ = odo
    prm = params()
    lib, h = ctx.lib, ctx._h
    fr = [f[:2000] for f in frames[:4]]
    xyz = np.ascontiguousarray(np.concatenate(fr), dtype=np.float32)
    off = np.zeros(5, dtype=np.int64)
    off[1:] = np.cumsum([len(f) for f in fr])
    so = np.array([0, 1, 4], dtype=np.int32)
    T = np.ascontiguousarray(T_init[:2])
    D = np.ascontiguousarray(deltas[:4])
    dp = C.POINTER(C.c_double)

    def call(n_seqs=2, seq_off=so, n_frames=4, pts=xyz, offsets=off, p=prm, handle=h, T0=T, cell=CELL, map_frames=3,
             motion=0, Dd=D, stride=3):
        Tout = np.empty((max(n_frames, 1), 4, 4))
        return api._odometry_call(lib, handle, "dcreg_icp_run_odometry", params=C.byref(p), n_seqs=n_seqs,
                                  seq_offsets=seq_off.ctypes.data_as(C.POINTER(C.c_int)), n_frames=n_frames,
                                  xyz=pts.ctypes.data_as(C.POINTER(C.c_float)),
                                  frame_offsets=offsets.ctypes.data_as(C.POINTER(C.c_int64)), stride=stride,
                                  cell_size=cell, map_frames=map_frames, motion=motion, T_init=T0.ctypes.data_as(dp),
                                  deltas=Dd.ctypes.data_as(dp) if Dd is not None else None,
                                  T_out=Tout.ctypes.data_as(dp), log_cap=0)

    assert call() == api.OK
    assert call(motion=1, Dd=None) == api.OK
    bad = [dict(n_seqs=0), dict(n_seqs=-1), dict(seq_off=np.array([0, 3, 2], np.int32)), dict(seq_off=np.array([0, 0, 4], np.int32)),
           dict(seq_off=np.array([0, 1, 3], np.int32)),
           dict(offsets=np.array([0, off[1], off[1], off[3], off[4]], np.int64)),
           dict(map_frames=0), dict(map_frames=-2), dict(motion=2), dict(motion=-1), dict(motion=1),   # cv with deltas
           dict(cell=0.0), dict(cell=0.1), dict(stride=2),
           dict(p=params(max_iterations=0)), dict(p=params(weight_gate=1.5))]
    launches = ctx.launch_count
    for kw in bad:
        assert call(**kw) == api.BAD_ARG, kw
        assert lib.dcreg_last_error(h).decode(), kw
    n_big = 65536
    big = dict(n_seqs=1, seq_off=np.array([0, n_big], np.int32), n_frames=n_big, pts=np.zeros((n_big, 3), np.float32),
               offsets=np.arange(n_big + 1, dtype=np.int64), T0=np.ascontiguousarray(np.eye(4)[None]), Dd=None)
    assert call(**big) == api.BAD_ARG
    assert ctx.launch_count == launches                     # nothing launched by any of them
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_odometry(prm, [], np.zeros((0, 4, 4)))
    assert e.value.status == api.BAD_ARG
    # a map box out of range at a later step: frame 2 of the sequence carries a point 30 km away, so the map of frame 3
    # has no dense grid; frames 0 - 2 keep their outputs, and the context stays usable
    seq = [f[:3000] for f in seqs[2][:5]]
    seq[2] = np.concatenate([seq[2], np.array([[3.0e4, 3.0e4, 0.0]], np.float32)])
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_odometry(prm, [seq], T_init[2:3], deltas[8:13], map_frames=3, cell_size=CELL)
    assert e.value.status == api.BAD_ARG
    msg = lib.dcreg_last_error(h).decode()
    assert "sequence 0" in msg and "frame 3" in msg, msg
    rc, out = raw_odometry(ctx, "dcreg_icp_run_odometry", prm, [seq], T_init[2:3], deltas[8:13])
    n_it, Tout = out["n_it"], out["T_out"]
    assert rc == api.BAD_ARG
    assert all(n_it[k] >= 0 for k in range(3)) and n_it[1] > 0 and n_it[3] == -1 and n_it[4] == -1
    assert np.all(Tout[3:] == -1.0) and Tout[2, 3, 3] == 1.0
    good = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    with Context(0) as fresh:
        ref = fresh.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
        for x, y in zip(good, ref):
            assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
            assert x.T.tobytes() == y.T.tobytes()
            assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]
        try:
            fresh.comm_init(fresh.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        assert call(handle=fresh._h) == api.BAD_ARG
        assert "rank" in lib.dcreg_last_error(fresh._h).decode()
