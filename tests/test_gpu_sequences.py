"""dcreg_icp_run_sequences: sequences of frames against one map, frame k+1 starting on the device from frame k's result
composed with its odometry increment.

A sequence of one frame is a scan batch bit for bit (same sort, grid and arithmetic: the lane / frame indirection adds
nothing).  Every chained frame is the registration dcreg_set_source(frame) + dcreg_icp_run(T_prior) gives, to the rounding
of FP64 sums grouped differently (the tolerances of tests/test_gpu_scans.py), and every prior is compose_prior of the
previous frame's result, byte for byte.  A call reproduces bit for bit and leaves the context's source untouched.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o
from harness import RADIUS, assert_same_run, ctx, params  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    """The 16 ragged frames (40 - 8 000 points) of tests/test_gpu_scans.py."""
    from dcreg_b200.scenes import make_parking_frames
    frames, T_true, T_init, tgt = make_parking_frames(16, seed=51, n_scan=8_400)
    sizes = [6_000, 40, 8_000, 5_120, 300, 7_311, 2_500, 6_666, 999, 4_097, 7_800, 3_333, 256, 5_555, 7_001, 1_234]
    rng = np.random.default_rng(52)
    cut = [f[np.sort(rng.choice(len(f), size=n, replace=False))] for f, n in zip(frames, sizes)]
    return cut, T_true, T_init, tgt


@pytest.fixture(scope="module")
def chain():
    """32 frames of one path with drifting odometry, cut to ragged sizes, split into sequences of 1, 7 and 24 frames."""
    from dcreg_b200.scenes import make_parking_sequence, make_parking_frames
    frames, T_true, _, deltas, tgt = make_parking_sequence(32, seed=61)
    _, _, T_init, _ = make_parking_frames(32, seed=61)
    rng = np.random.default_rng(62)
    sizes = rng.integers(300, 8_000, size=32)
    cut = [f[np.sort(rng.choice(len(f), size=min(int(n), len(f)), replace=False))] for f, n in zip(frames, sizes)]
    bounds = [0, 1, 8, 32]
    seqs = [cut[a:b] for a, b in zip(bounds[:-1], bounds[1:])]
    return seqs, cut, T_init[bounds[:-1]], deltas, T_true, tgt


def assert_chained_priors(res, seqs, T_init, deltas):
    """First prior of every sequence = T_init byte for byte; every later prior = compose_prior(previous result, delta)."""
    from dcreg_b200.api import compose_prior
    k = 0
    for s, seq in enumerate(seqs):
        assert res[k].T_prior.tobytes() == np.ascontiguousarray(T_init[s]).tobytes(), s
        for j in range(1, len(seq)):
            D = np.eye(4) if deltas is None else deltas[k + j - 1]
            assert res[k + j].T_prior.tobytes() == compose_prior(res[k + j - 1].T, D).tobytes(), (s, j)
        k += len(seq)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_one_frame_sequences_equal_scan_batch(ctx, scene, method):
    frames, _, T_init, tgt = scene
    prm = params(method)
    ctx.set_target(tgt, RADIUS)
    scans = ctx.icp_run_scans(prm, frames, T_init, want_log=True, want_cov=True)
    seqs = ctx.icp_run_sequences(prm, [[f] for f in frames], T_init, want_log=True, want_cov=True)
    assert len(seqs) == len(frames)
    for k, (a, b) in enumerate(zip(seqs, scans)):
        assert (a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged), k
        assert a.T.tobytes() == b.T.tobytes(), k
        assert a.cov.tobytes() == b.cov.tobytes(), k
        assert a.T_prior.tobytes() == np.ascontiguousarray(T_init[k]).tobytes(), k
        assert [np.array(L.H27).tobytes() for L in a.logs] == [np.array(L.H27).tobytes() for L in b.logs], k


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_chained_frames_equal_their_own_runs(ctx, chain, method):
    """Ours advances the frame in the loop kernel's folded step; ME-TSVD in the separate solve kernel (k2_step_kernel)."""
    seqs, frames, T_init, deltas, _, tgt = chain
    prm = params(method)
    ctx.set_target(tgt, RADIUS)
    res = ctx.icp_run_sequences(prm, seqs, T_init, deltas, want_log=True)
    assert len(res) == len(frames) == 32
    assert_chained_priors(res, seqs, T_init, deltas)
    for k, (f, r) in enumerate(zip(frames, res)):
        ctx.set_source(f)
        assert_same_run(r, ctx.icp_run(prm, r.T_prior))
    assert sum(r.converged for r in res) >= 24


def test_chained_frames_match_oracle(ctx, chain):
    import dcreg_oracle_c as oc
    seqs, frames, T_init, deltas, _, tgt = chain
    ctx.set_target(tgt, RADIUS)
    res = ctx.icp_run_sequences(params(), seqs, T_init, deltas, want_log=True)
    cp = oc.make_params(search_radius=RADIUS, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    for k in (9, 16, 23, 31):                               # frames deep in the 24-frame sequence
        b = res[k]
        sc = oc.Scene(frames[k], tgt)
        st, conv, n_it, Tc, clogs = sc.icp_run(cp, b.T_prior)
        sc.close()
        assert (b.status, b.converged, b.iterations) == (st, conv, n_it), k
        for Cl, G in zip(clogs, b.logs):
            assert G.n_effective == Cl.n_eff and G.n_corr_pt == Cl.n_pt
            assert list(G.analysis.degenerate_mask) == list(Cl.mask)
            assert np.allclose(G.analysis.np("lambda_schur_rot"), Cl.lam_schur_rot, rtol=1e-8)
            assert np.allclose(G.analysis.np("lambda_schur_trans"), Cl.lam_schur_trans, rtol=1e-8)
        assert o.se3_log_distance(Tc, b.T) < 1e-6, k


def test_abort_does_not_stop_the_sequence(ctx, chain):
    """A 5-point frame aborts with NOT_ENOUGH_POINTS after one iteration and returns its prior; the frame after it starts
    from that pose composed with the increment and runs as its own run would."""
    from dcreg_b200 import api
    _, frames, T_init, deltas, _, tgt = chain
    seq = [frames[8], frames[9], frames[10][:5], frames[11], frames[12]]
    d = deltas[8:13]
    prm = params()
    ctx.set_target(tgt, RADIUS)
    res = ctx.icp_run_sequences(prm, [seq], T_init[2:3], d, want_log=True)
    assert res[2].status == api.NOT_ENOUGH_POINTS and res[2].iterations == 1 and not res[2].converged
    assert res[2].T.tobytes() == res[2].T_prior.tobytes()
    assert res[3].T_prior.tobytes() == api.compose_prior(res[2].T, d[2]).tobytes()
    assert_chained_priors(res, [seq], T_init[2:3], d)
    for f, r in zip(seq, res):
        ctx.set_source(f)
        assert_same_run(r, ctx.icp_run(prm, r.T_prior))


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_fixed_iterations_run_every_frame_to_the_cap(ctx, chain, method):
    seqs, frames, T_init, deltas, _, tgt = chain
    prm = params(method, fixed_iterations=1, max_iterations=5)
    ctx.set_target(tgt, RADIUS)
    res = ctx.icp_run_sequences(prm, seqs, T_init, deltas)
    assert len(res) == len(frames)
    assert all(r.iterations == 5 and r.status == 0 and not r.converged for r in res)
    assert_chained_priors(res, seqs, T_init, deltas)


def test_identity_increments(ctx, chain):
    """deltas = None: every frame starts from the previous frame's result (the constant-position model)."""
    seqs, frames, T_init, _, _, tgt = chain
    ctx.set_target(tgt, RADIUS)
    short = [s[:3] for s in seqs]
    res = ctx.icp_run_sequences(params(), short, T_init)
    assert_chained_priors(res, short, T_init, None)


def test_sequences_reproducible_and_context_intact(ctx, scene, chain):
    seqs, _, T_init, deltas, _, tgt = chain
    frames16, _, T16, _ = scene
    prm = params()
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(frames16[0])
    one = ctx.icp_run(prm, T16[0])
    sb1 = ctx.icp_run_scans(prm, frames16[:6], T16[:6], want_log=True)
    a = ctx.icp_run_sequences(prm, seqs, T_init, deltas, want_log=True)
    b = ctx.icp_run_sequences(prm, seqs, T_init, deltas, want_log=True)
    for x, y in zip(a, b):                                  # two identical calls: identical bits
        assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
        assert x.T.tobytes() == y.T.tobytes() and x.T_prior.tobytes() == y.T_prior.tobytes()
        assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]
    again = ctx.icp_run(prm, T16[0])                        # the context's source and its sort are untouched
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]
    sb2 = ctx.icp_run_scans(prm, frames16[:6], T16[:6], want_log=True)
    for x, y in zip(sb1, sb2):
        assert x.T.tobytes() == y.T.tobytes() and x.iterations == y.iterations
        assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]


def test_sequences_bad_arguments(ctx, chain, cylinder):
    from dcreg_b200 import api
    _, frames, T_init, deltas, _, tgt = chain
    prm = params()
    ctx.set_target(tgt, RADIUS)
    lib, h = ctx.lib, ctx._h
    fr = frames[:4]
    xyz = np.ascontiguousarray(np.concatenate(fr), dtype=np.float32)
    off = np.zeros(5, dtype=np.int64)
    off[1:] = np.cumsum([len(f) for f in fr])
    so = np.array([0, 1, 4], dtype=np.int32)
    T = np.ascontiguousarray(T_init[:2])
    D = np.ascontiguousarray(deltas[:4])
    dp = C.POINTER(C.c_double)

    def call(n_seqs=2, seq_off=so, n_frames=4, pts=xyz, offsets=off, params=prm, handle=h, T0=T, Tout=None):
        Tout = np.empty((max(n_frames, 1), 4, 4)) if Tout is None else Tout
        Dd = D if n_frames == 4 else np.ascontiguousarray(np.broadcast_to(np.eye(4), (max(n_frames, 1), 4, 4)))
        return lib.dcreg_icp_run_sequences(handle, C.byref(params), n_seqs, seq_off.ctypes.data_as(C.POINTER(C.c_int)),
                                           n_frames, pts.ctypes.data_as(C.POINTER(C.c_float)),
                                           offsets.ctypes.data_as(C.POINTER(C.c_int64)), 3, T0.ctypes.data_as(dp),
                                           Dd.ctypes.data_as(dp), None, Tout.ctypes.data_as(dp), None, None, None, None,
                                           None, 0)

    assert call() == api.OK
    bad = [dict(n_seqs=0), dict(n_seqs=-1),
           dict(seq_off=np.array([0, 3, 2], np.int32)),                                 # not ascending
           dict(seq_off=np.array([0, 0, 4], np.int32)),                                 # an empty sequence
           dict(seq_off=np.array([1, 2, 4], np.int32)),                                 # not from 0
           dict(seq_off=np.array([0, 1, 3], np.int32)),                                 # seq_offsets[n_seqs] != n_frames
           dict(offsets=np.array([0, off[1], off[1], off[3], off[4]], np.int64)),       # an empty frame
           dict(params=params(max_iterations=0)), dict(params=params(max_iterations=-1)),
           dict(params=params(weight_gate=1.5))]
    for kw in bad:
        assert call(**kw) == api.BAD_ARG, kw
        assert lib.dcreg_last_error(h).decode(), kw
    # more frames than the loop's per-frame kernels hold (65535): rejected before anything is launched
    n_big = 65536
    big = dict(n_seqs=1, seq_off=np.array([0, n_big], np.int32), n_frames=n_big, pts=np.zeros((n_big, 3), np.float32),
               offsets=np.arange(n_big + 1, dtype=np.int64), T0=np.ascontiguousarray(np.eye(4)[None]))
    launches = ctx.launch_count
    assert call(**big) == api.BAD_ARG
    assert ctx.launch_count == launches
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_sequences(prm, [], np.zeros((0, 4, 4)))
    assert e.value.status == api.BAD_ARG
    # a target too large for a dense grid at this cell size: a sparse row index, which the call runs on
    far = np.concatenate([cylinder, cylinder + np.float32(4.0e4)])
    ctx.set_target(far, RADIUS)
    assert call() == api.OK
    # no target at all; a sharded context (a one-rank communicator)
    from dcreg_b200 import Context
    with Context(0) as fresh:
        assert call(handle=fresh._h) == api.BAD_ARG
        fresh.set_target(tgt, RADIUS)
        assert call(handle=fresh._h) == api.OK
        try:
            fresh.comm_init(fresh.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        assert call(handle=fresh._h) == api.BAD_ARG
        assert "rank" in lib.dcreg_last_error(fresh._h).decode()
