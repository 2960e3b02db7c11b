"""dcreg_icp_run_scans: many different scans (C3-shaped LiDAR frames) against one map in one batched call.

Every scan of a batch must be the registration dcreg_set_source(scan) + dcreg_icp_run would give: status, iteration
counts, flags, per-iteration counts and masks identical, sums / steps / poses equal to the rounding of FP64 sums grouped
differently (the same tolerances as the same-source trial batches, tests/test_gpu_configs.py).  A batch reproduces bit for
bit and leaves the context's own source, and what single runs and trial batches compute from it, untouched.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o
from harness import RADIUS, assert_same_run, ctx, params, rel_err  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    """16 frames along a path through the 0.5 M-point parking map, cut to ragged sizes from 40 to 8 000 points: one below
    a single 256-slot tile, one of exactly 20 tiles."""
    from dcreg_b200.scenes import make_parking_frames
    frames, T_true, T_init, tgt = make_parking_frames(16, seed=51, n_scan=8_400)
    sizes = [6_000, 40, 8_000, 5_120, 300, 7_311, 2_500, 6_666, 999, 4_097, 7_800, 3_333, 256, 5_555, 7_001, 1_234]
    rng = np.random.default_rng(52)
    cut = [f[np.sort(rng.choice(len(f), size=n, replace=False))] for f, n in zip(frames, sizes)]
    return cut, T_true, T_init, tgt


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_scans_equal_single_runs(ctx, scene, method):
    """Ours folds the solve step into the loop kernel; ME-TSVD takes the separate solve kernel (k2_step_kernel)."""
    frames, _, T_init, tgt = scene
    prm = params(method)
    ctx.set_target(tgt, RADIUS)
    batch = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    assert len(batch) == len(frames)
    n_conv = 0
    for k, (f, b) in enumerate(zip(frames, batch)):
        ctx.set_source(f)
        single = ctx.icp_run(prm, T_init[k])
        assert_same_run(b, single)
        n_conv += int(b.converged)
    assert n_conv >= 12                                     # the scans stop on their own convergence tests


def test_scans_match_oracle(ctx, scene):
    import dcreg_oracle_c as oc
    frames, _, T_init, tgt = scene
    pick = [0, 2, 3, 5, 7, 9, 10, 14]                       # 8 frames of 4 k - 8 k points
    ctx.set_target(tgt, RADIUS)
    batch = ctx.icp_run_scans(params(), [frames[k] for k in pick], T_init[pick], want_log=True)
    cp = oc.make_params(search_radius=RADIUS, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    for b, k in zip(batch, pick):
        sc = oc.Scene(frames[k], tgt)
        st, conv, n_it, Tc, clogs = sc.icp_run(cp, T_init[k])
        sc.close()
        assert (b.status, b.converged, b.iterations) == (st, conv, n_it), k
        for Cl, G in zip(clogs, b.logs):
            assert G.n_effective == Cl.n_eff and G.n_corr_pt == Cl.n_pt
            assert list(G.analysis.degenerate_mask) == list(Cl.mask)
            assert np.allclose(G.analysis.np("lambda_schur_rot"), Cl.lam_schur_rot, rtol=1e-8)
            assert np.allclose(G.analysis.np("lambda_schur_trans"), Cl.lam_schur_trans, rtol=1e-8)
        assert o.se3_log_distance(Tc, b.T) < 1e-6, k


def test_scans_reproducible_and_context_intact(ctx, scene, cylinder):
    frames, _, T_init, tgt = scene
    prm = params()
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(frames[0])
    one = ctx.icp_run(prm, T_init[0])
    trials = T_init[:5]
    tb1 = ctx.icp_run_batch(prm, trials)
    a = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    b = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    for x, y in zip(a, b):                                  # two identical calls: identical bits
        assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
        assert x.T.tobytes() == y.T.tobytes()
        assert [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs]
    again = ctx.icp_run(prm, T_init[0])                     # the context's source and its sort are untouched
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]
    tb2 = ctx.icp_run_batch(prm, trials)
    assert all(x.T.tobytes() == y.T.tobytes() and x.iterations == y.iterations for x, y in zip(tb1, tb2))
    # a different, smaller target and source afterwards: the scans' buffers do not leak into it
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    from dcreg_b200.scenes import g2_initial_pose
    r1 = ctx.icp_run(params(search_radius=1.0), g2_initial_pose())
    ctx.icp_run_scans(params(search_radius=1.0), [cylinder[:3000], cylinder[3000:]], [g2_initial_pose()] * 2)
    r2 = ctx.icp_run(params(search_radius=1.0), g2_initial_pose())
    assert r1.T.tobytes() == r2.T.tobytes()


def test_scans_mixed_outcomes(ctx, scene):
    """One scan starts 500 m away: NOT_ENOUGH_POINTS after one iteration with its pose untouched, as dcreg_icp_run
    returns it; its neighbours still equal their single runs."""
    from dcreg_b200 import api
    frames, _, T_init, tgt = scene
    prm = params()
    Ts = T_init[:5].copy()
    Ts[2] = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)
    ctx.set_target(tgt, RADIUS)
    batch = ctx.icp_run_scans(prm, frames[:5], Ts, want_log=True)
    assert batch[2].status == api.NOT_ENOUGH_POINTS and batch[2].iterations == 1 and not batch[2].converged
    assert np.array_equal(batch[2].T, Ts[2])
    for k in range(5):
        ctx.set_source(frames[k])
        assert_same_run(batch[k], ctx.icp_run(prm, Ts[k]))


def test_scans_covariance(ctx, scene):
    frames, _, T_init, tgt = scene
    prm = params()
    Ts = T_init[:6].copy()
    Ts[4] = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)        # not converged: 1e6 I
    ctx.set_target(tgt, RADIUS)
    batch = ctx.icp_run_scans(prm, frames[:6], Ts, want_cov=True)
    assert sum(b.converged for b in batch) >= 4
    for k, b in enumerate(batch):
        ctx.set_source(frames[k])
        single = ctx.icp_run(prm, Ts[k], want_log=False)
        ref = ctx.last_covariance()
        assert b.cov.shape == (6, 6) and b.converged == single.converged
        if b.converged:
            assert rel_err(b.cov, ref) < 1e-6, k
        else:
            assert np.array_equal(b.cov, 1e6 * np.eye(6)) and np.array_equal(ref, 1e6 * np.eye(6)), k


def test_scans_bad_arguments(ctx, scene, cylinder):
    from dcreg_b200 import api
    frames, _, T_init, tgt = scene
    prm = params()
    ctx.set_target(tgt, RADIUS)
    lib, h = ctx.lib, ctx._h
    xyz = np.ascontiguousarray(np.concatenate(frames[:3]), dtype=np.float32)
    off = np.array([0, len(frames[0]), len(frames[0]) + len(frames[1]), len(xyz)], dtype=np.int64)
    T = np.ascontiguousarray(T_init[:3])
    T_out = np.empty((3, 4, 4))

    def call(n=3, pts=xyz, offsets=off, stride=3, T0=T, Tout=T_out, params=prm, handle=h):
        fp = pts.ctypes.data_as(C.POINTER(C.c_float)) if pts is not None else None
        op = offsets.ctypes.data_as(C.POINTER(C.c_int64)) if offsets is not None else None
        dp = C.POINTER(C.c_double)
        return lib.dcreg_icp_run_scans(handle, C.byref(params), n, fp, op, stride,
                                       T0.ctypes.data_as(dp) if T0 is not None else None,
                                       Tout.ctypes.data_as(dp) if Tout is not None else None,
                                       None, None, None, None, None, 0)

    assert call() == api.OK
    bad = [dict(n=0), dict(n=-2), dict(pts=None), dict(offsets=None), dict(T0=None), dict(Tout=None), dict(stride=2),
           dict(offsets=np.array([1, 10, 20, 30], np.int64)),                                   # not from 0
           dict(offsets=np.array([0, 100, 50, len(xyz)], np.int64)),                            # descending
           dict(offsets=np.array([0, 100, 100, len(xyz)], np.int64)),                           # an empty scan
           dict(params=params(weight_gate=1.5)), dict(params=params(max_iterations=-1))]  # check_run_args
    for kw in bad:
        assert call(**kw) == api.BAD_ARG, kw
        assert lib.dcreg_last_error(h).decode(), kw
    # more scans than the loop kernel's grid y holds (65535): rejected before anything is launched
    n_big = 65536
    big = dict(n=n_big, pts=np.zeros((n_big, 3), np.float32), offsets=np.arange(n_big + 1, dtype=np.int64),
               T0=np.ascontiguousarray(np.broadcast_to(np.eye(4), (n_big, 4, 4))), Tout=np.empty((n_big, 4, 4)))
    launches = ctx.launch_count
    assert call(**big) == api.BAD_ARG
    assert ctx.launch_count == launches
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_scans(prm, [], np.zeros((0, 4, 4)))
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
        assert call(handle=fresh._h, Tout=np.empty((3, 4, 4))) == api.OK
        try:
            fresh.comm_init(fresh.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        assert call(handle=fresh._h) == api.BAD_ARG
        assert "ranks" in lib.dcreg_last_error(fresh._h).decode()
