"""dcreg_icp_run_pairs: many scan/target pairs, each source against its own target, in one batched call.

Every pair of a batch must be the registration dcreg_set_target(target) + dcreg_set_source(source) + dcreg_icp_run would
give: status, iteration counts, flags, per-iteration counts and masks identical, sums / steps / poses equal to the
rounding of FP64 sums grouped differently.  With one shared map as every target it must be bit-identical to
dcreg_icp_run_scans against that map (dcreg_set_target builds its grid with the same arena code, as one cloud).  A batch reproduces bit for
bit, leaves the context's own clouds alone, and its per-pair covariance and point-to-point metrics equal the single calls'.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o
from harness import RADIUS, assert_same_run, ctx, params, rel_err  # noqa: F401

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def scene():
    """16 scan-to-submap pairs: sources cut to ragged sizes from 40 to 8 000 points; targets from a full ~100 k-point
    submap down to a few thousand points, some cropped to a smaller box."""
    from dcreg_b200.scenes import make_parking_pairs
    src, tgt, T_true, T_init = make_parking_pairs(16, seed=55, n_scan=8_400)
    sizes = [6_000, 40, 8_000, 5_120, 300, 7_311, 2_500, 6_666, 999, 4_097, 7_800, 3_333, 256, 5_555, 7_001, 1_234]
    keep = [1.0, 0.05, 0.3, 1.0, 0.5, 0.04, 1.0, 0.2, 1.0, 0.6, 0.1, 1.0, 0.8, 0.07, 1.0, 0.4]
    rng = np.random.default_rng(56)
    src = [s[np.sort(rng.choice(len(s), size=n, replace=False))] for s, n in zip(src, sizes)]
    cut = []
    for k, (t, p) in enumerate(zip(tgt, keep)):
        t = t[rng.random(len(t)) < p]
        if k % 3 == 1:                                      # a smaller box around the sensor
            t = t[(np.abs(t[:, 0]) < 18.0) & (np.abs(t[:, 1]) < 12.0)]
        cut.append(np.ascontiguousarray(t))
    return src, cut, T_true, T_init


def single_run(ctx, prm, s, t, T, cell=RADIUS, **kw):
    ctx.set_target(t, cell)
    ctx.set_source(s)
    return ctx.icp_run(prm, T, **kw)


def same_bits(x, y):
    return ((x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged) and x.T.tobytes() == y.T.tobytes()
            and [np.array(L.H27).tobytes() for L in x.logs] == [np.array(L.H27).tobytes() for L in y.logs])


@pytest.mark.parametrize("method,cell", [pytest.param(m, c, id=m if c == RADIUS else f"{m}-cell{c}")
                                         for c in (RADIUS, RADIUS / 2) for m in ("Ours", "ME-TSVD")])
def test_pairs_equal_single_runs(ctx, scene, method, cell):
    """Ours folds the solve step into the loop kernel; ME-TSVD takes the separate solve kernel (k2_step_kernel).
    cell = RADIUS / 2: the targets' grids searched over 2 rings of cells."""
    src, tgt, _, T_init = scene
    assert min(len(t) for t in tgt) < 5_000 and max(len(t) for t in tgt) > 80_000
    prm = params(method)
    batch = ctx.icp_run_pairs(prm, src, tgt, T_init, cell_size=cell, want_log=True)
    assert len(batch) == len(src)
    n_conv = 0
    for k, b in enumerate(batch):
        assert_same_run(b, single_run(ctx, prm, src[k], tgt[k], T_init[k], cell=cell))
        n_conv += int(b.converged)
    assert n_conv >= 10                                     # the pairs stop on their own convergence tests


def test_pairs_shared_map_bit_identical_to_scans(ctx):
    """Every target is the same map: bit for bit what icp_run_scans gives after set_target(map)."""
    from dcreg_b200.scenes import make_parking_frames
    frames, _, T_init, park_map = make_parking_frames(6, seed=57, n_map=200_000, n_scan=3_000)
    prm = params()
    pairs = ctx.icp_run_pairs(prm, frames, [park_map] * len(frames), T_init, want_log=True)
    ctx.set_target(park_map, RADIUS)
    scans = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    for p, s in zip(pairs, scans):
        assert same_bits(p, s)
        assert [(L.n_effective, L.n_corr_pt) for L in p.logs] == [(L.n_effective, L.n_corr_pt) for L in s.logs]


def test_pairs_match_oracle(ctx, scene):
    import dcreg_oracle_c as oc
    src, tgt, _, T_init = scene
    pick = [0, 3, 5, 7, 9, 14]                              # 6 pairs of 4 k - 8 k source points
    batch = ctx.icp_run_pairs(params(), [src[k] for k in pick], [tgt[k] for k in pick], T_init[pick], want_log=True)
    cp = oc.make_params(search_radius=RADIUS, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    for b, k in zip(batch, pick):
        sc = oc.Scene(src[k], tgt[k])
        st, conv, n_it, Tc, clogs = sc.icp_run(cp, T_init[k])
        sc.close()
        assert (b.status, b.converged, b.iterations) == (st, conv, n_it), k
        for Cl, G in zip(clogs, b.logs):
            assert G.n_effective == Cl.n_eff and G.n_corr_pt == Cl.n_pt
            assert list(G.analysis.degenerate_mask) == list(Cl.mask)
            assert np.allclose(G.analysis.np("lambda_schur_rot"), Cl.lam_schur_rot, rtol=1e-8)
            assert np.allclose(G.analysis.np("lambda_schur_trans"), Cl.lam_schur_trans, rtol=1e-8)
        assert o.se3_log_distance(Tc, b.T) < 1e-6, k


def test_pairs_reproducible_and_context_intact(ctx, scene, cylinder):
    from dcreg_b200 import Context
    from dcreg_b200.scenes import g2_initial_pose, make_parking_frames
    src, tgt, _, T_init = scene
    frames, _, Tf, park_map = make_parking_frames(4, seed=58, n_map=200_000, n_scan=3_000)
    prm = params()
    ctx.set_target(park_map, RADIUS)
    ctx.set_source(frames[0])
    one = ctx.icp_run(prm, Tf[0])
    tb1 = ctx.icp_run_batch(prm, Tf)
    sc1 = ctx.icp_run_scans(prm, frames, Tf, want_log=True)
    a = ctx.icp_run_pairs(prm, src, tgt, T_init, want_log=True, want_cov=True, metrics_threshold=0.5)
    b = ctx.icp_run_pairs(prm, src, tgt, T_init, want_log=True, want_cov=True, metrics_threshold=0.5)
    for x, y in zip(a, b):                                  # two identical calls: identical bits
        assert same_bits(x, y)
        assert x.cov.tobytes() == y.cov.tobytes() and x.metrics == y.metrics
    again = ctx.icp_run(prm, Tf[0])                         # the context's source, target and grid are untouched
    assert same_bits(again, one)
    tb2 = ctx.icp_run_batch(prm, Tf)
    assert all(x.T.tobytes() == y.T.tobytes() and x.iterations == y.iterations for x, y in zip(tb1, tb2))
    sc2 = ctx.icp_run_scans(prm, frames, Tf, want_log=True)
    assert all(same_bits(x, y) for x, y in zip(sc1, sc2))
    # a smaller call after the large one: the grown arenas do not leak into it
    small = ([cylinder[:3000], cylinder[3000:]], [cylinder, cylinder[::2]], [g2_initial_pose()] * 2)
    p1 = params(search_radius=1.0)
    r1 = ctx.icp_run_pairs(p1, *small, want_log=True, metrics_threshold=1.0)
    with Context(0) as fresh:
        r2 = fresh.icp_run_pairs(p1, *small, want_log=True, metrics_threshold=1.0)
    for x, y in zip(r1, r2):
        assert same_bits(x, y) and x.metrics == y.metrics


def test_pairs_mixed_outcomes(ctx, scene):
    """One pair starts 500 m away: NOT_ENOUGH_POINTS after one iteration with its pose untouched, as dcreg_icp_run
    returns it; its neighbours still equal their single runs."""
    from dcreg_b200 import api
    src, tgt, _, T_init = scene
    prm = params()
    Ts = T_init[:5].copy()
    Ts[2] = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)
    batch = ctx.icp_run_pairs(prm, src[:5], tgt[:5], Ts, want_log=True)
    assert batch[2].status == api.NOT_ENOUGH_POINTS and batch[2].iterations == 1 and not batch[2].converged
    assert np.array_equal(batch[2].T, Ts[2])
    for k in range(5):
        assert_same_run(batch[k], single_run(ctx, prm, src[k], tgt[k], Ts[k]))


def test_pairs_covariance(ctx, scene):
    src, tgt, _, T_init = scene
    prm = params()
    Ts = T_init[:6].copy()
    Ts[4] = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)        # not converged: 1e6 I
    batch = ctx.icp_run_pairs(prm, src[:6], tgt[:6], Ts, want_cov=True)
    assert sum(b.converged for b in batch) >= 4
    for k, b in enumerate(batch):
        single = single_run(ctx, prm, src[k], tgt[k], Ts[k], want_log=False)
        ref = ctx.last_covariance()
        assert b.cov.shape == (6, 6) and b.converged == single.converged
        if b.converged:
            assert rel_err(b.cov, ref) < 1e-6, k
        else:
            assert np.array_equal(b.cov, 1e6 * np.eye(6)) and np.array_equal(ref, 1e6 * np.eye(6)), k


@pytest.mark.parametrize("threshold", [0.5, 0.05])
def test_pairs_metrics(ctx, scene, threshold):
    src, tgt, _, T_init = scene
    batch = ctx.icp_run_pairs(params(), src, tgt, T_init, metrics_threshold=threshold)
    for k, b in enumerate(batch):
        ctx.set_target(tgt[k], RADIUS)
        ctx.set_source(src[k])
        ref = ctx.point_to_point_metrics(b.T, threshold)
        assert b.metrics["n_valid"] == ref["n_valid"], k
        for key in ("rmse", "fitness", "chamfer"):
            assert abs(b.metrics[key] - ref[key]) <= 1e-12 * max(abs(ref[key]), 1e-300), (k, key)


def test_pairs_launch_count_does_not_grow(ctx, scene):
    src, tgt, _, T_init = scene
    prm = params(max_iterations=3, fixed_iterations=1)
    deltas = []
    for n in (2, 16, 2):
        l0 = ctx.launch_count
        ctx.icp_run_pairs(prm, src[:n], tgt[:n], T_init[:n], want_cov=True, metrics_threshold=0.5)
        deltas.append(ctx.launch_count - l0)
    assert deltas[0] == deltas[1] == deltas[2], deltas


def test_pairs_bad_arguments(ctx, scene, cylinder):
    from dcreg_b200 import api
    src, tgt, _, T_init = scene
    prm = params()
    lib, h = ctx.lib, ctx._h
    xs = np.ascontiguousarray(np.concatenate(src[:3]), dtype=np.float32)
    xt = np.ascontiguousarray(np.concatenate(tgt[:3]), dtype=np.float32)
    offs = np.array([0, len(src[0]), len(src[0]) + len(src[1]), len(xs)], dtype=np.int64)
    offt = np.array([0, len(tgt[0]), len(tgt[0]) + len(tgt[1]), len(xt)], dtype=np.int64)
    T = np.ascontiguousarray(T_init[:3])
    T_out = np.empty((3, 4, 4))
    fp, ip, dp = C.POINTER(C.c_float), C.POINTER(C.c_int64), C.POINTER(C.c_double)

    def call(n=3, s=xs, so=offs, t=xt, to=offt, stride=3, cell=RADIUS, T0=T, Tout=T_out, params=prm, handle=h):
        def ptr(a, typ):
            return a.ctypes.data_as(typ) if a is not None else None
        return lib.dcreg_icp_run_pairs(handle, C.byref(params), n, ptr(s, fp), ptr(so, ip), ptr(t, fp), ptr(to, ip), stride,
                                       cell, ptr(T0, dp), ptr(Tout, dp), None, None, None, None, 0.0, None, None, 0)

    assert call() == api.OK
    huge = 2 ** 29                                          # one more than the 2^29 - 1 points a side may have
    bad = [dict(n=0), dict(n=-2), dict(s=None), dict(so=None), dict(t=None), dict(to=None), dict(T0=None), dict(Tout=None),
           dict(n=65536), dict(stride=2), dict(cell=0.0), dict(cell=-1.0),
           dict(cell=0.1),                                                                           # radius / cell > 4
           dict(so=np.array([1, 10, 20, 30], np.int64)), dict(so=np.array([0, 100, 50, len(xs)], np.int64)),
           dict(so=np.array([0, 100, 100, len(xs)], np.int64)),
           dict(to=np.array([2, 10, 20, 30], np.int64)), dict(to=np.array([0, 100, 50, len(xt)], np.int64)),
           dict(to=np.array([0, 100, 100, len(xt)], np.int64)),
           dict(n=1, so=np.array([0, huge], np.int64)), dict(n=1, to=np.array([0, huge], np.int64)),   # int32 totals
           dict(params=params(weight_gate=1.5)), dict(params=params(max_iterations=-1))]      # check_run_args
    for kw in bad:
        assert call(**kw) == api.BAD_ARG, kw
        assert lib.dcreg_last_error(h).decode(), kw
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_pairs(prm, [], [], np.zeros((0, 4, 4)))
    assert e.value.status == api.BAD_ARG
    # a target whose box is too large for a dense grid; coordinates outside +-2^19 cells
    far = np.ascontiguousarray(np.concatenate([cylinder, cylinder + np.float32(4.0e4)]))
    one = np.array([0, len(src[0])], np.int64)
    for t, word in ((far, "dense"), (np.ascontiguousarray(cylinder + np.float32(1.0e6)), "2^19")):
        assert call(n=1, so=one, t=t, to=np.array([0, len(t)], np.int64)) == api.BAD_ARG
        assert word in lib.dcreg_last_error(h).decode()
    assert call() == api.OK                                 # and the context is still usable
    # no set_target / set_source needed; a sharded context (a one-rank communicator) is refused
    from dcreg_b200 import Context
    with Context(0) as fresh:
        assert call(handle=fresh._h, Tout=np.empty((3, 4, 4))) == api.OK
        try:
            fresh.comm_init(fresh.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        assert call(handle=fresh._h) == api.BAD_ARG
        assert "rank" in lib.dcreg_last_error(fresh._h).decode()
