"""GPU parity on BASELINE.json's own configurations and on the round-2 entry points, through the C ABI.

  C2  100 k-point cylinder, 50 fixed iterations, weight derivative off  - exactly what bench.py times
  C4  10 M-slot corridor: the K1 sums against the NumPy oracle; a 1 M-point corridor registration against the C oracle
  C5  batched trials (dcreg_icp_run_batch): equal to one dcreg_icp_run per trial (counts and flags exactly, poses to 1e-8), and against the C oracle
plus: EVD_SUB_CONDITION, the covariance branches, weight_slope / weight_gate, iter_time_ms, host-plane fitness.

Tolerances as in test_gpu_parity.py: pose 1e-6 on the SE(3) log, sums 1e-11 relative, integers identical.
"""
import math
import os

import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_c as oc
from harness import ctx, rel_err  # noqa: F401

pytestmark = pytest.mark.gpu


def host_threads():
    return max(1, min(32, len(os.sched_getaffinity(0))))


# ------------------------------------------------------------------------------------------------
# C2 exactly as benchmarked
# ------------------------------------------------------------------------------------------------
def test_c2_as_benchmarked_matches_oracle_every_iteration(ctx):
    """bench.py's step: 100 k-point synthetic cylinder, published perturbation, Ours, kappa 10, weight derivative
    off, 50 FIXED iterations.  Counts identical in every iteration, pose 1e-6 at the end and along the way."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import make_cylinder, g2_initial_pose
    pts = make_cylinder(100_000, seed=42)
    T0 = g2_initial_pose()
    sc = oc.Scene(pts, pts)
    prm_c = oc.make_params(max_iterations=50, fixed_iterations=True, kappa_target=10.0, use_weight_derivative=False,
                           n_threads=host_threads())
    st, conv, n_it, T_ref, logs = sc.icp_run(prm_c, T0, want_log=True)
    assert st == 0 and n_it == 50
    gp = default_params(search_radius=1.0, max_iterations=50, fixed_iterations=1, kappa_target=10.0, cond_thresh=10.0,
                        use_weight_derivative=0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    res = ctx.icp_run(gp, T0)
    assert res.status == 0 and res.iterations == 50 and len(res.logs) == 50
    for k, (a, b) in enumerate(zip(res.logs, logs)):
        assert a.n_effective == b.n_eff and a.n_corr_pt == b.n_pt, k
        assert list(a.analysis.degenerate_mask) == list(b.mask), k
        assert o.se3_log_distance(np.array(b.T).reshape(4, 4), np.array(a.T).reshape(4, 4)) < 1e-6, k
        assert rel_err(a.analysis.lambda_schur_rot, b.lam_schur_rot) < 1e-8, k
        assert rel_err(a.analysis.lambda_schur_trans, b.lam_schur_trans) < 1e-8, k
        assert a.iter_time_ms > 0.0
    assert o.se3_log_distance(T_ref, res.T) < 1e-6
    # a second run on the same context (graph replay, records of the previous run discarded) gives the same bits
    res2 = ctx.icp_run(gp, T0)
    assert np.array_equal(res2.T, res.T)
    # ... and so do runs queued back to back without any host synchronisation (dcreg_icp_enqueue / dcreg_icp_fetch)
    ctx.icp_enqueue(gp, T0)
    ctx.icp_enqueue(gp, T0)
    res3 = ctx.icp_fetch()
    assert res3.status == 0 and res3.iterations == 50 and np.array_equal(res3.T, res.T)
    sc.close()


# ------------------------------------------------------------------------------------------------
# C4: the 10 M-slot reduction and a corridor registration
# ------------------------------------------------------------------------------------------------
def test_c4_k1_sums_at_10m_slots_match_oracle(ctx):
    """bench.py's roofline workload: 10 M-slot corridor, planes from the device correspondence stage frozen as
    float4, K1 against the NumPy oracle on the very same (point, plane) slots, chunked."""
    from dcreg_b200.scenes import make_corridor
    n = 10_000_000
    scene = make_corridor(n, seed=44, noise=0.002)
    Tc = np.eye(4); Tc[:3, 3] = [0.004, 0.003, -0.002]
    ctx.set_target(scene, 0.05)
    ctx.set_source(scene)
    planes, npt = ctx.find_planes(Tc, 0.05, want_planes=True)
    ctx.freeze_planes_f32()
    planes32 = planes.astype(np.float32)
    for use_wd in (False, True):
        out, stats = ctx.reduce_device(False, Tc, use_wd)
        ref = np.zeros(27); rstats = np.zeros(3)
        step = 1_000_000
        for lo in range(0, n, step):
            src4 = np.concatenate([scene[lo:lo + step], np.zeros((min(step, n - lo), 1), np.float32)], axis=1)
            r27, rs = o.reduce_normal_equations(src4, planes32[lo:lo + step], Tc[:3, :3], Tc[:3, 3], use_wd)
            ref += r27; rstats += rs
        assert rel_err(out, ref) < 1e-11
        assert int(stats[1]) == int(rstats[1]) and int(stats[2]) == int(rstats[2])
        assert abs(stats[0] - rstats[0]) <= 1e-11 * abs(rstats[0])
        assert stats[1] > 0.5 * n            # the corridor really yields correspondences nearly everywhere


def test_c4_corridor_icp_1m_points_matches_oracle(ctx):
    """A 1 M-point corridor registration (degenerate scene) against the C oracle: counts, mask, pose."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import make_corridor
    n = 1_000_000
    pts = make_corridor(n, seed=44, noise=0.002)
    T0 = np.eye(4); T0[:3, 3] = [0.02, 0.015, -0.01]
    c, s = math.cos(0.002), math.sin(0.002)
    T0[:3, :3] = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]])
    radius = 0.1
    sc = oc.Scene(pts, pts)
    prm_c = oc.make_params(search_radius=radius, max_iterations=8, fixed_iterations=True, kappa_target=10.0,
                           n_threads=host_threads())
    st, conv, n_it, T_ref, logs = sc.icp_run(prm_c, T0, want_log=True)
    assert st == 0 and n_it == 8
    gp = default_params(search_radius=radius, max_iterations=8, fixed_iterations=1, kappa_target=10.0)
    ctx.set_target(pts, radius)
    ctx.set_source(pts)
    res = ctx.icp_run(gp, T0)
    assert res.iterations == 8
    for k, (a, b) in enumerate(zip(res.logs, logs)):
        assert a.n_effective == b.n_eff and a.n_corr_pt == b.n_pt, k
        assert list(a.analysis.degenerate_mask) == list(b.mask), k
    assert o.se3_log_distance(T_ref, res.T) < 1e-6
    assert all(L.analysis.is_degenerate for L in res.logs)            # a corridor is degenerate in every iteration
    sc.close()


# ------------------------------------------------------------------------------------------------
# C5: batched trials
# ------------------------------------------------------------------------------------------------
def perturbations(n, seed=45):
    rng = np.random.default_rng(seed)
    Ts = []
    for _ in range(n):
        t = rng.uniform(-1.0, 1.0, 3)
        rpy = np.deg2rad(rng.uniform(-3.0, 3.0, 3))
        Ts.append(o.pose6d_to_matrix(t[0], t[1], t[2], rpy[0], rpy[1], rpy[2]))
    return np.array(Ts)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_batched_trials_equal_single_runs(ctx, cylinder, method):
    """dcreg_icp_run_batch (icp_test_runner.cpp:331-345 side by side): every trial runs the same kernels as a
    dcreg_icp_run from the same initial pose - iteration counts, flags, per-iteration counts and masks identical, poses
    equal to summation-order rounding (the source is sorted by target cell under the FIRST trial's pose, and a single run
    of a small cloud cuts it into smaller tiles than a batch does: the partial sums are grouped differently)."""
    from dcreg_b200 import default_params
    det, hand = ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG") if method == "Ours" else ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD")
    gp = default_params(kappa_target=10.0, max_iterations=30, detection=det, handling=hand)
    Ts = perturbations(24)
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    batch = ctx.icp_run_batch(gp, Ts, want_log=True)
    again = ctx.icp_run_batch(gp, Ts)
    assert len(batch) == 24
    n_conv = 0
    for t, (b, T0) in enumerate(zip(batch, Ts)):
        single = ctx.icp_run(gp, T0)
        assert b.status == single.status and b.iterations == single.iterations and b.converged == single.converged
        assert np.array_equal(b.T, again[t].T)                                # a batch is reproducible bit for bit
        assert o.se3_log_distance(single.T, b.T) < 1e-8       # rounding of the sums, amplified by up to 30 PCG-stopped iterations
        assert len(b.logs) == len(single.logs)
        for x, y in zip(b.logs, single.logs):
            assert x.n_effective == y.n_effective and x.n_corr_pt == y.n_corr_pt
            assert rel_err(np.array(x.H27), np.array(y.H27)) < 1e-8 and np.max(np.abs(np.array(x.dx) - np.array(y.dx))) < 1e-8
            assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)
        n_conv += int(b.converged)
    assert n_conv >= 12                      # trials stop on their own convergence test


def test_batched_trials_match_oracle(ctx, cylinder):
    """A 64-trial perturbation Monte-Carlo of the shipped cylinder against the C oracle, trial by trial."""
    from dcreg_b200 import default_params
    gp = default_params(kappa_target=10.0, max_iterations=30)
    Ts = perturbations(64, seed=46)
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    batch = ctx.icp_run_batch(gp, Ts)
    sc = oc.Scene(cylinder, cylinder)
    prm_c = oc.make_params(max_iterations=30, kappa_target=10.0, n_threads=host_threads())
    worst = 0.0
    for b, T0 in zip(batch, Ts):
        st, conv, n_it, T_ref, _ = sc.icp_run(prm_c, T0, want_log=False)
        assert b.status == st and b.iterations == n_it and b.converged == conv
        worst = max(worst, o.se3_log_distance(T_ref, b.T))
    assert worst < 1e-6
    sc.close()


def test_batch_bad_arguments(ctx, cylinder):
    from dcreg_b200 import default_params
    from dcreg_b200.api import BAD_ARG, DcregError
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    with pytest.raises(DcregError):
        ctx.icp_run_batch(default_params(weight_gate=1.5), perturbations(2))
    # more trials than the loop kernel's grid y holds (65535): rejected before anything is launched
    launches = ctx.launch_count
    with pytest.raises(DcregError) as e:
        ctx.icp_run_batch(default_params(), np.broadcast_to(np.eye(4), (65536, 4, 4)))
    assert e.value.status == BAD_ARG and ctx.launch_count == launches
    res = ctx.icp_run_batch(default_params(max_iterations=0), perturbations(3))
    assert all(r.iterations == 0 and not r.converged for r in res)


# ------------------------------------------------------------------------------------------------
# EVD_SUB_CONDITION, covariance branches, weight parameters, host-plane fitness
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("handling", ["SOLUTION_REMAPPING", "STANDARD_REGULARIZATION"])
def test_evd_sub_condition_detection(ctx, cylinder, handling):
    """dcreg.hpp:112-126: the released code tests cond_diag_* it never fills (NaN), so nothing is ever flagged and
    every handler falls through to the plain QR solve - the trajectory equals NONE_DETE's and the oracle's."""
    from dcreg_b200 import default_params
    T0 = o.pose6d_to_matrix(0.01, 0.01, 0.01, 0, 0, 0)
    prm = o.Params(detection=o.DET_EVD_SUB_CONDITION, handling=getattr(o, "HAND_" + handling), conv_rot=1e-4)
    conv, T_ref, logs, status = o.icp_so3(cylinder, cylinder, T0, prm)
    gp = default_params(detection="EVD_SUB_CONDITION", handling=handling, conv_thresh_rot=1e-4)
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    res = ctx.icp_run(gp, T0)
    assert res.converged == conv and res.iterations == len(logs)
    assert o.se3_log_distance(T_ref, res.T) < 1e-6
    for a in res.logs:
        assert a.analysis.is_degenerate == 0 and not any(a.analysis.degenerate_mask)
        assert a.analysis.schur_singular == 0 and not np.any(np.array(a.analysis.W_adaptive))
    a, dx, rc = ctx.analyze_and_solve(o.pack27(logs[0].H, logs[0].g), gp)
    assert np.max(np.abs(dx - logs[0].dx)) < 1e-9


def test_covariance_not_converged_is_1e6_identity(ctx, cylinder):
    """icp_test_runner.cpp:2014-2037: a run that did not converge reports 1e6 * I."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import g2_initial_pose
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    res = ctx.icp_run(default_params(max_iterations=2, kappa_target=10.0), g2_initial_pose())
    assert not res.converged and res.iterations == 2
    assert np.array_equal(ctx.last_covariance(), 1e6 * np.eye(6))


def test_covariance_eigenvalue_floor_branch(ctx):
    """H with an eigenvalue above 1e12 (a room 4 km from the origin: the rotation block grows with |p|^2) makes the
    smallest eigenvalue of H^-1 drop under 1e-12: the covariance is rebuilt with the 1e-9 floor."""
    from dcreg_b200 import default_params
    rng = np.random.default_rng(7)
    n = 150_000
    face = rng.integers(0, 6, n)
    u, v = rng.uniform(0, 20, n), rng.uniform(0, 20, n)
    w = rng.uniform(0, 5, n)
    pts = np.zeros((n, 3))
    for f in range(6):
        m = face == f
        if f < 2:
            pts[m] = np.stack([u[m], v[m], np.full(m.sum(), 5.0 * f)], axis=1)
        elif f < 4:
            pts[m] = np.stack([u[m], np.full(m.sum(), 20.0 * (f - 2)), w[m]], axis=1)
        else:
            pts[m] = np.stack([np.full(m.sum(), 20.0 * (f - 4)), v[m], w[m]], axis=1)
    pts = (pts + np.array([4000.0, 4000.0, 0.0])).astype(np.float32)
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    # loose thresholds: float32 coordinates 4 km out leave ~1e-4 m of residual noise; the test is about the covariance
    res = ctx.icp_run(default_params(max_iterations=10, conv_thresh_rot=1e-2, conv_thresh_trans=1.0), np.eye(4))
    assert res.converged
    H, _ = o.unpack27(np.array(res.logs[-1].H27))
    lam_H = np.linalg.eigvalsh(H)
    assert lam_H[-1] > 1e12
    inv = np.linalg.inv(H)
    lam, V = np.linalg.eigh(0.5 * (inv + inv.T))
    assert lam[0] <= 1e-12
    ref = V @ np.diag(np.maximum(lam, 1e-9)) @ V.T
    cov = ctx.last_covariance()
    assert np.max(np.abs(cov - ref)) < 1e-6 * np.max(np.abs(ref))
    assert np.min(np.linalg.eigvalsh(0.5 * (cov + cov.T))) > 0.5e-9


def test_weight_slope_and_gate_are_honoured(ctx, cylinder):
    """dcreg_icp_params::weight_slope / weight_gate (icp_test_runner.cpp:1776, 1785) reach the kernels: N_eff, the
    sums and RMSE of the first iteration follow s = 1 - slope |r|, kept when s > gate."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import g2_initial_pose
    T0 = g2_initial_pose()
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    planes, npt = ctx.find_planes(T0, 1.0)
    q = (cylinder.astype(np.float64) @ T0[:3, :3].T + T0[:3, 3]).astype(np.float32).astype(np.float64)
    has = np.any(planes[:, :3] != 0.0, axis=1)
    r = np.einsum("kj,kj->k", planes[:, :3], q) + planes[:, 3]
    seen = set()
    for slope, gate in ((0.9, 0.1), (0.5, 0.1), (0.9, 0.6), (2.0, 0.3)):
        s = 1.0 - slope * np.abs(r)
        valid = has & (s > gate)
        res = ctx.icp_run(default_params(max_iterations=1, weight_slope=slope, weight_gate=gate, min_effective_points=0), T0)
        L = res.logs[0]
        assert L.n_effective == int(valid.sum()) and L.n_corr_pt == npt
        assert abs(L.rmse - math.sqrt(np.sum(r[valid] ** 2) / valid.sum())) < 1e-12
        b = -(s[valid] * r[valid]).astype(np.float32).astype(np.float64)
        assert abs(L.objective - 0.5 * np.sum(b * b)) < 1e-11 * max(1.0, L.objective)
        seen.add(L.n_effective)
    assert len(seen) >= 3                    # the parameters really change what is kept


def test_host_planes_fitness_uses_the_callers_count(ctx, golden, cylinder):
    """Host-kd-tree mode: n_corr_pt / fitness come from the callback's count (5th neighbour inside the radius, before
    the plane gates: icp_test_runner.cpp:1726-1731, 1856), as in the device-correspondence loop and the oracle."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import g2_initial_pose
    T0 = g2_initial_pose()
    tree = o.build_tree(cylinder)
    prm = o.Params(kappa_target=10.0, use_weight_derivative=True, max_iterations=4)
    _, _, logs, _ = o.icp_so3(cylinder, cylinder, T0, prm, tree)

    def plane_fn(Tc):
        c = o.find_correspondences(cylinder, cylinder, tree, Tc[:3, :3], Tc[:3, 3], 1.0, True)
        planes = np.zeros((len(cylinder), 4))
        planes[c.has_plane, :3] = c.n[c.has_plane]; planes[c.has_plane, 3] = c.d[c.has_plane]
        return planes, c.n_pt

    ctx.set_source(cylinder)
    gp = default_params(kappa_target=10.0, use_weight_derivative=1, max_iterations=4, fixed_iterations=1)
    res = ctx.icp_run_host_planes(gp, T0, plane_fn)
    for a, b in zip(res.logs, logs):
        assert a.n_effective == b.n_eff and a.n_corr_pt == b.n_pt
        assert abs(a.fitness - b.fitness) < 1e-15
    assert res.logs[0].n_corr_pt == 391 and abs(res.logs[0].fitness - 0.05170590) < 1e-8   # G2, iteration 0 (shipped)


# ------------------------------------------------------------------------------------------------
# sparse row index (bounding box too large for the dense cell table), aborting trials in a batch
# ------------------------------------------------------------------------------------------------
def test_sparse_index_path_matches_oracle(ctx, cylinder):
    """Two far outliers blow the target's bounding box up to ~1e11 cells: dcreg_set_target builds a sparse row index.
    Same trajectory as the oracle; a batch runs, every trial as its own icp_run; the point-to-point metrics (dense grids
    only) are refused.  Back on a dense target, the context's reused grid arena gives the bits of a fresh context."""
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import BAD_ARG, DcregError
    from dcreg_b200.scenes import g2_initial_pose
    tgt = np.concatenate([cylinder, np.array([[4000.0, 4500.0, 5000.0], [-4000.0, -3000.0, 2000.0]], np.float32)]).astype(np.float32)
    T0 = g2_initial_pose()
    prm = o.Params(kappa_target=10.0, use_weight_derivative=True)
    conv, T_ref, logs, status = o.icp_so3(cylinder, tgt, T0, prm)
    gp = default_params(kappa_target=10.0, use_weight_derivative=1)
    ctx.set_target(tgt, 1.0)
    ctx.set_source(cylinder)
    res = ctx.icp_run(gp, T0)
    assert res.converged == conv and res.iterations == len(logs)
    for a, b in zip(res.logs, logs):
        assert a.n_effective == b.n_eff and a.n_corr_pt == b.n_pt
    assert o.se3_log_distance(T_ref, res.T) < 1e-6
    Ts = perturbations(2)
    batch = ctx.icp_run_batch(gp, Ts)
    for t in range(len(Ts)):
        single = ctx.icp_run(gp, Ts[t])
        assert (batch[t].status, batch[t].iterations, batch[t].converged) == (single.status, single.iterations, single.converged)
        assert o.se3_log_distance(single.T, batch[t].T) < 1e-8
    with pytest.raises(DcregError) as e:
        ctx.point_to_point_metrics(res.T, 0.2)
    assert e.value.status == BAD_ARG
    ctx.set_target(cylinder, 1.0)            # back to a dense grid for the tests that follow
    dense = ctx.icp_run(gp, T0)
    m = ctx.point_to_point_metrics(dense.T, 0.2)
    with Context(0) as fresh:
        fresh.set_target(cylinder, 1.0)
        fresh.set_source(cylinder)
        ref = fresh.icp_run(gp, T0)
        assert m == fresh.point_to_point_metrics(ref.T, 0.2)
    assert (dense.status, dense.iterations, dense.converged) == (ref.status, ref.iterations, ref.converged)
    assert dense.T.tobytes() == ref.T.tobytes()
    assert [np.array(L.H27).tobytes() for L in dense.logs] == [np.array(L.H27).tobytes() for L in ref.logs]


def test_sparse_index_target_equals_dense_target(ctx, cylinder):
    """Target A is the cylinder plus two far outliers (a sparse row index), target B the cylinder alone (a dense grid);
    the outliers come last, so the cylinder's point indices (the tie rule) agree and no query ever reaches them.  Seam 1
    gives the same planes bit for bit; a fixed-iteration run on A gives the counts of the run on B and its poses to
    rounding.  Coherent mode can be timed on A."""
    from dcreg_b200 import default_params
    far = np.array([[4000.0, 4500.0, 5000.0], [-4000.0, -3000.0, 2000.0]], np.float32)
    tgt_a = np.concatenate([cylinder, far]).astype(np.float32)
    T0 = o.pose6d_to_matrix(0.1, 0.3, 0.2, math.radians(0.1), math.radians(-0.1), math.radians(1.0))
    methods = [("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG"), ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD")]
    prms = [default_params(max_iterations=30, fixed_iterations=1, kappa_target=10.0, detection=d, handling=h)
            for d, h in methods]
    ctx.set_source(cylinder)
    out = {}
    for name, tgt in (("A", tgt_a), ("B", cylinder)):
        ctx.set_target(tgt, 1.0)
        out[name] = (ctx.find_planes(T0, 1.0), [ctx.icp_run(p, T0) for p in prms])
        if name == "A":
            assert 0.0 < ctx.time_iteration(prms[0], T0, 0, 2) < 5.0
    (planes_a, npt_a), runs_a = out["A"]
    (planes_b, npt_b), runs_b = out["B"]
    assert npt_a == npt_b > 0
    assert planes_a.tobytes() == planes_b.tobytes()
    for a, b in zip(runs_a, runs_b):
        assert (a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged) and a.iterations == 30
        for la, lb in zip(a.logs, b.logs):
            assert la.n_effective == lb.n_effective and la.n_corr_pt == lb.n_corr_pt
            assert list(la.analysis.degenerate_mask) == list(lb.analysis.degenerate_mask)
            assert o.se3_log_distance(np.array(la.T).reshape(4, 4), np.array(lb.T).reshape(4, 4)) < 1e-9
        assert o.se3_log_distance(a.T, b.T) < 1e-9


def test_batch_with_aborting_trials(ctx, cylinder):
    """A trial that starts 100 m away finds no correspondences and aborts (NOT_ENOUGH_POINTS, icp_test_runner.cpp:1847)
    without disturbing its neighbours in the batch."""
    from dcreg_b200 import default_params
    from dcreg_b200.api import NOT_ENOUGH_POINTS
    gp = default_params(kappa_target=10.0, max_iterations=30)
    Ts = perturbations(5, seed=47)
    far = np.eye(4); far[:3, 3] = [100.0, 0.0, 50.0]
    Ts[2] = far
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    batch = ctx.icp_run_batch(gp, Ts, want_log=True)
    assert batch[2].status == NOT_ENOUGH_POINTS and not batch[2].converged and batch[2].iterations == 1
    assert np.allclose(batch[2].T, far)
    for t in (0, 1, 3, 4):
        single = ctx.icp_run(gp, Ts[t])
        assert batch[t].status == single.status == 0 and batch[t].iterations == single.iterations
        assert o.se3_log_distance(single.T, batch[t].T) < 1e-8
