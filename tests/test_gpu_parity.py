"""GPU parity tests: the CUDA path, called through the C ABI, against the CPU oracle and the golden dumps.

Tolerances (north_star): pose 1e-6 on the SE(3) log, Schur eigenvalues 1e-8 relative; the
27 reduced scalars are compared at 1e-11 relative to the largest entry (FP64 sums in a
different order).  Integer outputs (counts, masks, iteration counts) must be identical.
"""
import math
import os

import numpy as np
import pytest

import dcreg_oracle as o
from test_oracle_golden import METHODS, init_T, params_from

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def tree(cylinder):
    return o.build_tree(cylinder)


def gpu_params(prm: o.Params, **over):
    from dcreg_b200 import default_params
    p = default_params(search_radius=prm.search_radius, max_iterations=prm.max_iterations,
                       detection=prm.detection, handling=prm.handling,
                       use_weight_derivative=int(prm.use_weight_derivative), conv_thresh_rot=prm.conv_rot,
                       conv_thresh_trans=prm.conv_trans, cond_thresh=prm.cond_thresh, eig_thresh=prm.eig_thresh,
                       kappa_target=prm.kappa_target, pcg_tol=prm.pcg_tol, pcg_max_iter=prm.pcg_max_iter,
                       std_reg_gamma=prm.std_reg_gamma)
    for k, v in over.items():
        setattr(p, k, v)
    return p


def src4_of(pts):
    return np.concatenate([pts, np.zeros((len(pts), 1), np.float32)], axis=1)


# ------------------------------------------------------------------------------------------------
# seam 3: K2 (analysis + solve)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setup,method", [("G2", "Ours"), ("G1", "ME-SR"), ("G1", "ME-TSVD"), ("G1", "ME-TReg"),
                                          ("G1", "FCN-SR"), ("G2", "ME-TReg"), ("G2", "FCN-SR")])
def test_k2_analysis_and_solve_matches_oracle(ctx, golden, cylinder, tree, setup, method):
    g = golden[setup]
    prm = params_from(g["setup"], method)
    _, _, logs, _ = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), prm, tree)
    gp = gpu_params(prm)
    for L in logs:
        a, dx, rc = ctx.analyze_and_solve(o.pack27(L.H, L.g), gp)
        assert rc == 0
        A = L.analysis
        assert np.abs(dx - L.dx).max() <= 1e-9 * max(1.0, np.abs(L.dx).max())
        assert list(a.degenerate_mask) == [int(m) for m in A.mask] and a.is_degenerate == int(A.is_degenerate)
        assert np.allclose(a.np("eigenvalues_full"), A.eigenvalues_full, rtol=1e-9, atol=1e-9 * A.eigenvalues_full[-1])
        assert np.allclose(a.np("singular_values"), A.singular_values, rtol=1e-9, atol=1e-9 * A.singular_values[0])
        assert np.allclose(a.np("lambda_schur_rot"), A.lambda_schur_rot, rtol=1e-8, atol=0)      # contract: 1e-8 rel
        assert np.allclose(a.np("lambda_schur_trans"), A.lambda_schur_trans, rtol=1e-8, atol=0)
        assert np.allclose(a.np("lambda_sub_rot"), A.lambda_sub_rot, rtol=1e-9)
        assert np.allclose(a.np("lambda_sub_trans"), A.lambda_sub_trans, rtol=1e-9)
        for nm, ref in (("cond_schur_rot", A.cond_schur_rot), ("cond_schur_trans", A.cond_schur_trans),
                        ("cond_diag_rot", A.cond_diag_rot), ("cond_diag_trans", A.cond_diag_trans),
                        ("cond_full", A.cond_full), ("cond_full_sub_rot", A.cond_full_sub_rot),
                        ("cond_full_sub_trans", A.cond_full_sub_trans)):
            assert abs(getattr(a, nm) - ref) <= 1e-8 * abs(ref), nm
        if prm.detection == o.DET_SCHUR_CONDITION_NUMBER:
            assert np.allclose(a.np("P_preconditioner").reshape(6, 6), A.P, rtol=1e-8, atol=1e-14)
            assert a.pcg_iterations == A.pcg_iterations
            # eigenvectors: same subspaces (sign-free comparison through the projectors)
            for nm, ref in (("schur_V_rot", A.schur_V_rot), ("schur_V_trans", A.schur_V_trans)):
                V = a.np(nm).reshape(3, 3)
                for k in range(3):
                    assert abs(abs(V[:, k] @ ref[:, k]) - 1.0) < 1e-8


def test_k2_golden_first_iteration_ours(ctx, golden, cylinder, tree):
    """GPU K2 on the oracle's H of G2 iteration 0 against the numbers the reference shipped."""
    g = golden["G2"]
    prm = params_from(g["setup"], "Ours", max_iterations=1)
    _, _, logs, _ = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), prm, tree)
    a, dx, _ = ctx.analyze_and_solve(o.pack27(logs[0].H, logs[0].g), gpu_params(prm))
    row = g["iterations"]["Ours"][0]
    fi = g["first_iter"]["Ours"]
    assert np.abs(dx - np.array(row["dx"])).max() < 5e-7
    assert list(a.degenerate_mask) == fi["mask"] == [0, 0, 0, 1, 0, 0]
    assert np.allclose(a.np("lambda_schur_rot"), g["schur_lambda_rot"], rtol=3e-7)
    assert np.allclose(a.np("lambda_schur_trans"), g["schur_lambda_trans"], atol=1e-6)
    assert np.allclose(a.np("eigenvalues_full"), fi["eigenvalues_full"], atol=6e-4)
    assert abs(a.cond_schur_rot - row["cond_schur_rot"]) < 1e-5 and abs(a.cond_schur_trans - row["cond_schur_trans"]) < 1e-5
    # alignment report (paper Alg. 2): orig_idx per slot as logged
    al = fi["alignment"]
    assert list(a.rot_indices) == [x["orig_idx"] for x in al[:3]]
    assert list(a.trans_indices) == [x["orig_idx"] for x in al[3:]]
    pi = list(a.rot_indices) + [3 + k for k in a.trans_indices]
    P = a.np("P_preconditioner").reshape(6, 6)
    assert np.allclose(P[np.ix_(pi, pi)], np.array(fi["P_logged"]), atol=1.5e-6)
    Va = a.np("aligned_V_trans").reshape(3, 3)
    for j, x in enumerate(al[3:]):
        raw = a.np("schur_V_trans").reshape(3, 3)[:, x["orig_idx"]]
        assert abs(math.degrees(math.acos(min(1.0, abs(raw[j])))) - x["angle_deg"]) < 1e-4


def test_pcg_seam(ctx):
    rng = np.random.default_rng(7)
    M = rng.normal(size=(6, 6)); A = M @ M.T + 0.1 * np.eye(6)
    b = rng.normal(size=6); P = np.diag(1.0 / np.diag(A))
    x, it = ctx.solve_pcg(A, b, P, 20, 1e-10)
    xr, itr = o.pcg(A, b, P, 20, 1e-10)
    assert it == itr and np.abs(x - xr).max() < 1e-10
    assert np.abs(A @ x - b).max() < 1e-9


def test_k2_singular_and_nonfinite(ctx):
    from dcreg_b200 import default_params, api
    # H = 0: singular blocks -> Schur conds = inf (icp_test_runner.cpp:2464-2469); the pivoted-QR solve of an
    # all-zero matrix divides by a zero pivot exactly like Eigen's, the loop then aborts (:1942-1950)
    v = np.zeros(27)
    a, dx, rc = ctx.analyze_and_solve(v, default_params())
    assert rc == api.NONFINITE_UPDATE and math.isinf(a.cond_schur_rot) and math.isinf(a.cond_full)
    assert a.is_degenerate == 0
    # rank-deficient but non-zero H (pure translation information): finite basic solution, zero rotation part
    H = np.zeros((6, 6)); H[3:, 3:] = np.diag([4.0, 2.0, 1.0]); g = np.array([0, 0, 0, 4.0, 2.0, 1.0])
    a, dx, rc = ctx.analyze_and_solve(o.pack27(H, g), default_params(handling="NONE_HAND", detection="NONE_DETE"))
    assert rc == 0 and np.allclose(dx, [0, 0, 0, 1, 1, 1])
    v[:] = np.nan
    a, dx, rc = ctx.analyze_and_solve(v, default_params(handling="NONE_HAND", detection="NONE_DETE"))
    assert rc == api.NONFINITE_UPDATE


# ------------------------------------------------------------------------------------------------
# seam 2: K1 (fused residual / weight / Jacobian / reduction)
# ------------------------------------------------------------------------------------------------
def frozen_planes(cylinder, tree, T, use_wd):
    corr = o.find_correspondences(cylinder, cylinder, tree, T[:3, :3], T[:3, 3], 1.0, use_wd)
    plane = np.concatenate([corr.n, corr.d[:, None]], axis=1)
    plane[~corr.valid] = 0.0
    return plane, corr


@pytest.mark.parametrize("use_wd", [False, True])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_k1_matches_oracle_on_cylinder(ctx, golden, cylinder, tree, use_wd, dtype):
    T = init_T(golden["G2"]["setup"])
    plane, corr = frozen_planes(cylinder, tree, T, use_wd)
    plane = plane.astype(dtype)
    ref, rstats = o.reduce_normal_equations(src4_of(cylinder), plane, T[:3, :3], T[:3, 3], use_wd)
    out, stats = ctx.reduce_normal_equations(src4_of(cylinder), plane, T, use_wd)
    scale = np.abs(ref).max()
    assert np.abs(out - ref).max() <= 1e-11 * scale
    assert int(stats[1]) == int(rstats[1]) and int(stats[2]) == int(rstats[2])
    assert abs(stats[0] - rstats[0]) <= 1e-11 * max(1.0, rstats[0])
    if dtype == np.float64 and use_wd:
        # with FP64 planes the seam reproduces the loop's H: eig(H) equals the shipped G2 values
        H, _ = o.unpack27(out)
        assert np.allclose(np.linalg.eigvalsh(H), golden["G2"]["first_iter"]["Ours"]["eigenvalues_full"], atol=6e-4)


def test_k1_g1_eigenvalues(ctx, golden, cylinder, tree):
    T = init_T(golden["G1"]["setup"])
    plane, _ = frozen_planes(cylinder, tree, T, False)
    out, stats = ctx.reduce_normal_equations(src4_of(cylinder), plane, T, False)
    H, _ = o.unpack27(out)
    assert np.allclose(np.linalg.eigvalsh(H), [15.296, 128.819, 179.792, 16680.091, 60715.675, 68461.177], atol=6e-4)
    assert int(stats[1]) == 871


@pytest.mark.parametrize("n", [1, 31, 257, 4099, 100_003])
def test_k1_ragged_sizes_and_empty_slots(ctx, n):
    rng = np.random.default_rng(n)
    src = rng.uniform(-30, 30, (n, 4)).astype(np.float32)
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    T = o.pose6d_to_matrix(0.1, -0.2, 0.05, 0.01, -0.02, 0.03)
    q = src[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]
    d = -(nrm * q).sum(1) + rng.uniform(-1.3, 1.3, n)          # residuals in [-1.3, 1.3]: some gated out
    plane = np.concatenate([nrm, d[:, None]], axis=1)
    plane[rng.uniform(size=n) < 0.3] = 0.0                       # empty slots
    for dtype in (np.float32, np.float64):
        pl = plane.astype(dtype)
        for wd in (False, True):
            ref, rs = o.reduce_normal_equations(src, pl, T[:3, :3], T[:3, 3], wd)
            out, st = ctx.reduce_normal_equations(src, pl, T, wd)
            assert np.abs(out - ref).max() <= 1e-11 * max(1.0, np.abs(ref).max())
            assert int(st[1]) == int(rs[1]) and int(st[2]) == int(rs[2])


def test_k1_all_slots_empty(ctx):
    src = np.ones((1000, 4), np.float32)
    out, st = ctx.reduce_normal_equations(src, np.zeros((1000, 4), np.float32), np.eye(4), False)
    assert np.all(out == 0) and st[1] == 0 and st[2] == 0


def test_k1_linearity_at_scale(ctx):
    """Size-independent property at 4M slots: reduce(A u B) == reduce(A) + reduce(B); deterministic re-run."""
    n = 4_000_000
    rng = np.random.default_rng(1)
    src = rng.uniform(-50, 50, (n, 4)).astype(np.float32)
    nrm = rng.normal(size=(n, 3)).astype(np.float32)
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    T = o.pose6d_to_matrix(0.3, 0.1, -0.2, 0.02, 0.01, -0.03)
    q = (src[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3])
    d = (-(nrm.astype(np.float64) * q).sum(1) + rng.uniform(-0.5, 0.5, n)).astype(np.float32)
    plane = np.concatenate([nrm, d[:, None]], axis=1).astype(np.float32)
    whole, sw = ctx.reduce_normal_equations(src, plane, T, True)
    again, _ = ctx.reduce_normal_equations(src, plane, T, True)
    assert np.array_equal(whole, again)                            # deterministic reduction order
    h = n // 2 + 12345
    a, sa = ctx.reduce_normal_equations(src[:h], plane[:h], T, True)
    b, sb = ctx.reduce_normal_equations(src[h:], plane[h:], T, True)
    assert np.abs(a + b - whole).max() <= 1e-11 * np.abs(whole).max()
    assert int(sa[1] + sb[1]) == int(sw[1])
    # spot-check against the oracle on a 200k sample
    ref, _ = o.reduce_normal_equations(src[:200_000], plane[:200_000], T[:3, :3], T[:3, 3], True)
    out, _ = ctx.reduce_normal_equations(src[:200_000], plane[:200_000], T, True)
    assert np.abs(out - ref).max() <= 1e-11 * np.abs(ref).max()


# ------------------------------------------------------------------------------------------------
# seam 1: correspondences (grid exact 5-NN + plane fit)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("setup", ["G1", "G2"])
def test_find_planes_matches_oracle(ctx, golden, cylinder, tree, setup):
    T = init_T(golden[setup]["setup"])
    ctx.set_source(cylinder)
    ctx.set_target(cylinder, 1.0)
    planes, npt = ctx.find_planes(T, 1.0)
    q32 = o.transform_points_f32(cylinder, T[:3, :3], T[:3, 3])
    dist, idx = tree.query(q32.astype(np.float64), k=5)
    near = (dist[:, 4] ** 2) < 1.0
    assert npt == int(near.sum())
    nn, dd, ok = o.fit_planes(cylinder[idx[near]].astype(np.float64))
    ref = np.zeros((len(cylinder), 4))
    sel = np.nonzero(near)[0]
    ref[sel[ok], :3] = nn[ok]; ref[sel[ok], 3] = dd[ok]
    has_ref = np.abs(ref[:, :3]).sum(1) > 0
    has_gpu = np.abs(planes[:, :3]).sum(1) > 0
    assert np.array_equal(has_ref, has_gpu)
    assert np.abs(planes - ref).max() < 1e-9


@pytest.mark.parametrize("div", [1, 2, 3, 4])
def test_find_planes_finer_grids_are_exact(ctx, golden, cylinder, tree, div):
    """cell = radius / div (div rings of cells per direction): same accept set and planes as the kd-tree."""
    T = init_T(golden["G2"]["setup"])
    ctx.set_source(cylinder)
    ctx.set_target(cylinder, 1.0 / div)
    planes, npt = ctx.find_planes(T, 1.0)
    corr = o.find_correspondences(cylinder, cylinder, tree, T[:3, :3], T[:3, 3], 1.0, False)
    assert npt == corr.n_pt
    ref = np.concatenate([corr.n, corr.d[:, None]], axis=1); ref[~corr.has_plane] = 0
    assert np.array_equal(np.abs(ref[:, :3]).sum(1) > 0, np.abs(planes[:, :3]).sum(1) > 0)
    assert np.abs(planes - ref).max() < 1e-9


def test_find_planes_random_cloud_radius_half(ctx):
    rng = np.random.default_rng(3)
    tgt = rng.uniform(-5, 5, (60_000, 3)).astype(np.float32)
    tgt[:, 2] *= 0.05                                            # slab: planes exist
    src = (tgt[::7] + rng.normal(0, 0.02, tgt[::7].shape)).astype(np.float32)
    T = o.pose6d_to_matrix(0.02, -0.01, 0.01, 0.002, 0.001, -0.004)
    ctx.set_source(src); ctx.set_target(tgt, 0.5)
    planes, npt = ctx.find_planes(T, 0.5)
    tr = o.build_tree(tgt)
    corr = o.find_correspondences(src, tgt, tr, T[:3, :3], T[:3, 3], 0.5, False)
    assert npt == corr.n_pt
    # oracle planes before the weight gate
    q32 = o.transform_points_f32(src, T[:3, :3], T[:3, 3])
    dist, idx = tr.query(q32.astype(np.float64), k=5)
    near = (dist[:, 4] ** 2) < 0.25
    nn, dd, ok = o.fit_planes(tgt[idx[near]].astype(np.float64))
    sel = np.nonzero(near)[0]
    ref = np.zeros((len(src), 4)); ref[sel[ok], :3] = nn[ok]; ref[sel[ok], 3] = dd[ok]
    assert np.array_equal(np.abs(ref[:, :3]).sum(1) > 0, np.abs(planes[:, :3]).sum(1) > 0)
    assert np.abs(planes - ref).max() < 1e-8


# ------------------------------------------------------------------------------------------------
# the outer loop
# ------------------------------------------------------------------------------------------------
def check_against_oracle(res, conv, T, logs, status):
    assert res.status == {"ok": 0, "not_enough_points": 1, "nonfinite": 2}[status]
    assert res.converged == conv and res.iterations == len(logs) + (1 if status == "not_enough_points" else 0)
    for L, G in zip(logs, res.logs):
        assert G.n_effective == L.n_eff and G.n_corr_pt == L.n_pt
        assert o.se3_log_distance(L.T, np.array(G.T).reshape(4, 4)) < 1e-6          # contract
        assert np.abs(np.array(G.dx) - L.dx).max() < 1e-8
        assert abs(G.rmse - L.rmse) < 1e-10 and abs(G.fitness - L.fitness) < 1e-12
        assert abs(G.objective - L.objective) < 1e-9 * max(1.0, L.objective)
        assert list(G.analysis.degenerate_mask) == [int(m) for m in L.analysis.mask]
        assert np.allclose(G.analysis.np("lambda_schur_rot"), L.analysis.lambda_schur_rot, rtol=1e-8)
        assert np.allclose(G.analysis.np("lambda_schur_trans"), L.analysis.lambda_schur_trans, rtol=1e-8)
    assert o.se3_log_distance(T, res.T) < 1e-6


@pytest.mark.parametrize("setup,method", [("G2", "Ours"), ("G1", "ME-SR"), ("G1", "ME-TSVD"), ("G1", "ME-TReg"),
                                          ("G1", "FCN-SR")])
def test_icp_run_matches_oracle_and_golden(ctx, golden, cylinder, tree, setup, method):
    g = golden[setup]
    prm = params_from(g["setup"], method)
    conv, T, logs, status = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), prm, tree)
    ctx.set_source(cylinder); ctx.set_target(cylinder, prm.search_radius)
    res = ctx.icp_run(gpu_params(prm), init_T(g["setup"]))
    check_against_oracle(res, conv, T, logs, status)
    rows = g["iterations"][method]
    assert res.iterations == len(rows)
    for r, G in zip(rows, res.logs):                                    # shipped numbers, print precision
        assert np.abs(np.array(r["T"]).reshape(4, 4) - np.array(G.T).reshape(4, 4)).max() < 5e-7
        assert np.abs(np.array(r["dx"]) - np.array(G.dx)).max() < 5e-7
        assert list(G.analysis.degenerate_mask) == r["mask"]


def test_icp_host_planes_mode(ctx, golden, cylinder, tree):
    """PR1 mode: correspondences from the host (here: the oracle's kd-tree), K1+K2 on the device."""
    g = golden["G2"]
    prm = params_from(g["setup"], "Ours")
    conv, T, logs, status = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), prm, tree)

    def plane_fn(Tc):
        corr = o.find_correspondences(cylinder, cylinder, tree, Tc[:3, :3], Tc[:3, 3], prm.search_radius, True)
        pl = np.concatenate([corr.n, corr.d[:, None]], axis=1)
        pl[~corr.has_plane] = 0          # the weight gate is re-evaluated on the device
        return pl, corr.n_pt

    ctx.set_source(cylinder)
    res = ctx.icp_run_host_planes(gpu_params(prm), init_T(g["setup"]), plane_fn)
    assert res.converged == conv and res.iterations == len(logs)
    for L, G in zip(logs, res.logs):
        assert G.n_effective == L.n_eff
        assert o.se3_log_distance(L.T, np.array(G.T).reshape(4, 4)) < 1e-9
    cov = ctx.last_covariance()
    assert np.allclose(cov, np.linalg.inv(logs[-1].H), rtol=1e-7, atol=1e-12)


def test_icp_fixed_iterations_synthetic_cylinder(ctx):
    """BASELINE config C2 shape at reduced size: synthetic cylinder, fixed iteration count, pose vs oracle."""
    from dcreg_b200.scenes import make_cylinder, make_corridor
    pts = make_cylinder(20_000, seed=42)
    T0 = o.pose6d_to_matrix(0.2, 0.8, 0.5, math.radians(0.1), math.radians(0.1), math.radians(2.0))
    prm = o.Params(max_iterations=12, conv_rot=0.0, conv_trans=0.0, kappa_target=10.0, use_weight_derivative=True)
    conv, T, logs, status = o.icp_so3(pts, pts, T0, prm)
    ctx.set_source(pts); ctx.set_target(pts, 1.0)
    res = ctx.icp_run(gpu_params(prm, fixed_iterations=1), T0)
    assert res.iterations == 12 and not res.converged
    check_against_oracle(res, conv, T, logs, status)


def loop_reuse_cases():
    """(method, target cell, shift of the scene): cell = radius (rings 1, the usual set-up; ids as before), finer cells
    (rings 2, 3 with a non-integer radius / cell, 4) and the cylinder far from the origin"""
    far = (4096.3, -2047.7, 130.1)
    cases = [pytest.param(m, 1.0, None, id=m) for m in ("Ours", "ME-TSVD")]
    cases += [pytest.param(m, c, None, id=f"{m}-cell{c}") for m in ("Ours", "ME-TSVD") for c in (0.5, 0.4, 0.25)]
    cases += [pytest.param("Ours", 1.0, far, id="Ours-far")]
    return cases


@pytest.mark.parametrize("method,cell,shift", loop_reuse_cases())
def test_loop_with_reused_correspondences_equals_full_search_every_iteration(ctx, method, cell, shift):
    """The loop's iteration kernel reuses neighbour lists (gap certificate) and plane fits (same five points) once the
    pose moves little.  Against the same loop with a full search and a fresh fit in EVERY iteration (the loop kernel's
    lean mode in every iteration, DCREG_FUSED_SEARCH=1) the per-iteration counts must be identical and the poses equal
    to rounding; the counters show that the reuse paths were actually taken.  Target cells finer than the search
    radius (1.0) run the warp and bounded searches over 2-4 rings of cells."""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import make_cylinder
    pts = make_cylinder(30_000, seed=7)
    T0 = o.pose6d_to_matrix(0.1, 0.3, 0.2, math.radians(0.1), math.radians(-0.1), math.radians(1.0))
    if shift is not None:                                   # the same motion, about the moved cylinder
        S = np.eye(4)
        S[:3, 3] = shift
        pts = (pts.astype(np.float64) + shift).astype(np.float32)
        T0 = S @ T0 @ np.linalg.inv(S)
    det, hand = METHODS[method]
    prm = default_params(max_iterations=40, fixed_iterations=1, kappa_target=10.0, detection=det, handling=hand)
    ctx.set_source(pts); ctx.set_target(pts, cell)
    ctx.iteration_counters(True)
    res = ctx.icp_run(prm, T0)
    searched, fitted = ctx.iteration_counters(False)
    os.environ["DCREG_FUSED_SEARCH"] = "1"
    try:
        ref = ctx.icp_run(prm, T0)
    finally:
        del os.environ["DCREG_FUSED_SEARCH"]
    assert res.iterations == ref.iterations == 40
    for A, B in zip(res.logs, ref.logs):
        assert A.n_effective == B.n_effective and A.n_corr_pt == B.n_corr_pt
        assert o.se3_log_distance(np.array(A.T).reshape(4, 4), np.array(B.T).reshape(4, 4)) < 1e-11
        assert abs(A.rmse - B.rmse) < 1e-12
    # 40 iterations x 30k slots = 1.2 M slot-iterations: well under half of them searched / fitted
    assert 30_000 <= searched < 600_000 and 30_000 <= fitted < 600_000


def test_loop_reuse_on_a_lattice_with_duplicates_and_ties(ctx):
    """Worst case for the neighbour bookkeeping: a regular lattice (many exactly equal distances -> index rule),
    duplicated target points, a dense patch (more than 64 candidates inside a loose bound -> the warp search gives up
    and the slot searches sequentially) and a source that is not a multiple of the tile size.  The reference is a full
    search and a fresh fit in every iteration (lean mode throughout, DCREG_FUSED_SEARCH=1)."""
    check_lattice_reuse(ctx, 1.0)


@pytest.mark.parametrize("cell", [0.5, 0.25])
def test_loop_reuse_on_a_lattice_at_finer_cells(ctx, cell):
    """The lattice scene above with target cells of half and a quarter of the search radius: the warp and bounded
    searches over 2 and 4 rings of cells; at 0.25 the lattice points lie on cell faces."""
    check_lattice_reuse(ctx, cell)


def check_lattice_reuse(ctx, cell):
    from dcreg_b200 import default_params
    g = np.arange(-6, 6, 0.25, dtype=np.float32)
    X, Y = np.meshgrid(g, g)
    floor = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, np.float32)], axis=1)
    wall = np.stack([X.ravel(), np.full(X.size, 6.0, np.float32), (Y.ravel() + 6.0) * 0.5], axis=1)
    wall2 = np.stack([np.full(X.size, -6.0, np.float32), X.ravel(), (Y.ravel() + 6.0) * 0.5], axis=1)
    d = np.arange(-1, 1, 0.05, dtype=np.float32)
    DX, DY = np.meshgrid(d, d)
    dense = np.stack([DX.ravel(), DY.ravel(), np.zeros(DX.size, np.float32)], axis=1)
    tgt = np.concatenate([floor, wall, wall2, dense, floor[::5]]).astype(np.float32)       # floor[::5]: exact duplicates
    rng = np.random.default_rng(5)
    src = tgt[rng.permutation(len(tgt))[:7001]].copy()
    T0 = o.pose6d_to_matrix(0.06, -0.05, 0.04, math.radians(0.2), math.radians(-0.1), math.radians(0.4))
    prm = default_params(max_iterations=25, fixed_iterations=1, kappa_target=10.0)
    ctx.set_source(src); ctx.set_target(tgt, cell)
    res = ctx.icp_run(prm, T0)
    os.environ["DCREG_FUSED_SEARCH"] = "1"
    try:
        ref = ctx.icp_run(prm, T0)
    finally:
        del os.environ["DCREG_FUSED_SEARCH"]
    assert res.status == ref.status and res.iterations == ref.iterations
    for A, B in zip(res.logs, ref.logs):
        assert A.n_effective == B.n_effective and A.n_corr_pt == B.n_corr_pt
        # same correspondences, same planes; the 27 sums are added in a different order and this lattice scene is
        # ill-conditioned (many rank-deficient neighbourhoods), so the poses agree to ~1e-10 rather than 1e-12
        assert o.se3_log_distance(np.array(A.T).reshape(4, 4), np.array(B.T).reshape(4, 4)) < 1e-8


def test_iteration_timing_entry_point(ctx):
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import make_cylinder
    pts = make_cylinder(20_000, seed=3)
    ctx.set_source(pts); ctx.set_target(pts, 1.0)
    prm = default_params(kappa_target=10.0)
    T0 = o.pose6d_to_matrix(0.05, 0.05, 0.05, 0.0, 0.0, math.radians(0.5))
    assert 0.0 < ctx.time_iteration(prm, T0, 0, 5) < 5.0
    assert 0.0 < ctx.time_iteration(prm, T0, 1, 5) < 5.0


def test_icp_corridor_weakest_translation_is_the_axis(ctx):
    """C4-shaped scene at test size: two walls + floor + ceiling; the least-constrained translation is along x."""
    from dcreg_b200.scenes import make_corridor
    pts = make_corridor(40_000, seed=44, length=60.0, noise=0.002)
    T0 = o.pose6d_to_matrix(0.05, 0.04, 0.03, 0.0, 0.0, math.radians(0.3))
    prm = o.Params(max_iterations=6, kappa_target=10.0, search_radius=0.5)
    conv, T, logs, status = o.icp_so3(pts, pts, T0, prm)
    ctx.set_source(pts); ctx.set_target(pts, 0.5)
    res = ctx.icp_run(gpu_params(prm), T0)
    check_against_oracle(res, conv, T, logs, status)
    v = res.logs[0].analysis.np("schur_V_trans").reshape(3, 3)[:, 0]
    assert abs(v[0]) > 0.99                                        # weakest translation direction = corridor axis x
    assert res.logs[0].analysis.is_degenerate == int(logs[0].analysis.is_degenerate)


def test_icp_parking_lot_standin_c3(ctx):
    """BASELINE config C3 (icp_pk01.yaml shapes; the real pair is not shipped): ~6 k-point scan vs a 0.5 M-point
    ground-dominated map, radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, init offset of icp_pk01.yaml:30-44.
    Degeneracy eigenvalues, masks and the pose against the C oracle."""
    import dcreg_oracle_c as oc
    from dcreg_b200.scenes import make_parking
    scan, tgt = make_parking(n_map=500_000, n_scan=6_000, seed=43)
    T0 = o.pose6d_to_matrix(0.15, 0.12, 0.13, math.radians(0.015), math.radians(1.31), math.radians(2.17))
    prm = o.Params(search_radius=0.5, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    sc = oc.Scene(scan, tgt)
    cp = oc.make_params(search_radius=0.5, max_iterations=30, conv_rot=1e-5, conv_trans=1e-3, kappa_target=10.0)
    st, conv, n_it, Tc, clogs = sc.icp_run(cp, T0)
    sc.close()
    ctx.set_source(scan); ctx.set_target(tgt, 0.5)
    res = ctx.icp_run(gpu_params(prm), T0)
    assert res.status == st and res.converged == conv and res.iterations == n_it
    for C, G in zip(clogs, res.logs):
        assert G.n_effective == C.n_eff and G.n_corr_pt == C.n_pt
        assert list(G.analysis.degenerate_mask) == list(C.mask)
        assert np.allclose(G.analysis.np("lambda_schur_rot"), C.lam_schur_rot, rtol=1e-8)
        assert np.allclose(G.analysis.np("lambda_schur_trans"), C.lam_schur_trans, rtol=1e-8)
        assert np.abs(np.array(G.dx) - np.array(C.dx)).max() < 1e-8
    assert o.se3_log_distance(Tc, res.T) < 1e-6
    assert any(G.analysis.is_degenerate for G in res.logs)          # planar scene: x / y / yaw weakly constrained


def test_icp_monte_carlo_trials_c5(ctx, cylinder):
    """BASELINE config C5 at test size: seeded perturbations of the cylinder pair (t ~ U[-1,1]^3 m, rpy ~ U[-3,3]^3 deg,
    seed 45), one independent run per trial (replicas; no collective), every final pose against the C oracle."""
    import dcreg_oracle_c as oc
    rng = np.random.default_rng(45)
    sc = oc.Scene(cylinder, cylinder)
    ctx.set_source(cylinder); ctx.set_target(cylinder, 1.0)
    prm = o.Params(kappa_target=10.0, conv_rot=1e-5, conv_trans=1e-3)
    cp = oc.make_params(kappa_target=10.0, conv_rot=1e-5, conv_trans=1e-3)
    for trial in range(12):
        t = rng.uniform(-1, 1, 3); rpy = np.radians(rng.uniform(-3, 3, 3))
        T0 = o.pose6d_to_matrix(t[0], t[1], t[2], rpy[0], rpy[1], rpy[2])
        st, conv, n_it, Tc, clogs = sc.icp_run(cp, T0)
        res = ctx.icp_run(gpu_params(prm), T0, want_log=False)
        assert res.status == st and res.converged == conv and res.iterations == n_it, trial
        assert o.se3_log_distance(Tc, res.T) < 1e-6, trial
    sc.close()


@pytest.mark.parametrize("thr", [0.2, 0.03])
def test_point_to_point_metrics_device(ctx, golden, cylinder, tree, thr):
    """Device P2P RMSE / fitness / Chamfer (exact 1-NN both ways) against the oracle and the shipped summary."""
    g = golden["G2"]
    conv, T, logs, status = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), params_from(g["setup"], "Ours"), tree)
    ctx.set_source(cylinder); ctx.set_target(cylinder, 1.0)
    for Tm in (T, init_T(g["setup"]), o.pose6d_to_matrix(30.0, -5.0, 2.0, 0.0, 0.0, 0.3)):   # aligned, initial, far away
        ref = o.point_to_point_metrics(cylinder, cylinder, Tm, thr, tree)
        got = ctx.point_to_point_metrics(Tm, thr)
        assert got["n_valid"] == ref["n_valid"]
        assert abs(got["rmse"] - ref["rmse"]) < 1e-9 and abs(got["chamfer"] - ref["chamfer"]) < 1e-9
        assert abs(got["fitness"] - ref["fitness"]) < 1e-12
    if thr == 0.2:
        got = ctx.point_to_point_metrics(T, thr)
        assert abs(got["rmse"] - 0.036217) < 2e-6 and abs(got["chamfer"] - 0.032915) < 2e-6


def test_icp_abort_not_enough_points(ctx, cylinder):
    from dcreg_b200 import api
    far = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)
    ctx.set_source(cylinder); ctx.set_target(cylinder, 1.0)
    res = ctx.icp_run(gpu_params(o.Params()), far)
    assert res.status == api.NOT_ENOUGH_POINTS and not res.converged and res.iterations == 1
    assert np.allclose(res.T, far)                                  # pose untouched, as in the reference


def test_bad_arguments(ctx):
    from dcreg_b200 import api
    with pytest.raises(api.DcregError) as e:
        ctx.set_source(np.zeros((0, 3), np.float32))
    assert e.value.status == api.BAD_ARG
    with pytest.raises(api.DcregError):
        ctx.set_target(np.zeros((10, 3), np.float32), 0.0)
