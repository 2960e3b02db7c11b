"""The rest of the solve step against the high-precision reference (oracle/dcreg_oracle_mp.py): the baseline methods'
analysis and solve (k2::analyze_and_solve<false> in k2::icp_step, run by k2_step_kernel), the log-only half of every
record (log_fill_kernel -> analyze_and_solve<true>, "Ours" records included), both pose updates (k2::boxplus and the
lane-spread one of icp_step_warp_ours) with the convergence decision, and the post-run covariance (covariance_kernel).

Per record, at every entry point:
  * seam identity, no mp needed: a baseline record's dx and analysis block are byte for byte what the host seam
    (dcreg_analyze_and_solve) computes from its H27 with the same settings; an "Ours" record's analysis is too, except
    the decisions the step itself wrote (mask, is_degenerate, schur_singular, PCG count and residual);
  * against analysis_reference (every K-th record on the batched calls): every field inside its bound, masks and
    branch equal on clear records, dx inside its bound; inside the band only the seam identity holds;
  * README's "Schur eigenvalues to 1e-8 relative": asserted where the reference's bound allows it, and the records
    where it cannot hold are counted with their worst relative error;
  * the pose: rec.T within boxplus_reference(T_{k-1}, rec.dx), an aborting record keeps T_{k-1} byte for byte with
    dx = 0, and `converged` / `iterations` follow from the records' dx wherever the threshold decision is clear.
Each test prints one line per label: records, records against mp, clear / band, worst error of each field in units of
its bound.
"""
import math

import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_mp as m
from test_gpu_k2_step import designed, run_designed

pytestmark = pytest.mark.gpu

METHODS = {                       # the six methods of the CLI's SO(3) path, and the two handled as plain QR
    "Ours": ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG"),
    "NONE": ("NONE_DETE", "NONE_HAND"),
    "ME-SR": ("FULL_EVD_MIN_EIGENVALUE", "SOLUTION_REMAPPING"),
    "FCN-SR": ("FULL_SVD_CONDITION", "SOLUTION_REMAPPING"),
    "ME-TSVD": ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD"),
    "ME-TReg": ("FULL_EVD_MIN_EIGENVALUE", "STANDARD_REGULARIZATION"),
}
QR_LIKE = {"ADAPTIVE": ("NONE_DETE", "ADAPTIVE_REGULARIZATION"), "EVD_SUB": ("EVD_SUB_CONDITION", "NONE_HAND")}
STATS = {}


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


def params(method, **over):
    from dcreg_b200 import default_params
    det, hand = {**METHODS, **QR_LIKE}[method]
    kw = dict(detection=det, handling=hand, kappa_target=10.0)
    kw.update(over)
    return default_params(**kw)


def is_ours(prm):
    return prm.detection == 1 and prm.handling == 3


def dev_fields(an):
    d = {n: np.array(getattr(an, n), dtype=np.float64).ravel() for n in m.ANALYSIS_FIELDS}
    for n in m.INT_FIELDS:
        d[n] = np.atleast_1d(np.array(getattr(an, n)))
    return d


def without_kept(a):
    """the analysis block's bytes with the decisions an "Ours" step writes itself zeroed"""
    b = type(a).from_buffer_copy(bytes(a))
    for k in range(6):
        b.degenerate_mask[k] = 0
    b.is_degenerate = b.schur_singular = b.pcg_iterations = 0
    b.pcg_residual = 0.0
    return bytes(b)


def stats(label):
    return STATS.setdefault(label, dict(records=0, mp=0, clear=0, band=0, schur_1e8=0, schur_not_1e8=0,
                                        schur_worst_rel=0.0, worst={}))


def note(st, name, v):
    st["worst"][name] = max(st["worst"].get(name, 0.0), v)


def report(label):
    s = STATS[label]
    print(f"{label}: {s['records']} records, {s['mp']} against mp ({s['clear']} clear, {s['band']} inside the band); "
          f"Schur 1e-8: {s['schur_1e8']} eigenvalues held to it, {s['schur_not_1e8']} where the bound cannot "
          f"(worst relative error there {s['schur_worst_rel']:.2g}); worst / bound: "
          + " ".join(f"{k}={v:.2g}" for k, v in sorted(s["worst"].items())))


def check_record(ctx, prm, rec, label, mp=True):
    """One OK record: seam identity, and against the reference when mp"""
    st = stats(label)
    st["records"] += 1
    H27 = np.array(rec.H27)
    a_seam, dx_seam, _ = ctx.analyze_and_solve(H27, prm)
    if not is_ours(prm):
        assert bytes(rec.analysis) == bytes(a_seam), (label, rec.iter)
        assert np.array(rec.dx).tobytes() == dx_seam.tobytes(), (label, rec.iter)
    else:
        assert without_kept(rec.analysis) == without_kept(a_seam), (label, rec.iter)
    if not mp:
        return None
    st["mp"] += 1
    ref = m.analysis_reference(H27, prm)
    got = dev_fields(rec.analysis)
    if is_ours(prm):                              # the step's own decisions: test_gpu_k2_step.py checks them
        for k in ("degenerate_mask", "is_degenerate"):
            ref.ints.pop(k, None)
    worst, bad = m.compare_analysis(ref, got)
    assert not bad, (label, rec.iter, bad[:3])
    for k, v in worst.items():
        note(st, k, v)
    st["clear" if ref.clear else "band"] += 1
    if ref.dx is not None and math.isfinite(ref.dx_bound):
        e = float(np.max(np.abs(np.array(rec.dx) - np.array(ref.dx))))
        assert e <= ref.dx_bound, (label, rec.iter, ref.branch, e, ref.dx_bound)
        note(st, "dx", e / ref.dx_bound if ref.dx_bound > 0 else 0.0)
    for nm in ("rot", "trans"):                   # README: Schur eigenvalues to 1e-8 relative
        r, b = ref.vals["lambda_schur_" + nm], ref.bound["lambda_schur_" + nm]
        for k in range(3):
            if not (math.isfinite(b[k]) and math.isfinite(r[k]) and r[k] != 0):
                continue
            rel = abs(got["lambda_schur_" + nm][k] - r[k]) / abs(r[k])
            if b[k] <= 1e-8 * abs(r[k]):
                st["schur_1e8"] += 1
                assert rel <= 1e-8, (label, rec.iter, nm, k, rel)
            else:
                st["schur_not_1e8"] += 1
                st["schur_worst_rel"] = max(st["schur_worst_rel"], rel)
    return ref


def check_pose_chain(prm, res, T_start, label):
    """rec.T = T_{k-1} Exp(dx_k) within the bound, aborts keep the pose, converged / iterations from the records.
    Returns the largest |R^T R - I| along the chain."""
    st = stats(label)
    T_prev = np.asarray(T_start, dtype=np.float64).reshape(4, 4)
    clear_conv = None
    for k, rec in enumerate(res.logs):
        T = np.array(rec.T).reshape(4, 4)
        if rec.status != 0:
            assert T.tobytes() == T_prev.tobytes() and not np.any(np.array(rec.dx)), (label, k)
            continue
        p = m.boxplus_reference(T_prev, np.array(rec.dx), prm.conv_thresh_rot, prm.conv_thresh_trans)
        eR = np.max(np.abs(T[:3, :3].ravel() - p.R)) / p.bound_R
        et = np.max(np.abs(T[:3, 3] - p.t)) / p.bound_t
        assert eR <= 1 and et <= 1, (label, k, eR, et)
        note(st, "T", max(eR, et))
        if p.clear and not prm.fixed_iterations:
            last = k == len(res.logs) - 1
            assert p.converged == (last and res.converged), (label, k, p.theta, p.vnorm, res.converged)
            clear_conv = p.converged
        T_prev = T
    if res.status == 0 and len(res.logs) == res.iterations and clear_conv is not None:
        assert res.converged or res.iterations == prm.max_iterations, (label, res.iterations)
    R = T_prev[:3, :3]
    return float(np.max(np.abs(R.T @ R - np.eye(3))))


def check_run(ctx, prm, res, T_start, label, mp_every=1):
    for i, rec in enumerate(res.logs):
        if rec.status == 0:
            check_record(ctx, prm, rec, label, mp=(i % mp_every == 0))
    return check_pose_chain(prm, res, T_start, label)


def check_cov(cov, prm, res, label):
    """The post-run covariance of a run against covariance_reference(H of its last OK record)"""
    st = stats(label)
    ok = [r for r in res.logs if r.status == 0]
    conv = bool(res.converged)
    if not conv:
        assert np.array_equal(cov, 1e6 * np.eye(6)), label
        note(st, "cov", 0.0)
        return None
    H, _ = o.unpack27(np.array(ok[-1].H27))
    c = m.covariance_reference(H.ravel(), conv)
    if c.clear:
        err = float(np.max(np.abs(np.asarray(cov).ravel() - np.array(c.cov))))
        assert err <= c.bound, (label, err, c.bound, c.floored)
        note(st, "cov", err / c.bound if c.bound else 0.0)
    return c


# ------------------------------------------------------------------------------------------------------------------
# 3a. records at every entry point
# ------------------------------------------------------------------------------------------------------------------
def g1_setup(golden):
    s = golden["G1"]["setup"]
    x, y, z = s["init_xyz"]
    r, p, yw = [math.radians(a) for a in s["init_rpy_deg"]]
    kw = dict(search_radius=s["search_radius"], max_iterations=s["max_iterations"], conv_thresh_rot=s["conv_rot"],
              conv_thresh_trans=s["conv_trans"], cond_thresh=s["cond_thresh"], kappa_target=s["kappa_target"],
              eig_thresh=s["eig_thresh"], std_reg_gamma=s["std_reg_gamma"],
              use_weight_derivative=int(s["use_weight_derivative"]))
    return kw, o.pose6d_to_matrix(x, y, z, r, p, yw)


def test_icp_run_every_method(ctx, golden, cylinder):
    kw, T0 = g1_setup(golden)
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    for meth in list(METHODS) + list(QR_LIKE):
        prm = params(meth, **kw)
        res = ctx.icp_run(prm, T0)
        assert res.status == 0 and res.logs
        check_run(ctx, prm, res, T0, "icp_run G1")
        check_cov(ctx.last_covariance(), prm, res, "icp_run G1")
        short = params(meth, **dict(kw, max_iterations=1))             # not converged: 1e6 I
        r1 = ctx.icp_run(short, T0)
        if not r1.converged:
            check_cov(ctx.last_covariance(), short, r1, "icp_run G1")
    report("icp_run G1")


def test_icp_run_corridor(ctx):
    from dcreg_b200.scenes import make_corridor
    pts = make_corridor(200_000, seed=44, noise=0.002)
    T0 = np.eye(4); T0[:3, 3] = [0.02, 0.015, -0.01]
    ctx.set_target(pts, 0.1)
    ctx.set_source(pts)
    for meth in ("Ours", "FCN-SR", "ME-TSVD"):
        prm = params(meth, search_radius=0.1, max_iterations=12, fixed_iterations=1)
        res = ctx.icp_run(prm, T0)
        worst = check_run(ctx, prm, res, T0, "icp_run corridor")
        print(f"corridor {meth}: |R^T R - I| = {worst:.2g} after {res.iterations} iterations")
    report("icp_run corridor")


def test_icp_run_host_planes(ctx):
    sysd = designed("generic")
    for meth in ("NONE", "ME-SR", "ME-TSVD", "FCN-SR", "ME-TReg", "Ours"):
        prm = params(meth, max_iterations=4, fixed_iterations=1, eig_thresh=50.0, cond_thresh=20.0, pcg_max_iter=2)
        res = run_designed(ctx, sysd, prm)
        check_run(ctx, prm, res, np.eye(4), "icp_run_host_planes")
    report("icp_run_host_planes")


def mixed(n, **kw):
    names = list(METHODS) + list(QR_LIKE)
    return [params(names[k % len(names)], **kw) for k in range(n)]


def test_icp_run_batch_mixed_lanes(ctx, cylinder):
    from dcreg_b200.scenes import g2_initial_pose, trial_poses
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    T = g2_initial_pose() @ trial_poses(16, seed=5, max_trans=0.3, max_rot_deg=2.0)
    entries = mixed(16, search_radius=1.0, max_iterations=30, use_weight_derivative=1, conv_thresh_rot=1e-5,
                    conv_thresh_trans=1e-3)
    longest = 0.0
    for b, r in enumerate(ctx.icp_run_batch(entries, T, want_log=True)):
        longest = max(longest, check_run(ctx, entries[b], r, T[b], "icp_run_batch", mp_every=3))
    report("icp_run_batch")


@pytest.fixture(scope="module")
def parking():
    from dcreg_b200.scenes import make_parking_frames, make_parking_pairs, make_parking_sequence
    frames, _, T_init, tgt = make_parking_frames(8, seed=51, n_scan=4_000)
    src, ptgt, _, P_init = make_parking_pairs(8, seed=55, n_scan=4_000)
    seq, S_true, _, deltas, _ = make_parking_sequence(5, seed=61, n_scan=4_000)
    return frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_true[:1]


def test_scans_pairs_sequences(ctx, parking):
    frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_init = parking
    kw = dict(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    ctx.set_target(tgt, 0.5)
    e = mixed(len(frames), **kw)
    for b, r in enumerate(ctx.icp_run_scans(e, frames, T_init, want_log=True, want_cov=True)):
        check_run(ctx, e[b], r, T_init[b], "icp_run_scans", mp_every=3)
        check_cov(r.cov, e[b], r, "icp_run_scans")
    e = mixed(len(src), **kw)
    for b, r in enumerate(ctx.icp_run_pairs(e, src, ptgt, P_init, want_log=True, want_cov=True)):
        check_run(ctx, e[b], r, P_init[b], "icp_run_pairs", mp_every=3)
        check_cov(r.cov, e[b], r, "icp_run_pairs")
    for meth in ("ME-SR", "ME-TSVD"):
        prm = params(meth, **kw)
        for r in ctx.icp_run_sequences(prm, [seq], S_init, deltas, want_log=True, want_cov=True):
            check_run(ctx, prm, r, r.T_prior, "icp_run_sequences", mp_every=3)
            check_cov(r.cov, prm, r, "icp_run_sequences")
    for lab in ("icp_run_scans", "icp_run_pairs", "icp_run_sequences"):
        report(lab)


def test_odometry_baseline(ctx):
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(6, seed=71, n_scan=8_000, max_range=20.0)
    prm = params("ME-SR", search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    res = ctx.icp_run_odometry(prm, [frames], T_true[:1], deltas, map_frames=3, cell_size=0.5, want_log=True)
    for r in res[1:]:
        check_run(ctx, prm, r, r.T_prior, "icp_run_odometry", mp_every=3)
    assert stats("icp_run_odometry")["mp"] > 0
    report("icp_run_odometry")


# ------------------------------------------------------------------------------------------------------------------
# 3b. designed systems at the seam: H = Q diag(lambda) Q^T rounded to doubles, thresholds swept through the values
# ------------------------------------------------------------------------------------------------------------------
def designed_H(lams, seed=0, zero=None):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    H = Q @ np.diag(lams) @ Q.T
    H = 0.5 * (H + H.T)
    g = Q @ rng.uniform(0.5, 1.5, 6) * np.sqrt(np.abs(np.asarray(lams, dtype=np.float64)) + 1.0)
    if zero is not None:
        H[zero, :] = 0.0; H[:, zero] = 0.0; g[zero] = 0.0
    return o.pack27(H, g)


def seam(ctx, v27, prm, label):
    """One seam call against the reference.  Returns the reference (with .seen: the device's mask and dx)"""
    st = stats(label)
    st["records"] += 1; st["mp"] += 1
    a, dx, rc = ctx.analyze_and_solve(v27, prm)
    ref = m.analysis_reference(v27, prm)
    worst, bad = m.compare_analysis(ref, dev_fields(a))
    assert not bad, (label, bad[:3])
    for k, v in worst.items():
        note(st, k, v)
    st["clear" if ref.clear else "band"] += 1
    if ref.dx is not None and math.isfinite(ref.dx_bound):
        e = float(np.max(np.abs(dx - np.array(ref.dx))))
        assert e <= ref.dx_bound, (label, ref.branch, e, ref.dx_bound)
        note(st, "dx", e / ref.dx_bound if ref.dx_bound > 0 else 0.0)
    ref.seen = (list(a.degenerate_mask), int(a.is_degenerate), dx)
    return ref


DELTAS = (1e-4, 1e-8, 1e-11)
LAMS = [3.0, 7.0, 40.0, 300.0, 2e3, 1e4]


def sweep_sides(refs):
    """both sides of every clear threshold were reached: per threshold value, the clear records give two masks"""
    return {tuple(r.mask) for r in refs if r.clear}


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 40, 2.0 ** -40])
def test_sweep_eig_thresh(ctx, scale):
    """ME: eig_thresh = lambda_i (1 +- delta) for every lambda_i, under SR, TSVD and TReg"""
    v27 = designed_H([l * scale for l in LAMS], seed=1)
    lab = f"seam eig_thresh x{scale:.3g}"
    for meth in ("ME-SR", "ME-TSVD", "ME-TReg"):
        base = m.analysis_reference(v27, params(meth, eig_thresh=1.0))
        for i in range(6):
            lam = float(base.lam[i])
            refs = [seam(ctx, v27, params(meth, eig_thresh=lam * (1 + s * d), std_reg_gamma=lam), lab)
                    for d in DELTAS for s in (1, -1)]
            # delta 1e-4: both sides are clear and differ in exactly mask[i]
            assert refs[0].clear and refs[1].clear and refs[0].mask[i] == 1 and refs[1].mask[i] == 0, (meth, i)
            for r in refs:
                if r.clear:
                    assert r.seen[0] == r.mask
    report(lab)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 40, 2.0 ** -40])
def test_sweep_cond_thresh(ctx, scale):
    """FCN: cond_thresh = cond_full (1 +- delta) and lambda_max / lambda_i (1 +- delta)"""
    v27 = designed_H([l * scale for l in LAMS], seed=2)
    lab = f"seam cond_thresh x{scale:.3g}"
    base = m.analysis_reference(v27, params("FCN-SR", cond_thresh=1.0))
    targets = [float(base.lam[5] / base.lam[i]) for i in range(5)]
    for c in targets:
        refs = [seam(ctx, v27, params("FCN-SR", cond_thresh=c * (1 + s * d)), lab) for d in DELTAS for s in (1, -1)]
        assert refs[0].clear and refs[1].clear and refs[0].mask != refs[1].mask
        for r in refs:
            if r.clear:
                assert r.seen[0] == r.mask and r.seen[1] == r.is_degenerate
    report(lab)


def test_std_reg_gamma(ctx):
    v27 = designed_H(LAMS, seed=3)
    lab = "seam std_reg_gamma"
    dxs = []
    for gam in (0.0, 1e-300, LAMS[0], 1e8):
        r = seam(ctx, v27, params("ME-TReg", eig_thresh=5.0, std_reg_gamma=gam), lab)
        assert r.clear and r.is_degenerate
        dxs.append(r.seen[2])
        r = seam(ctx, v27, params("ME-TReg", eig_thresh=1.0, std_reg_gamma=gam), lab)   # not degenerate: no gamma
        assert r.clear and not r.is_degenerate
    assert np.max(np.abs(dxs[2] - dxs[0])) > 1e-3 * np.max(np.abs(dxs[0]))
    report(lab)


def test_tsvd_sigma_cut(ctx):
    """sigma around 1e-9: the TSVD keeps the smallest position only above the cut"""
    lab = "seam TSVD 1e-9"
    kept = set()
    for d in DELTAS:
        for s in (1, -1):
            v27 = designed_H([1e-9 * (1 + s * d), 1.0, 2.0, 3.0, 4.0, 5.0], seed=4)
            # eig_thresh below everything: no mask, the cut alone decides
            r = seam(ctx, v27, params("ME-TSVD", eig_thresh=-1.0), lab)
            if r.clear:
                kept.add(float(abs(r.lam[0])) > 1e-9)
    assert kept == {True, False}
    report(lab)


@pytest.mark.parametrize("scale", [1.0, 2.0 ** 40, 2.0 ** -40])
def test_clusters_signs_and_zero_rows(ctx, scale):
    """equal eigenvalues masked whole and through the middle, a lambda of +-1e-14 lambda_max, an exactly zero row"""
    lab = f"seam clusters x{scale:.3g}"
    for lams in ([2.0, 2.0, 50.0, 50.0, 50.0, 900.0], [1e-14 * 900, 3.0, 3.0, 40.0, 300.0, 900.0],
                 [-1e-14 * 900, 3.0, 3.0, 40.0, 300.0, 900.0]):
        v27 = designed_H([l * scale for l in lams], seed=5)
        for meth in ("ME-SR", "ME-TSVD", "FCN-SR", "ME-TReg", "NONE", "Ours"):
            for thr in (10.0 * scale, 100.0 * scale, 1e4):      # whole clusters, through the 50-cluster's middle
                seam(ctx, v27, params(meth, eig_thresh=thr, cond_thresh=thr / scale), lab)
    for zero in (0, 4):                                           # the QR rank cut and schur_singular
        v27 = designed_H([l * scale for l in LAMS], seed=6, zero=zero)
        for meth in ("NONE", "ME-SR", "ME-TReg", "Ours"):
            r = seam(ctx, v27, params(meth, eig_thresh=1.0), lab)
            assert r.ints.get("schur_singular") == [1]
            if r.branch == "qr":
                assert r.clear and r.seen[2][zero] == 0.0
    report(lab)


# ------------------------------------------------------------------------------------------------------------------
# 3c. designed systems through the loop: both boxplus branches and the convergence thresholds
# ------------------------------------------------------------------------------------------------------------------
def scaled(sysd, f):
    p, nrm, rho = sysd
    return p, nrm, rho * f


@pytest.mark.parametrize("meth", ["NONE", "Ours"])
def test_boxplus_theta_branch(ctx, meth):
    """theta of the first step at 1e-10 (1 +- 1e-3): the small-angle branch and Rodrigues, each within the pose bound"""
    sysd = designed("generic")
    prm = params(meth, max_iterations=1, fixed_iterations=1, pcg_max_iter=2)
    th0 = np.linalg.norm(np.array(run_designed(ctx, sysd, prm).logs[0].dx[:3]))
    # the weights 1 - 0.9 |rho| change with the scale: a second pass at the small scale, where dx is linear in rho
    f = 1e-10 / th0
    f *= 1e-10 / np.linalg.norm(np.array(run_designed(ctx, scaled(sysd, f), prm).logs[0].dx[:3]))
    lab = f"boxplus theta {meth}"
    sides = set()
    T0 = o.pose6d_to_matrix(0.3, -0.2, 0.1, 0.2, -0.1, 0.4)
    for s in (1, -1):
        res = run_designed(ctx, scaled(sysd, f * (1 + s * 1e-3)), prm, T0=T0)
        th = np.linalg.norm(np.array(res.logs[0].dx[:3]))
        sides.add(th < 1e-10)
        check_run(ctx, prm, res, T0, lab)
    assert sides == {True, False}
    report(lab)


@pytest.mark.parametrize("meth", ["ME-SR", "Ours"])
def test_convergence_thresholds(ctx, meth):
    """conv_thresh_rot / _trans at the step's |omega| and |v| times (1 +- delta): the run stops after that step
    exactly when both comparisons hold (its normal equations do not depend on the pose, so every step is the same)"""
    sysd = designed("generic")
    prm = params(meth, max_iterations=1, fixed_iterations=1, pcg_max_iter=2, eig_thresh=50.0)
    dx = np.array(run_designed(ctx, sysd, prm).logs[0].dx)
    w, v = np.linalg.norm(dx[:3]), np.linalg.norm(dx[3:])
    lab = f"convergence {meth}"
    seen = set()
    for d in DELTAS:
        for sr in (1, -1):
            for st in (1, -1):
                q = params(meth, max_iterations=3, pcg_max_iter=2, eig_thresh=50.0,
                           conv_thresh_rot=w * (1 + sr * d), conv_thresh_trans=v * (1 + st * d))
                res = run_designed(ctx, sysd, q)
                check_run(ctx, q, res, np.eye(4), lab)
                p = m.boxplus_reference(np.eye(4), np.array(res.logs[0].dx), q.conv_thresh_rot, q.conv_thresh_trans)
                if p.clear:
                    seen.add(res.converged)
                if d == DELTAS[0]:                # later steps repeat dx to rounding, far inside 1e-4
                    assert p.clear and res.iterations == (1 if p.converged else 3), (d, sr, st)
    assert seen == {True, False}
    report(lab)


# ------------------------------------------------------------------------------------------------------------------
# 3d. covariance
# ------------------------------------------------------------------------------------------------------------------
def test_covariance_floor_straddles_1e12(ctx):
    """lambda_max(H) 30 % above and 30 % below 1e12 (a million host-plane points whose lever arm scales the rotation
    block): the floor decision goes both ways, each clear, and each covariance is the reference's.  (A room 4 km out
    also crosses 1e12, but its cond(H) of 5e13 puts lambda_min(H^-1) inside the band of the floor.)"""
    p, nrm, rho = designed("generic", n=1_000_000)
    lab = "covariance floor"
    prm = params("NONE", max_iterations=2, conv_thresh_rot=1e3, conv_thresh_trans=1e3)

    def run(L):
        res = run_designed(ctx, ((p * L).astype(np.float32), nrm, rho), prm)
        assert res.converged
        lam_max = float(np.max(np.linalg.eigvalsh(o.unpack27(np.array(res.logs[-1].H27))[0])))
        return res, lam_max

    _, lam1 = run(1.0)
    floors = set()
    for target in (1.3e12, 0.7e12):
        res, lam_max = run(math.sqrt(target / lam1))
        c = check_cov(ctx.last_covariance(), prm, res, lab)
        print(f"lambda_max(H) {lam_max:.4g}: floored {c.floored}, clear {c.clear}, floor margin {c.floor_margin:.3g}, "
              f"cond(H) {c.cond_H:.3g}")
        assert c.clear and c.floored == (lam_max > 1e12)
        floors.add(c.floored)
    assert floors == {True, False}
    report(lab)


def test_covariance_fullpiv_threshold(ctx):
    """A translation block of rank 2 (an exactly zero row of H): FullPivLU declares H singular, the run converged, and
    the covariance is 1e6 I; the same block tilted out of its plane by 1e-3 is invertible and gives H^-1"""
    lab = "covariance FullPivLU"
    for kind, tilt, singular in (("rank2", 0.0, True), ("tilt", 1e-3, False)):
        sysd = designed(kind, tilt=tilt)
        prm = params("NONE", max_iterations=2, conv_thresh_rot=1e3, conv_thresh_trans=1e3)
        res = run_designed(ctx, sysd, prm)
        assert res.converged
        c = check_cov(ctx.last_covariance(), prm, res, lab)
        assert c.clear and c.invertible == (not singular), (kind, c.pivot_ratio)
    report(lab)
