"""The "Ours" solve step that moves the pose (k2_solve.cuh: icp_step_warp_ours, in the loop kernel's solver block and in
k2_step_kernel) against the high-precision reference oracle/dcreg_oracle_mp.py, record by record.

The step has its own FP64 arithmetic (MUFU-seeded reciprocals, warm-started Jacobi, L D L^T block inverses, a
lane-parallel PCG with FMAs and a squared stop rule), so it is checked on the records it wrote:
  * branch: the step took QR iff rec.dx is, bit for bit, the seam's qr6 solution of the same H, g (the seam with
    detection NONE_DETE); the record's is_degenerate / mask / pcg_iterations must say so (they are the step's own);
  * clear margins (dcreg_oracle_mp: EIG_BAND 1e-12 of the eigenvalue scale, the PCG band max(1e-6 tol, 8 eps cond(H)
    ||g||), pivot ratio > PIVOT_CLEAR = 16 eps):
    branch, mask and PCG count are the reference's, and rec.dx is within DX_TOL * cond(H) * eps (relative, max-norm)
    of the reference's dx;
  * inside the band: only consistency (the record describes the step that ran).
Designed systems (host planes, K1 + k2_step_kernel) put thresholds on the system's own Schur ratios, clamps and PCG
residuals; pcg_max_iter 1-2 keeps the PCG and QR answers clearly apart.
"""
import math

import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_mp as m

pytestmark = pytest.mark.gpu

DX_TOL = 64.0          # rec.dx vs the reference: |dx - dx_ref|_max <= DX_TOL * cond(H) * eps * |dx_ref|_max
WORST = {}             # label -> [records, clear, checked against mp, worst dx error in units of cond(H) eps]


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


def ours(**over):
    from dcreg_b200 import default_params
    kw = dict(detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG", kappa_target=10.0)
    kw.update(over)
    return default_params(**kw)


def qr_params(prm):
    from dcreg_b200 import default_params
    q = default_params(detection="NONE_DETE", handling="PRECONDITIONED_CG")
    q.min_effective_points = prm.min_effective_points
    return q


def check_record(ctx, prm, rec, label, mp=True):
    """One record of an "Ours" run.  Returns the branch it took ("qr" / "pcg")."""
    H27 = np.array(rec.H27)
    dx = np.array(rec.dx)
    a = rec.analysis
    _, dx_qr, _ = ctx.analyze_and_solve(H27, qr_params(prm))
    took_qr = dx.tobytes() == dx_qr.tobytes()
    mask = list(a.degenerate_mask)
    assert a.is_degenerate == int(any(mask)), (label, rec.iter)
    assert a.is_degenerate == (0 if took_qr else 1), (label, rec.iter, mask)
    if took_qr:
        assert a.pcg_iterations == 0 and a.pcg_residual == 0.0, (label, rec.iter)
    else:
        assert 1 <= a.pcg_iterations <= max(prm.pcg_max_iter, 0) and a.schur_singular == 0, (label, rec.iter)
        if a.pcg_iterations < prm.pcg_max_iter:                       # it stopped on the tolerance
            assert a.pcg_residual <= prm.pcg_tol, (label, rec.iter, a.pcg_residual)
    stats = WORST.setdefault(label, [0, 0, 0, 0.0])
    stats[0] += 1
    if not mp:
        return "qr" if took_qr else "pcg"
    ref = m.step_reference(H27, prm.cond_thresh, prm.kappa_target, prm.pcg_tol, prm.pcg_max_iter)
    stats[2] += 1
    if all(ref.block_clear):             # FullPivLU's invertibility, decided from the block alone
        assert a.schur_singular == (0 if ref.schur_ok else 1), (label, rec.iter, ref.pivot_ratio)
    if ref.clear:
        stats[1] += 1
        assert mask == ref.mask, (label, rec.iter, mask, ref.mask, ref.mask_margin)
        assert took_qr == (not ref.is_degenerate), (label, rec.iter)
        assert a.pcg_iterations == ref.pcg_stop, (label, rec.iter, a.pcg_iterations, ref.pcg_stop)
        if ref.dx is not None and math.isfinite(ref.cond_H):
            x = np.array(m.to_float(ref.dx))
            e = np.max(np.abs(dx - x)) / (np.max(np.abs(x)) * ref.cond_H * m.EPS)
            stats[3] = max(stats[3], e)
            assert e < DX_TOL, (label, rec.iter, e)
    elif not took_qr and ref.pcg_x:
        # inside the band: the PCG iterate the record names is the reference's iterate of that count (the clamp is
        # continuous in lambda, so an in-band clamp or stop decision cannot move it by more than the margin)
        k = a.pcg_iterations
        assert abs(k - ref.pcg_stop) <= 1 or ref.pcg_stop == 0, (label, rec.iter, k, ref.pcg_stop)
        if ref.schur_ok and all(ref.block_clear) and k <= len(ref.pcg_x):
            x = np.array(m.to_float(ref.pcg_x[k - 1]))
            assert np.max(np.abs(dx - x)) <= 1e-6 * np.max(np.abs(x)), (label, rec.iter)
    return "qr" if took_qr else "pcg"


def check_run(ctx, prm, logs, label, mp_every=1):
    branches = []
    for i, rec in enumerate(logs):
        if rec.status != 0:
            continue
        branches.append(check_record(ctx, prm, rec, label, mp=(i % mp_every == 0)))
    return branches


def params_copy(prm, **over):
    from dcreg_b200 import IcpParams
    q = IcpParams.from_buffer_copy(prm)
    for k, v in over.items():
        setattr(q, k, v)
    return q


def assert_count_is_the_steps(rerun, prm, rec):
    """The logged PCG count is the number of iterations the step ran: rerun(prm') repeats the record's step (same H27,
    a cold start) in a one-iteration run; with pcg_max_iter = the logged count and no tolerance it must give the logged
    dx bit for bit.  When the tolerance stopped it (count < pcg_max_iter), one iteration fewer must give a different
    dx (past convergence to rounding, as when a zero tolerance runs out pcg_max_iter, more iterations change no bit)."""
    k = rec.analysis.pcg_iterations
    if not rec.analysis.is_degenerate:
        return
    again = rerun(params_copy(prm, pcg_max_iter=k, pcg_tol=0.0, max_iterations=1, fixed_iterations=1))
    assert np.array(again.H27).tobytes() == np.array(rec.H27).tobytes()
    assert np.array(again.dx).tobytes() == np.array(rec.dx).tobytes(), (rec.iter, k)
    if 1 < k < prm.pcg_max_iter:
        fewer = rerun(params_copy(prm, pcg_max_iter=k - 1, pcg_tol=0.0, max_iterations=1, fixed_iterations=1))
        assert np.array(fewer.dx).tobytes() != np.array(rec.dx).tobytes(), (rec.iter, k)


def report(label):
    n, clear, n_mp, worst = WORST[label]
    print(f"{label}: {n} records, {n_mp} against the mp reference, {clear} clear ({n_mp - clear} inside the band), "
          f"worst dx error {worst:.3g} cond(H) eps")


# ------------------------------------------------------------------------------------------------------------------
# the entry points, record by record
# ------------------------------------------------------------------------------------------------------------------
def test_icp_run_c2_and_corridor(ctx):
    from dcreg_b200.scenes import make_cylinder, make_corridor, g2_initial_pose
    pts = make_cylinder(100_000, seed=42)
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    prm = ours(search_radius=1.0, max_iterations=50, fixed_iterations=1, use_weight_derivative=0)
    res = ctx.icp_run(prm, g2_initial_pose())
    assert res.iterations == 50
    br = check_run(ctx, prm, res.logs, "icp_run C2")
    assert "pcg" in br
    assert_count_is_the_steps(lambda p: ctx.icp_run(p, g2_initial_pose()).logs[0], prm, res.logs[0])
    report("icp_run C2")
    pts = make_corridor(200_000, seed=44, noise=0.002)
    T0 = np.eye(4); T0[:3, 3] = [0.02, 0.015, -0.01]
    ctx.set_target(pts, 0.1)
    ctx.set_source(pts)
    prm = ours(search_radius=0.1, max_iterations=12, fixed_iterations=1)
    res = ctx.icp_run(prm, T0)
    br = check_run(ctx, prm, res.logs, "icp_run corridor")
    assert br and all(b == "pcg" for b in br)                       # degenerate in every iteration
    # iteration 0: the FP64 residual ends at ~8e-7 against tol 1e-6 in the 6th iteration (the exact one at 1e-52), so
    # the step's squared FMA rule and the seam's may part; the record must name the count the step ran
    assert_count_is_the_steps(lambda p: ctx.icp_run(p, T0).logs[0], prm, res.logs[0])
    seam = [ctx.analyze_and_solve(np.array(r.H27), prm)[0].pcg_iterations for r in res.logs]
    print("corridor PCG iterations, step:", [r.analysis.pcg_iterations for r in res.logs], "seam:", seam)
    report("icp_run corridor")


def test_icp_run_batch(ctx, cylinder):
    from dcreg_b200.scenes import trial_poses
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    prm = ours(max_iterations=30)
    batch = ctx.icp_run_batch(prm, trial_poses(8, seed=45), want_log=True)
    for b in batch:
        check_run(ctx, prm, b.logs, "icp_run_batch", mp_every=2)
    report("icp_run_batch")


@pytest.fixture(scope="module")
def parking():
    from dcreg_b200.scenes import make_parking_frames, make_parking_pairs, make_parking_sequence
    frames, _, T_init, tgt = make_parking_frames(4, seed=51, n_scan=4_000)
    src, ptgt, _, P_init = make_parking_pairs(3, seed=55, n_scan=4_000)
    seq, S_true, _, deltas, _ = make_parking_sequence(5, seed=61, n_scan=4_000)
    return frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_true[:1]


def test_scans_pairs_sequences(ctx, parking):
    frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_init = parking
    prm = ours(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    ctx.set_target(tgt, 0.5)
    for r in ctx.icp_run_scans(prm, frames, T_init, want_log=True):
        check_run(ctx, prm, r.logs, "icp_run_scans", mp_every=2)
    for r in ctx.icp_run_pairs(prm, src, ptgt, P_init, want_log=True):
        check_run(ctx, prm, r.logs, "icp_run_pairs", mp_every=2)
    for r in ctx.icp_run_sequences(prm, [seq], S_init, deltas, want_log=True):
        check_run(ctx, prm, r.logs, "icp_run_sequences", mp_every=2)
    for lab in ("icp_run_scans", "icp_run_pairs", "icp_run_sequences"):
        report(lab)


def test_odometry(ctx):
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(6, seed=71, n_scan=8_000, max_range=20.0)
    prm = ours(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    res = ctx.icp_run_odometry(prm, [frames], T_true[:1], deltas, map_frames=3, cell_size=0.5, want_log=True)
    for r in res[1:]:
        check_run(ctx, prm, r.logs, "icp_run_odometry", mp_every=2)
    report("icp_run_odometry")


# ------------------------------------------------------------------------------------------------------------------
# designed systems through the host-plane loop (K1 + k2_step_kernel)
# ------------------------------------------------------------------------------------------------------------------
def designed(kind, rng_seed=5, n=900, tilt=0.0):
    """Source points and world planes whose normal equations do not depend on the pose (to rounding): each point keeps
    its normal (rotated with the pose) and its residual rho.  Returns (points f32, normals, rho)."""
    rng = np.random.default_rng(rng_seed)
    if kind == "generic":                       # anisotropic translation and rotation blocks, all ratios distinct
        p = rng.uniform(-5.0, 5.0, (n, 3)) * np.array([1.0, 0.6, 0.3])
        u = rng.standard_normal((n, 3)) * np.array([1.0, 0.35, 0.12])
        nrm = u / np.linalg.norm(u, axis=1, keepdims=True)
        rho = rng.uniform(-2e-3, 2e-3, n)
    elif kind in ("box2", "box3"):              # axis-aligned faces of a symmetric box: equal Schur eigenvalues
        # every face point comes with its reflections in the face's two other coordinates, so the coupling H_Rt and
        # the off-diagonal entries vanish; box3: the same count per axis (H_tt = c I), box2: fewer on the z faces
        per = n // 24
        ext = np.array([4.0, 4.0, 0.5])
        p, nrm = [], []
        for ax in range(3):
            cnt = per if kind == "box3" or ax < 2 else max(1, per // 20)
            for sgn in (-1.0, 1.0):
                q = rng.uniform(-1.0, 1.0, (cnt, 3)) * ext
                q[:, ax] = sgn * ext[ax]
                for f in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
                    s = np.ones(3); s[[a for a in range(3) if a != ax]] = f
                    p.append(q * s); nrm.append(np.tile(np.eye(3)[ax] * sgn, (cnt, 1)))
        p, nrm = np.concatenate(p), np.concatenate(nrm)
        rho = 1e-3 * rng.choice([-1.0, 1.0], len(p))                    # |rho| equal: every point has the same weight
    elif kind in ("rank2", "rank2_rot", "tilt"):   # translation block of rank 2 (+ tilt out of the plane)
        p = rng.uniform(-5.0, 5.0, (n, 3))
        ang = rng.uniform(0.0, 2.0 * math.pi, n)
        nrm = np.stack([np.cos(ang), np.sin(ang), np.zeros(n)], axis=1)
        if kind == "tilt":
            nrm[:, 2] = tilt * np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
            nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        if kind == "rank2_rot":
            Rg = o.pose6d_to_matrix(0, 0, 0, 0.7, -0.4, 1.1)[:3, :3]
            nrm = nrm @ Rg.T
        rho = rng.uniform(-2e-3, 2e-3, n)
    else:
        raise ValueError(kind)
    return p.astype(np.float32), nrm, rho


def run_designed(ctx, sysd, prm, T0=None):
    p, nrm, rho = sysd
    p64 = p.astype(np.float64)

    def plane_fn(T):
        R, t = T[:3, :3], T[:3, 3]
        q = (p64 @ R.T + t).astype(np.float32).astype(np.float64)          # fl32(R p + t), as K1 forms it
        nw = nrm @ R.T
        planes = np.empty((len(p), 4))
        planes[:, :3] = nw
        planes[:, 3] = rho - np.einsum("kj,kj->k", nw, q)
        return planes, len(p)

    ctx.set_source(p)
    return ctx.icp_run_host_planes(prm, np.eye(4) if T0 is None else T0, plane_fn)


def sweep(ctx, sysd, label, prms, iters, mp_at):
    out = []
    for prm in prms:
        prm.max_iterations = iters
        prm.fixed_iterations = 1
        res = run_designed(ctx, sysd, prm)
        out.append(res)
        for rec in res.logs:
            if rec.status == 0:
                check_record(ctx, prm, rec, label, mp=rec.iter in mp_at)
    return out


COLD_WARM = (0, 1, 2, 63, 64, 65, 129)


def base_reference(ctx, sysd, **over):
    prm = ours(max_iterations=1, fixed_iterations=1, **over)
    res = run_designed(ctx, sysd, prm)
    return m.step_reference(np.array(res.logs[0].H27), prm.cond_thresh, prm.kappa_target, prm.pcg_tol, prm.pcg_max_iter)


def assert_branches_differ(ctx, sysd, **over):
    """With a short PCG the two branches give clearly different dx on this system."""
    prm = ours(max_iterations=1, fixed_iterations=1, **over)
    rec = run_designed(ctx, sysd, prm).logs[0]
    _, dx_qr, _ = ctx.analyze_and_solve(np.array(rec.H27), qr_params(prm))
    assert rec.analysis.is_degenerate == 1
    assert np.max(np.abs(np.array(rec.dx) - dx_qr)) > 1e-3 * np.max(np.abs(dx_qr))


def test_sweep_cond_thresh(ctx):
    sysd = designed("generic")
    ref = base_reference(ctx, sysd, pcg_max_iter=2)
    assert ref.clear and ref.is_degenerate
    assert_branches_differ(ctx, sysd, pcg_max_iter=2)
    ratios = sorted({r for i, r in enumerate(ref.cond_ratio) if i % 3 != 2})
    prms = [ours(cond_thresh=rho * (1 + s * d), pcg_max_iter=2) for rho in ratios for d in (1e-4, 1e-8, 1e-11)
            for s in (1, -1)]
    runs = sweep(ctx, sysd, "sweep cond_thresh", prms, 130, COLD_WARM)
    # just under the largest ratio the step is degenerate, just over it not: both branches are taken
    assert runs[-6].logs[0].analysis.is_degenerate == 0 and runs[-5].logs[0].analysis.is_degenerate == 1
    report("sweep cond_thresh")


def test_sweep_kappa_target(ctx):
    sysd = designed("generic")
    ref = base_reference(ctx, sysd, pcg_max_iter=2)
    ratios = sorted({r for i, r in enumerate(ref.cond_ratio) if i % 3 != 2})
    assert_branches_differ(ctx, sysd, pcg_max_iter=2, cond_thresh=2.0, kappa_target=ratios[0])
    prms = [ours(kappa_target=rho * (1 + s * d), pcg_max_iter=2, cond_thresh=2.0) for rho in ratios
            for d in (1e-4, 1e-8, 1e-11) for s in (1, -1)]
    runs = sweep(ctx, sysd, "sweep kappa_target", prms, 130, COLD_WARM)
    # kappa = rho_i (1 -+ 1e-4): lambda_i is clamped on one side and not on the other.  The two sides' dx differ, and by
    # what the reference says they differ: a clamp in the wrong place or at the wrong value moves that difference
    for j, rho in enumerate(ratios):
        lo, hi = runs[6 * j + 1], runs[6 * j]                         # kappa below / above rho_i
        refs = [m.step_reference(np.array(r.logs[0].H27), p.cond_thresh, p.kappa_target, p.pcg_tol, p.pcg_max_iter)
                for r, p in ((lo, prms[6 * j + 1]), (hi, prms[6 * j]))]
        assert all(r.clear for r in refs)
        i = [abs(r - rho) for r in refs[0].cond_ratio].index(min(abs(r - rho) for r in refs[0].cond_ratio))
        lam_i, lam_max = refs[0].lam[i // 3][i % 3], refs[0].lam[i // 3][2]
        assert lam_i < lam_max / prms[6 * j + 1].kappa_target and lam_i > lam_max / prms[6 * j].kappa_target
        d_dev = np.array(lo.logs[0].dx) - np.array(hi.logs[0].dx)
        d_ref = np.array(m.to_float(refs[0].dx)) - np.array(m.to_float(refs[1].dx))
        assert np.max(np.abs(d_ref)) > 1e-7 * np.max(np.abs(np.array(hi.logs[0].dx)))
        assert np.max(np.abs(d_dev - d_ref)) <= 1e-3 * np.max(np.abs(d_ref)), (rho, d_dev, d_ref)
    report("sweep kappa_target")


def test_sweep_pcg_tol(ctx):
    sysd = designed("generic")
    ref = base_reference(ctx, sysd, pcg_max_iter=8)
    rn = [float(v) for v in ref.pcg_rnorm[:5]]
    prms = [ours(pcg_tol=r * (1 + s * d), pcg_max_iter=8) for r in rn for d in (1e-4, 1e-8, 1e-11) for s in (1, -1)]
    prms += [ours(pcg_tol=0.0, pcg_max_iter=8), ours(pcg_tol=1e-170, pcg_max_iter=8)]
    runs = sweep(ctx, sysd, "sweep pcg_tol", prms, 3, (0, 1, 2))
    for r, p in zip(runs, prms):
        assert_count_is_the_steps(lambda q: run_designed(ctx, sysd, q).logs[0], p, r.logs[0])
    its = {r.logs[0].analysis.pcg_iterations for r in runs}
    assert len(its) >= 5                                              # the stop moves with the tolerance
    assert runs[-1].logs[0].analysis.pcg_iterations == 8 and runs[-2].logs[0].analysis.pcg_iterations == 8
    report("sweep pcg_tol")


@pytest.mark.parametrize("kind,kappa", [("box2", 3.0), ("box3", 1.5)])
def test_equal_schur_eigenvalues(ctx, kind, kappa):
    """box2: two translation eigenvalues equal; box3: all three.  kappa below the rotation block's ratios, so P is
    not H^-1 and two PCG iterations stop short of the QR answer."""
    sysd = designed(kind)
    ref = base_reference(ctx, sysd, pcg_max_iter=2, kappa_target=kappa, cond_thresh=2.0)
    assert ref.is_degenerate
    lam = [float(v) for v in ref.lam[1]]
    assert abs(lam[2] - lam[1]) <= 1e-12 * lam[2]                    # at least two translation eigenvalues equal
    assert_branches_differ(ctx, sysd, pcg_max_iter=2, kappa_target=kappa, cond_thresh=2.0)
    prm = ours(pcg_max_iter=2, kappa_target=kappa, cond_thresh=2.0)
    sweep(ctx, sysd, "equal eigenvalues " + kind, [prm], 130, COLD_WARM)
    report("equal eigenvalues " + kind)


def test_rank2_translation_blocks(ctx):
    from dcreg_b200.api import NONFINITE_UPDATE
    # exactly rank 2 and axis-aligned: H_tt has a zero row, clearly singular, QR branch
    res = sweep(ctx, designed("rank2"), "rank-2 axis-aligned", [ours(pcg_max_iter=2)], 3, (0,))
    assert all(r.analysis.schur_singular == 1 and r.analysis.is_degenerate == 0 for r in res[0].logs if r.status == 0)
    # rank 2 under a generic rotation: at FullPivLU's threshold, consistency only; a non-finite abort only where the
    # seam's dx is non-finite too
    res = sweep(ctx, designed("rank2_rot"), "rank-2 rotated", [ours(pcg_max_iter=2)], 3, (0,))[0]
    for rec in res.logs:
        if rec.status == NONFINITE_UPDATE:
            _, dx_seam, _ = ctx.analyze_and_solve(np.array(rec.H27), ours(pcg_max_iter=2))
            assert not np.all(np.isfinite(dx_seam))
    # tilted out of the plane by eps: the smallest pivot ratio sweeps down through 3 eps
    ratios = []
    # ratio ~ 2 tilt^2: coarse from 1e-3, then steps of 1.5x in the ratio through [3 eps, 64 eps]
    for e in np.concatenate([np.logspace(-3, -6, 4)[:-1], np.logspace(-6, -8.5, 30)]):
        sysd = designed("tilt", tilt=float(e))
        ref = base_reference(ctx, sysd, pcg_max_iter=2)
        ratios.append(ref.pivot_ratio[1])
        sweep(ctx, sysd, "tilt sweep", [ours(pcg_max_iter=2)], 2, (0, 1))
    assert max(ratios) > 1e-8 and min(ratios) < 3 * m.EPS
    report("rank-2 rotated")
    report("tilt sweep")


def test_cold_restart_every_64_iterations(ctx):
    """The Jacobi starts warm from the previous iteration's eigenvectors and cold every 64 iterations.  Iteration 64 of a
    run is therefore bit for bit a fresh run's iteration 0 from the same pose (same H27, cold start), while a warm
    iteration is not (the warm start changes the last bits of V, hence of P and dx)."""
    sysd = designed("generic")
    prm = ours(pcg_max_iter=2, max_iterations=66, fixed_iterations=1)
    res = run_designed(ctx, sysd, prm)
    one = params_copy(prm, max_iterations=1)

    def fresh(k, p=one):
        return run_designed(ctx, sysd, p, T0=np.array(res.logs[k - 1].T).reshape(4, 4)).logs[0]

    r64 = fresh(64)
    assert np.array(r64.H27).tobytes() == np.array(res.logs[64].H27).tobytes()
    assert np.array(r64.dx).tobytes() == np.array(res.logs[64].dx).tobytes()
    assert_count_is_the_steps(lambda q: fresh(64, q), prm, res.logs[64])
    warm = [fresh(k) for k in (1, 2, 33, 63)]
    assert all(np.array(w.H27).tobytes() == np.array(res.logs[k].H27).tobytes() for w, k in zip(warm, (1, 2, 33, 63)))
    assert any(np.array(w.dx).tobytes() != np.array(res.logs[k].dx).tobytes() for w, k in zip(warm, (1, 2, 33, 63)))
