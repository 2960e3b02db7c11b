"""The high-precision reference of the "Ours" step (oracle/dcreg_oracle_mp.py) against the FP64 NumPy oracle
(dcreg_oracle.analyze_degeneracy / solve_degenerate_system) on every record of the G1 and G2 registrations.

Both evaluate the same mathematics, so on records whose decisions are clear of the band they must agree on the mask,
the PCG iteration count and the branch, and the FP64 values must sit within rounding of the exact ones: eigenvalues
within EIG_BAND * scale (which is what justifies the band), P and dx within a bound from the conditioning.
"""
import copy
import math

import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_mp as m
from harness import METHODS, oracle_method


def _records(golden, cylinder, name, **over):
    s = golden[name]["setup"]
    x, y, z = s["init_xyz"]
    r, p, yw = [math.radians(a) for a in s["init_rpy_deg"]]
    prm = o.Params(search_radius=s["search_radius"], max_iterations=s["max_iterations"], conv_rot=s["conv_rot"],
                   conv_trans=s["conv_trans"], cond_thresh=s["cond_thresh"], kappa_target=s["kappa_target"],
                   use_weight_derivative=s["use_weight_derivative"])
    for k, v in over.items():
        setattr(prm, k, v)
    _, _, logs, status = o.icp_so3(cylinder, cylinder, o.pose6d_to_matrix(x, y, z, r, p, yw), prm)
    assert status == "ok" and len(logs) >= 3
    return prm, logs


@pytest.mark.parametrize("name,over", [("G1", {}), ("G2", {}), ("G2", {"kappa_target": 1.0, "pcg_max_iter": 3})])
def test_mp_reference_matches_fp64_oracle(golden, cylinder, name, over):
    prm, logs = _records(golden, cylinder, name, **over)
    worst = {"eig/scale": 0.0, "P": 0.0, "dx/(cond eps)": 0.0}
    n_clear = 0
    for L in logs:
        H, g = L.H, L.g
        ref = m.step_reference(o.pack27(H, g), prm.cond_thresh, prm.kappa_target, prm.pcg_tol, prm.pcg_max_iter)
        a = o.analyze_degeneracy(H, prm)
        dx = o.solve_degenerate_system(H, g, prm, a)
        assert ref.schur_ok and all(ref.block_clear)
        for blk, lam in enumerate((a.lambda_schur_rot, a.lambda_schur_trans)):
            err = np.max(np.abs(lam - np.array([float(v) for v in ref.lam[blk]]))) / float(ref.scale[blk])
            worst["eig/scale"] = max(worst["eig/scale"], err)
            assert err < m.EIG_BAND                               # the band covers FP64's eigenvalue error
        P = np.array(ref.P.tolist(), dtype=np.float64)
        worst["P"] = max(worst["P"], np.max(np.abs(a.P - P)) / np.max(np.abs(P)))
        assert np.max(np.abs(a.P - P)) < 1e-9 * np.max(np.abs(P))
        if not ref.clear:
            continue
        n_clear += 1
        assert [int(v) for v in a.mask] == ref.mask and int(a.is_degenerate) == ref.is_degenerate
        assert a.pcg_iterations == ref.pcg_stop
        x = np.array(m.to_float(ref.dx))
        e = np.max(np.abs(dx - x)) / (np.max(np.abs(x)) * ref.cond_H * m.EPS)
        worst["dx/(cond eps)"] = max(worst["dx/(cond eps)"], e)
        assert e < 64.0
    print(name, over, f"{len(logs)} records, {n_clear} clear, worst", worst)
    assert n_clear >= len(logs) - 1
    assert any(L.analysis.is_degenerate for L in logs)            # the PCG branch is exercised


def test_mp_reference_reports_margins_and_branches():
    """Designed systems: a threshold placed on a Schur ratio is inside the band, one far away is clear; a rank-2
    axis-aligned translation block is clearly singular (QR branch, Schur singular)."""
    rng = np.random.default_rng(3)
    A = rng.standard_normal((40, 6))
    A[:, 5] *= 1e-2
    H, g = A.T @ A, A.T @ rng.standard_normal(40)
    v27 = o.pack27(H, g)
    ref = m.step_reference(v27, cond_thresh=10.0, kappa_target=10.0)
    assert ref.clear and ref.is_degenerate and ref.mask[3] == 1 and ref.pcg_stop > 0
    rho = ref.cond_ratio[3]
    on = m.step_reference(v27, cond_thresh=rho * (1 + 1e-14), kappa_target=10.0)
    assert not on.clear and min(on.mask_margin) < m.EIG_BAND
    near = m.step_reference(v27, cond_thresh=rho * (1 + 1e-4), kappa_target=10.0)
    assert near.clear and near.mask[3] == 0
    # PCG stop margins: a tolerance equal to ||r_2|| stops at 3 in exact arithmetic, inside the band
    r2 = float(ref.pcg_rnorm[1])
    t = m.step_reference(v27, cond_thresh=10.0, kappa_target=10.0, pcg_tol=r2)
    assert t.pcg_stop == 3 and not t.clear
    t = m.step_reference(v27, cond_thresh=10.0, kappa_target=10.0, pcg_tol=r2 * (1 + 1e-3))
    assert t.pcg_stop == 2 and t.clear
    # axis-aligned rank-2 translation block: exactly singular
    B = A.copy()
    B[:, 5] = 0.0
    ref = m.step_reference(o.pack27(B.T @ B, B.T @ rng.standard_normal(40)))
    assert not ref.schur_ok and ref.block_clear == [True, True] and not ref.is_degenerate and ref.x_qr is None


# ------------------------------------------------------------------------------------------------------------------
# every analysis field, the baseline methods, the pose update and the covariance (dcreg_oracle_mp.analysis_reference,
# boxplus_reference, covariance_reference) against the FP64 oracle, and the slips those checks must catch
# ------------------------------------------------------------------------------------------------------------------
def align_fp64(V, sign_fix=True):
    """FP64 twin of k2_solve.cuh's align_axes (V: 3x3, eigenvectors in columns)"""
    used_v, used_e, ind = set(), set(), [0, 0, 0]
    for _ in range(3):
        best = max(((abs(V[j, i]), i, j) for j in range(3) if j not in used_e for i in range(3) if i not in used_v),
                   key=lambda c: c[0])
        used_v.add(best[1]); used_e.add(best[2]); ind[best[2]] = best[1]
    Va = np.zeros((3, 3))
    for j in range(3):
        v = V[:, ind[j]].copy()
        if sign_fix and v[j] < 0:
            v = -v
        for k in range(j):
            v = v - (v @ Va[:, k]) * Va[:, k]
        Va[:, j] = v / np.linalg.norm(v)
    return Va, ind


def oracle_fields(a, sign_fix=True):
    """The FP64 oracle's Analysis under dcreg_analysis' field names"""
    d = {n: np.atleast_1d(np.asarray(getattr(a, n), dtype=np.float64)).ravel()
         for n in ("eigenvalues_full", "singular_values", "cond_full", "cond_full_sub_rot", "cond_full_sub_trans",
                   "lambda_sub_rot", "lambda_sub_trans", "cond_diag_rot", "cond_diag_trans", "lambda_schur_rot",
                   "lambda_schur_trans", "cond_schur_rot", "cond_schur_trans")}
    d["schur_V_rot"], d["schur_V_trans"] = a.schur_V_rot.ravel(), a.schur_V_trans.ravel()
    for nm in ("rot", "trans"):
        Va, ind = align_fp64(getattr(a, "schur_V_" + nm), sign_fix)
        d["aligned_V_" + nm], d[nm + "_indices"] = Va.ravel(), ind
    d["P_preconditioner"] = a.P.ravel()
    d["degenerate_mask"] = [int(v) for v in a.mask]
    d["is_degenerate"] = [int(a.is_degenerate)]
    d["schur_singular"] = [0]
    return d


def _method_runs(golden, cylinder):
    out = []
    for name in ("G1", "G2"):
        s = golden[name]["setup"]
        for meth in METHODS:
            det, hand = oracle_method(meth)
            x, y, z = s["init_xyz"]
            r, p, yw = [math.radians(v) for v in s["init_rpy_deg"]]
            prm = o.Params(search_radius=s["search_radius"], max_iterations=s["max_iterations"], conv_rot=s["conv_rot"],
                           conv_trans=s["conv_trans"], cond_thresh=s["cond_thresh"], kappa_target=s["kappa_target"],
                           use_weight_derivative=s["use_weight_derivative"], eig_thresh=s["eig_thresh"],
                           std_reg_gamma=s["std_reg_gamma"], detection=det, handling=hand)
            _, _, logs, status = o.icp_so3(cylinder, cylinder, o.pose6d_to_matrix(x, y, z, r, p, yw), prm)
            assert status == "ok" and logs, (name, meth)
            out.append((name, meth, prm, logs))
    return out


@pytest.fixture(scope="module")
def method_runs(golden, cylinder):
    return _method_runs(golden, cylinder)


def dx_error(ref, dx):
    return float(np.max(np.abs(np.asarray(dx) - np.asarray(ref.dx))))


def test_analysis_reference_matches_fp64_oracle(method_runs):
    """On every record of G1 and G2 under each of the six methods: every analysis field of the FP64 oracle inside its
    bound, masks and branches equal on clear records, dx inside its bound, the pose inside boxplus_reference's."""
    total = {}
    for name, meth, prm, logs in method_runs:
        worst, n_clear = {}, 0
        for k, L in enumerate(logs):
            ref = m.analysis_reference(o.pack27(L.H, L.g), prm)
            w, bad = m.compare_analysis(ref, oracle_fields(L.analysis))
            assert not bad, (name, meth, k, bad[:3])
            for f, v in w.items():
                worst[f] = max(worst.get(f, 0.0), v)
            if ref.dx is not None and math.isfinite(ref.dx_bound):
                n_clear += 1
                e = dx_error(ref, L.dx)
                assert e <= ref.dx_bound, (name, meth, k, e, ref.dx_bound)
                worst["dx"] = max(worst.get("dx", 0.0), e / ref.dx_bound if ref.dx_bound else 0.0)
            if k > 0:
                p = m.boxplus_reference(logs[k - 1].T, L.dx, prm.conv_rot, prm.conv_trans)
                e = max(np.max(np.abs(L.T[:3, :3].ravel() - p.R)) / p.bound_R, np.max(np.abs(L.T[:3, 3] - p.t)) / p.bound_t)
                assert e <= 1.0, (name, meth, k, e)
                worst["T"] = max(worst.get("T", 0.0), e)
                if p.clear:
                    assert not p.converged or k == len(logs) - 1, (name, meth, k)     # a converged step ends the run
        print(f"{name} {meth}: {len(logs)} records, {n_clear} with dx clear, worst / bound "
              + " ".join(f"{f}={v:.2g}" for f, v in sorted(worst.items())))
        total[meth] = total.get(meth, 0) + n_clear
        if meth != "Ours":
            assert n_clear >= len(logs) - 1, (name, meth)
    assert all(total[k] > 0 for k in METHODS if k != "Ours")
    # both sides of the ME threshold and a degenerate TReg / SR / TSVD step occur in these runs
    assert any(L.analysis.is_degenerate for _, meth, _, logs in method_runs if meth == "ME-TSVD" for L in logs)


def _mutants(prm, L, ref):
    """(slip, what it produces) for the record L of the FP64 oracle: each must fail the checks somewhere"""
    a, H, g = L.analysis, L.H, L.g
    lam, V = a.eigenvalues_full, a.eigenvectors_full
    out = []
    f = oracle_fields(a)
    phys = [0] * 6                                    # the mask indexed by the physical axis of each eigenvector
    for i in range(6):
        if a.mask[i]:
            phys[int(np.argmax(np.abs(V[:, i])))] = 1
    out.append(("mask by physical axis", dict(f, degenerate_mask=phys), None))
    order = np.argsort(-np.abs(lam), kind="stable")
    out.append(("mask by sigma order", dict(f, degenerate_mask=[int(a.mask[order[i]]) for i in range(6)]), None))
    if prm.handling == o.HAND_TRUNCATED_SVD:           # TSVD pairing "fixed": mask of sigma_i's own eigenvector
        x = np.zeros(6)
        for i in range(6):
            e = order[i]
            if not a.mask[e] and a.singular_values[i] > 1e-9:
                x += V[:, e] * (V[:, e] @ g) / a.singular_values[i] * np.sign(lam[e])
        out.append(("TSVD pairing fixed", None, x))
    if prm.handling == o.HAND_SOLUTION_REMAPPING and a.is_degenerate:     # SR keeps one more vector
        kept = [not v for v in a.mask]
        extra = max((i for i in range(6) if not kept[i]), key=lambda i: lam[i])
        kept[extra] = True
        x0 = o.qr_solve(H, g)
        out.append(("SR keeps one extra", None, sum(V[:, i] * (V[:, i] @ x0) for i in range(6) if kept[i])))
    if prm.handling == o.HAND_STANDARD_REGULARIZATION:  # under an eig_thresh no eigenvalue is below: not degenerate
        low = copy.copy(prm)
        low.eig_thresh = float(lam[0]) / 2
        ref = m.analysis_reference(o.pack27(H, g), low)
        assert ref.clear and not ref.is_degenerate
        out.append(("gamma when not degenerate", None, o.qr_solve(H + prm.std_reg_gamma * np.eye(6), g), ref))
    Vf = a.schur_V_rot.copy()                         # a sign flip that reaches aligned_V (no sign fix)
    Vf[:, 0] = -Vf[:, 0]; Vf[:, 1] = -Vf[:, 1]; Vf[:, 2] = -Vf[:, 2]
    Va, _ = align_fp64(Vf, sign_fix=False)
    out.append(("sign flip into aligned_V", dict(f, aligned_V_rot=Va.ravel()), None))
    return [c if len(c) == 4 else c + (ref,) for c in out]


def test_slips_fail_the_checks(method_runs):
    caught = {}
    for name, meth, prm, logs in method_runs:
        for k, L in enumerate(logs):
            ref = m.analysis_reference(o.pack27(L.H, L.g), prm)
            for slip, fields, dx, ref in _mutants(prm, L, ref):
                hit = caught.setdefault(slip, [0, 0])
                hit[1] += 1
                if fields is not None:
                    hit[0] += bool(m.compare_analysis(ref, fields)[1])
                elif ref.dx is not None and math.isfinite(ref.dx_bound):
                    hit[0] += dx_error(ref, dx) > ref.dx_bound
            if k > 0:                                 # the pose update: t + R_new v, a transposed Exp
                Tp = logs[k - 1].T
                p = m.boxplus_reference(Tp, L.dx)
                Rn = Tp[:3, :3] @ o.so3_exp(L.dx[:3])
                for slip, R, t in (("t + R_new v", Rn, Tp[:3, 3] + Rn @ L.dx[3:]),
                                   ("transposed Exp", Tp[:3, :3] @ o.so3_exp(L.dx[:3]).T, Tp[:3, 3] + Tp[:3, :3] @ L.dx[3:])):
                    hit = caught.setdefault(slip, [0, 0])
                    hit[1] += 1
                    hit[0] += bool(np.max(np.abs(R.ravel() - p.R)) > p.bound_R or np.max(np.abs(t - p.t)) > p.bound_t)
    print({k: f"{v[0]}/{v[1]}" for k, v in caught.items()})
    for slip in ("mask by physical axis", "mask by sigma order", "TSVD pairing fixed", "SR keeps one extra",
                 "gamma when not degenerate", "sign flip into aligned_V", "t + R_new v", "transposed Exp"):
        assert caught[slip][0] > 0, (slip, caught.get(slip))


def _designed(lams, seed=0):
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.standard_normal((6, 6)))
    H = Q @ np.diag(lams) @ Q.T
    return 0.5 * (H + H.T)


def _cov_fp64(H, floor="as released"):
    inv = np.linalg.inv(H)
    lam, V = np.linalg.eigh(0.5 * (inv + inv.T))
    if floor == "always" or (floor == "as released" and lam[0] <= 1e-12):
        return V @ np.diag(np.maximum(lam, 1e-9)) @ V.T
    return inv


@pytest.mark.parametrize("lams,floored,slip", [
    ([3e11, 4e11, 6e11, 8e11, 1.2e12, 2e12], True, "never"),       # lambda_max(H) > 1e12: floored
    ([1e10, 2e10, 5e10, 1e11, 2e11, 5e11], False, "always"),       # < 1e12, every eigenvalue of H^-1 under 1e-9
    ([3e2, 1e3, 5e3, 2e4, 1e11, 2e12], True, None),                 # cond 7e9: floored, inside the cond(H) bound
])
def test_covariance_reference_and_its_slips(lams, floored, slip):
    """lambda_max(H) on both sides of 1e12 decides the floor.  Without the floor, or with it always on, the covariance
    of a well-conditioned H leaves its bound (the floor moves eigenvalues far above cond(H) eps ||H^-1||)."""
    H = _designed(lams)
    c = m.covariance_reference(H.ravel(), True)
    assert c.clear and c.invertible and c.floored == floored
    err = np.max(np.abs(_cov_fp64(H).ravel() - c.cov))
    print(lams[-1], "cov error / bound", err / c.bound, "floor margin", c.floor_margin)
    assert err <= c.bound
    if slip:
        assert np.max(np.abs(_cov_fp64(H, slip).ravel() - c.cov)) > c.bound
    assert m.covariance_reference(H.ravel(), False).cov == [1e6 if i % 7 == 0 else 0.0 for i in range(36)]
    # a zero row: clearly not invertible by FullPivLU, 1e6 I
    Z = H.copy(); Z[2, :] = 0; Z[:, 2] = 0
    z = m.covariance_reference(Z.ravel(), True)
    assert z.clear and not z.invertible and z.cov[0] == 1e6


def test_qr_reference_rank_rule():
    """An exactly zero column gives the basic solution with that component 0; a nearly dependent one is in the band"""
    H = _designed([1.0, 2.0, 3.0, 4.0, 5.0, 6.0])
    H[4, :] = 0; H[:, 4] = 0
    g = np.arange(1.0, 7.0)
    with m.mpmath.workdps(m.DPS):
        Hm, gm = m._unpack27(o.pack27(H, g))
        x, cond, ok = m.qr_reference(Hm, gm)
    keep = [0, 1, 2, 3, 5]
    assert ok and float(x[4]) == 0.0
    assert np.allclose(m.to_float(x)[:4] + [m.to_float(x)[5]], np.linalg.solve(H[np.ix_(keep, keep)], g[keep]))
    H2 = _designed([1e-17, 2.0, 3.0, 4.0, 5.0, 6.0])
    with m.mpmath.workdps(m.DPS):
        _, _, ok = m.qr_reference(*m._unpack27(o.pack27(H2, g)))
    assert not ok
