"""The high-precision reference of the "Ours" step (oracle/dcreg_oracle_mp.py) against the FP64 NumPy oracle
(dcreg_oracle.analyze_degeneracy / solve_degenerate_system) on every record of the G1 and G2 registrations.

Both evaluate the same mathematics, so on records whose decisions are clear of the band they must agree on the mask,
the PCG iteration count and the branch, and the FP64 values must sit within rounding of the exact ones: eigenvalues
within EIG_BAND * scale (which is what justifies the band), P and dx within a bound from the conditioning.
"""
import math

import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_mp as m


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
