"""Pin the C/OpenMP oracle (the CPU baseline) against the reference's shipped dumps and the NumPy twin."""
import numpy as np
import pytest

import dcreg_oracle as o
import dcreg_oracle_c as oc
from harness import init_T, params_from


def c_params(prm: o.Params, **kw):
    return oc.make_params(search_radius=prm.search_radius, max_iterations=prm.max_iterations, detection=prm.detection,
                          handling=prm.handling, use_weight_derivative=prm.use_weight_derivative, conv_rot=prm.conv_rot,
                          conv_trans=prm.conv_trans, cond_thresh=prm.cond_thresh, eig_thresh=prm.eig_thresh,
                          kappa_target=prm.kappa_target, pcg_tol=prm.pcg_tol, pcg_max_iter=prm.pcg_max_iter,
                          std_reg_gamma=prm.std_reg_gamma, **kw)


@pytest.fixture(scope="module")
def scene(cylinder):
    s = oc.Scene(cylinder, cylinder)
    yield s
    s.close()


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("setup,method", [("G1", "ME-SR"), ("G1", "ME-TSVD"), ("G1", "ME-TReg"), ("G1", "FCN-SR"), ("G2", "Ours")])
def test_c_oracle_reproduces_shipped_trajectories(golden, scene, setup, method, mode):
    g = golden[setup]
    prm = params_from(g["setup"], method)
    st, conv, n_it, T, logs = scene.icp_run(c_params(prm, thread_mode=mode), init_T(g["setup"]))
    rows = g["iterations"][method]
    tol = 1e-8 if setup == "G1" else 5e-7
    assert st == 0 and conv and n_it == len(rows)
    for r, L in zip(rows, logs):
        assert np.abs(np.array(r["dx"]) - np.array(L.dx)).max() < tol
        assert np.abs(np.array(r["T"]) - np.array(L.T)).max() < tol
        assert list(L.mask) == r["mask"]
        assert abs(r["rmse"] - L.rmse) < 5e-8 and abs(r["fitness"] - L.fitness) < 1e-8


def test_c_oracle_matches_numpy_twin(golden, cylinder, scene):
    g = golden["G2"]
    prm = params_from(g["setup"], "Ours")
    conv, T, logs, status = o.icp_so3(cylinder, cylinder, init_T(g["setup"]), prm)
    st, convc, n_it, Tc, clogs = scene.icp_run(c_params(prm), init_T(g["setup"]))
    assert st == 0 and convc == conv and n_it == len(logs)
    for L, C in zip(logs, clogs):
        assert C.n_eff == L.n_eff and C.n_pt == L.n_pt
        assert np.abs(np.array(C.H).reshape(6, 6) - L.H).max() <= 1e-10 * np.abs(L.H).max()
        assert np.abs(np.array(C.dx) - L.dx).max() < 1e-9
        assert np.allclose(C.lam_schur_rot, L.analysis.lambda_schur_rot, rtol=1e-9)
        assert np.allclose(C.lam_schur_trans, L.analysis.lambda_schur_trans, rtol=1e-9)
        assert np.allclose(np.array(C.P).reshape(6, 6), L.analysis.P, rtol=1e-8, atol=1e-14)
        assert C.pcg_iterations == L.analysis.pcg_iterations
    assert o.se3_log_distance(T, Tc) < 1e-9


def test_c_oracle_synthetic_scene_and_abort(cylinder):
    from dcreg_b200.scenes import make_cylinder, g2_initial_pose
    pts = make_cylinder(20_000, seed=42)
    prm = o.Params(max_iterations=4, conv_rot=0.0, conv_trans=0.0, kappa_target=10.0, use_weight_derivative=True)
    conv, T, logs, status = o.icp_so3(pts, pts, g2_initial_pose(), prm)
    sc = oc.Scene(pts, pts)
    st, convc, n_it, Tc, clogs = sc.icp_run(c_params(prm, fixed_iterations=True), g2_initial_pose())
    assert st == 0 and n_it == 4 and [c.n_eff for c in clogs] == [l.n_eff for l in logs]
    assert o.se3_log_distance(T, Tc) < 1e-9
    far = o.pose6d_to_matrix(500.0, 0, 0, 0, 0, 0)
    st, convc, n_it, Tc, clogs = sc.icp_run(c_params(prm), far)
    assert st == 1 and n_it == 1 and np.allclose(Tc, far)
    sc.close()
