"""The host CLI (`dcreg_b200/icp_test_runner`, the reference's experiment harness on the C ABI).

CPU tests: YAML subset parser on a reference-style config (DCReg/config/icp.yaml layout: comments, quoted keys, flow
sequences), PCD reader/writer round trip, pose-error metric against the oracle, and the loud failure without a device.
GPU test: the binary reproduces the reference's shipped per-iteration CSV rows (tests/golden/golden.json) on the shipped
cylinder cloud for every method of the SO(3) path.
"""
import math
import os
import subprocess

import numpy as np
import pytest

import dcreg_oracle as o
from dcreg_b200 import build as b
from harness import GOLD, METHODS, dump, read_csv, write_config


@pytest.fixture(scope="module")
def runner():
    return b.build_runner()


def test_yaml_config_parses_like_the_reference(runner, golden, tmp_path):
    cfg = tmp_path / "icp.yaml"
    write_config(cfg, tmp_path / "out", golden["G2"]["setup"], ["Ours", "ME-SR", "FCN-SR"],
                 extra_methods='  "XICP": [ "XICP_INEQUALITY", "XICP_CONSTRAINT"]')
    kv, methods = dump(runner, str(cfg))
    assert kv["num_runs"] == "1" and kv["save_pcd"] == "1" and kv["visualize"] == "0"
    assert kv["source_pcd"] == "cylinder_7562.pcd" and kv["folder_path"] == GOLD + "/"
    assert float(kv["search_radius"]) == 1.0 and int(kv["max_iterations"]) == 30 and int(kv["normal_nn"]) == 5
    assert float(kv["CONVERGENCE_THRESH_ROT"]) == 1e-5 and float(kv["CONVERGENCE_THRESH_TRANS"]) == 1e-3
    assert float(kv["STD_REG_GAMMA"]) == 100.0 and float(kv["KAPPA_TARGET"]) == 10.0 and int(kv["PCG_MAX_ITER"]) == 10
    assert float(kv["PCG_TOLERANCE"]) == 1e-6 and kv["use_weight_derivative"] == "1"
    T0 = np.array([float(v) for v in kv["initial_matrix"].split(",")]).reshape(4, 4)
    d = math.pi / 180
    assert np.abs(T0 - o.pose6d_to_matrix(0.2, 0.8, 0.5, 0.1 * d, 0.1 * d, 2.0 * d)).max() < 1e-15
    # std::map order (alphabetical), enum mapping, unknown enum strings fall back to the first enumerator
    assert [m[0] for m in methods] == ["FCN-SR", "ME-SR", "Ours", "XICP"]
    assert methods[0][3:] == ["4", "4"] and methods[1][3:] == ["2", "4"] and methods[2][3:] == ["1", "3"]
    assert methods[3][3:] == ["0", "0"]


def test_yaml_monte_carlo_block(runner, golden, tmp_path):
    """The optional perturbation-study block (an extension; absent = off, like the reference)."""
    cfg = tmp_path / "icp.yaml"
    write_config(cfg, tmp_path / "out", golden["G2"]["setup"], ["Ours"])
    kv, _ = dump(runner, str(cfg))
    assert kv["mc_trials"] == "0" and kv["mc_seed"] == "45"
    write_config(cfg, tmp_path / "out", golden["G2"]["setup"], ["Ours"],
                 extra="monte_carlo:\n  trials: 64\n  seed: 7\n  max_trans_m: 0.5\n  max_rot_deg: 2.0\n")
    kv, _ = dump(runner, str(cfg))
    assert kv["mc_trials"] == "64" and kv["mc_seed"] == "7" and float(kv["mc_max_trans"]) == 0.5 and float(kv["mc_max_rot_deg"]) == 2.0
    write_config(cfg, tmp_path / "out", golden["G2"]["setup"], ["Ours"], extra="monte_carlo:\n  trials: 70000\n")
    res = subprocess.run([runner, "--dump-config", str(cfg)], capture_output=True, text=True)
    assert res.returncode != 0 and "monte_carlo.trials" in res.stderr


def test_yaml_missing_required_key_fails(runner, tmp_path):
    cfg = tmp_path / "bad.yaml"
    cfg.write_text("test:\n  num_runs: 1\n")
    res = subprocess.run([runner, "--dump-config", str(cfg)], capture_output=True, text=True)
    assert res.returncode != 0 and "Error loading YAML config" in res.stderr


def test_pcd_round_trip(runner, cylinder, tmp_path):
    out = tmp_path / "copy.pcd"
    res = subprocess.run([runner, "--pcd-roundtrip", os.path.join(GOLD, "cylinder_7562.pcd"), str(out)],
                         capture_output=True, text=True, check=True)
    assert "points=7562" in res.stdout
    assert np.array_equal(o.read_pcd_xyz(str(out)), cylinder)
    # ascii input
    asc = tmp_path / "a.pcd"
    pts = cylinder[:50]
    with open(asc, "w") as f:
        f.write("# .PCD v0.7\nVERSION 0.7\nFIELDS x y z\nSIZE 4 4 4\nTYPE F F F\nCOUNT 1 1 1\nWIDTH 50\nHEIGHT 1\n"
                "VIEWPOINT 0 0 0 1 0 0 0\nPOINTS 50\nDATA ascii\n")
        for p in pts:
            f.write(f"{p[0]!r} {p[1]!r} {p[2]!r}\n".replace("np.float32(", "").replace(")", ""))
    subprocess.run([runner, "--pcd-roundtrip", str(asc), str(out)], capture_output=True, text=True, check=True)
    assert np.array_equal(o.read_pcd_xyz(str(out)), pts)


def test_pose_error_metric_matches_oracle(runner):
    rng = np.random.default_rng(3)
    for _ in range(6):
        Ts = []
        for _k in range(2):
            a = rng.uniform(-3, 3, 6)
            Ts.append(o.pose6d_to_matrix(a[0], a[1], a[2], a[3], a[4] * 0.4, a[5]))
        args = [repr(float(v)) for T in Ts for v in T.reshape(-1)]
        out = subprocess.run([runner, "--pose-error"] + args, capture_output=True, text=True, check=True).stdout.split()
        te, re_ = o.pose_error(Ts[0], Ts[1])
        assert abs(float(out[0]) - te) < 1e-12 and abs(float(out[1]) - re_) < 1e-9


def test_runner_fails_loudly_without_a_device(runner, golden, tmp_path):
    import torch
    if torch.cuda.is_available():
        pytest.skip("device present")
    cfg = tmp_path / "icp.yaml"
    write_config(cfg, tmp_path / "out", golden["G2"]["setup"], ["Ours"])
    res = subprocess.run([runner, str(cfg)], capture_output=True, text=True)
    assert res.returncode != 0
    assert "no CUDA device" in res.stderr and "Test run failed!" in res.stderr


@pytest.mark.gpu
@pytest.mark.parametrize("setup", ["G1", "G2"])
def test_runner_reproduces_shipped_iteration_csv(runner, golden, tmp_path, setup):
    g = golden[setup]
    methods = sorted(g["iterations"].keys())
    cfg = tmp_path / "icp.yaml"
    out_dir = tmp_path / "out"
    write_config(cfg, out_dir, g["setup"], methods)
    res = subprocess.run([runner, str(cfg)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "=== All tests completed successfully! ===" in res.stdout
    for fn in ("statistics_summary.txt", "complete_log.txt", "transform_details.csv", "condition_numbers_detailed.csv",
               "all_results.csv", "degeneracy_analysis_first_iter.txt", "degeneracy_analysis_last_iter.txt",
               "iteration_history.csv", "iteration_details_with_dx.csv", "initial_clouds.pcd", "target_clouds.pcd"):
        assert (out_dir / fn).exists(), fn
    rows = read_csv(out_dir / "iteration_details_with_dx.csv")
    assert [r["Method"] for r in rows if r["Iteration"] == "0"] == methods          # alphabetical, like std::map
    for m in methods:
        mine = [r for r in rows if r["Method"] == m]
        ref = g["iterations"][m]
        assert len(mine) == len(ref), m
        for r, G in zip(ref, mine):
            T = np.array([float(G[f"T_{i}{j}"]) for i in range(4) for j in range(4)])
            assert np.abs(T - np.array(r["T"])).max() < 5e-7
            dx = np.array([float(G[k]) for k in ("dx_wx", "dx_wy", "dx_wz", "dx_x", "dx_y", "dx_z")])
            assert np.abs(dx - np.array(r["dx"])).max() < 5e-7
            assert abs(float(G["RMSE"]) - r["rmse"]) < 5e-7 and abs(float(G["Fitness"]) - r["fitness"]) < 5e-7
            assert [int(G[f"Degenerate_{i}"]) for i in range(6)] == r["mask"]
            assert int(G["Is_Degenerate"]) == r["is_degenerate"]
            for mine_k, ref_k in (("Cond_Schur_Rot", "cond_schur_rot"), ("Cond_Schur_Trans", "cond_schur_trans"),
                                  ("Cond_Sub_Rot", "cond_sub_rot"), ("Cond_Sub_Trans", "cond_sub_trans"),
                                  ("Cond_Full_SVD", "cond_full_svd")):
                if math.isnan(r[ref_k]):      # the shipped G1 dump left the Schur / sub-block numbers unset (NaN)
                    continue
                assert abs(float(G[mine_k]) - r[ref_k]) <= 2e-4 * abs(r[ref_k]), (m, mine_k)
            # the swapped error columns (icp_test_runner.cpp:1457-1458): "Trans_Error_m" holds degrees
            # (angle from the skew part: T is printed with 8 decimals, acos(trace) would amplify that rounding)
            R = T.reshape(4, 4)[:3, :3]
            sk = 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
            re_ = math.degrees(math.atan2(np.linalg.norm(sk), 0.5 * (np.trace(R) - 1.0)))
            te = float(np.linalg.norm(T.reshape(4, 4)[:3, 3]))
            assert abs(float(G["Trans_Error_m"]) - re_) < 2e-6 and abs(float(G["Rot_Error_deg"]) - te) < 1e-6
    stats = (out_dir / "statistics_summary.txt").read_text()
    assert "ICP Test Statistics Summary" in stats and "Cloud size: 7562 7562" in stats
    if setup == "G2":
        # shipped statistics_summary.txt of the reference for "Ours": 0.0271 m / 0.0507 deg, 10 iterations
        line = [ln for ln in stats.splitlines() if ln.strip().startswith("Ours")][0].split()
        assert line[1] == "100.0" and line[2] == "0.0271" and line[3] == "0.0507" and line[5] == "10.0"
        final = read_csv(out_dir / "all_results.csv")
        ours = [r for r in final if r["Method"] == "Ours"][0]
        assert ours["Converged"] == "1" and ours["Iterations"] == "10"
        assert abs(float(ours["P2P_RMSE"]) - 0.036217) < 2e-6 and abs(float(ours["Chamfer_Distance"]) - 0.032915) < 2e-6
    # aligned cloud dump = fl32(T_final * source)
    first = methods[0]
    aligned = o.read_pcd_xyz(str(out_dir / f"{first}_aligned_clouds_sig.pcd"))
    Tf = np.array(g["iterations"][first][-1]["T"]).reshape(4, 4)
    src = o.read_pcd_xyz(os.path.join(GOLD, "cylinder_7562.pcd")).astype(np.float64)
    assert np.abs(aligned - (src @ Tf[:3, :3].T + Tf[:3, 3])).max() < 1e-4


@pytest.mark.gpu
def test_runner_monte_carlo_matches_the_batched_api(runner, golden, tmp_path):
    """monte_carlo: block of the CLI = dcreg_icp_run_batch on the poses it drew (written to the CSV) - same poses through
    the Python binding must give the same iterations / flags and poses to 1e-8 (trial 0 sorts the source, see the header),
    and a handful of trials are checked against the oracle loop."""
    from dcreg_b200 import api, default_params
    g = golden["G2"]
    cfg = tmp_path / "icp.yaml"
    out_dir = tmp_path / "out"
    write_config(cfg, out_dir, g["setup"], ["Ours", "ME-TSVD"],
                 extra="monte_carlo:\n  trials: 48\n  seed: 11\n  max_trans_m: 0.6\n  max_rot_deg: 2.0\n")
    res = subprocess.run([runner, str(cfg)], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    summary = (out_dir / "monte_carlo_summary.txt").read_text()
    assert "48 trials, seed 11" in summary and "Ours" in summary and "ME-TSVD" in summary
    pts = o.read_pcd_xyz(os.path.join(GOLD, "cylinder_7562.pcd"))
    d = math.pi / 180
    with api.Context() as ctx:
        ctx.set_source(pts)
        ctx.set_target(pts, g["setup"]["search_radius"])
        for m in ("Ours", "ME-TSVD"):
            rows = read_csv(out_dir / f"monte_carlo_{m}.csv")
            assert len(rows) == 48 and [int(r["Trial"]) for r in rows] == list(range(48))
            init = np.array([o.pose6d_to_matrix(float(r["Init_x"]), float(r["Init_y"]), float(r["Init_z"]), float(r["Init_roll_deg"]) * d,
                                                float(r["Init_pitch_deg"]) * d, float(r["Init_yaw_deg"]) * d) for r in rows])
            assert np.abs(init[:, :3, 3]).max() <= 0.6 and np.abs(init[:, :3, 3]).max() > 0.3     # the draws fill the box
            s = g["setup"]
            p = default_params(search_radius=s["search_radius"], max_iterations=s["max_iterations"], detection=METHODS[m][0],
                               handling=METHODS[m][1], use_weight_derivative=int(s["use_weight_derivative"]),
                               conv_thresh_rot=s["conv_rot"], conv_thresh_trans=s["conv_trans"], cond_thresh=s["cond_thresh"],
                               eig_thresh=s["eig_thresh"], kappa_target=s["kappa_target"], std_reg_gamma=s["std_reg_gamma"])
            res = ctx.icp_run_batch(p, init)
            for i, r in enumerate(rows):
                Tc = np.array([float(r[f"T{k // 4}{k % 4}"]) for k in range(12)]).reshape(3, 4)
                assert int(r["Iterations"]) == res[i].iterations and int(r["Converged"]) == int(res[i].converged), (m, i)
                assert int(r["Status"]) == res[i].status, (m, i)
                assert np.abs(Tc - res[i].T[:3]).max() < 1e-8, (m, i)
                te = float(np.linalg.norm(Tc[:, 3]))
                assert abs(float(r["Trans_Error_m"]) - te) < 1e-9                              # gt = identity in this config
