"""Per-lane solver settings (dcreg_set_lane_params): M settings as the lanes of one batched call against M uniform calls.

Workloads:
- "methods": the six SO(3) methods of the CLI x 512 perturbations (trial_poses, seed 45) of the shipped 7 562-point
  cylinder in the G2 setup (radius 1, weight derivative, ROT 1e-5 / TRANS 1e-3, kappa 10): one dcreg_icp_run_batch call
  of 3 072 lanes against six calls of 512.
- "kappa": Fig. 19's 15 values (cond_thresh = kappa_target = k, "Ours") on tools/bench_odometry.py's 256-frame sequence
  (make_parking_sequence seed 47, 20 k points per frame, map_frames 10, radius and cell 0.5): one dcreg_icp_run_odometry
  call of 15 sequences against 15 calls of one.
Both sides are timed on the host clock around calls that return their results (each ends in a device synchronise),
after a warm-up of both; --runs alternating pairs, medians reported.

Contract (asserted; the tool exits non-zero if it fails): every lane of the per-lane call has the status, iterations and
converged flag of the same lane of the call whose entries all are that lane's, and the same T_out and T_prior bytes.
Logs, covariances and radii are not requested here; tests/test_gpu_lane_params.py compares those byte for byte.
Prints one JSON line with the card name and power limit."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_scans import card  # noqa: E402

METHODS = {                       # the six methods the CLI's SO(3) path recognises
    "Ours": ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG"),
    "NONE": ("NONE_DETE", "NONE_HAND"),
    "ME-SR": ("FULL_EVD_MIN_EIGENVALUE", "SOLUTION_REMAPPING"),
    "FCN-SR": ("FULL_SVD_CONDITION", "SOLUTION_REMAPPING"),
    "ME-TSVD": ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD"),
    "ME-TReg": ("FULL_EVD_MIN_EIGENVALUE", "STANDARD_REGULARIZATION"),
}
KAPPAS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 20, 30, 40, 50, 100]


def same(a, b):
    pa, pb = getattr(a, "T_prior", None), getattr(b, "T_prior", None)
    return ((a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged) and
            a.T.tobytes() == b.T.tobytes() and (pa is None) == (pb is None) and (pa is None or pa.tobytes() == pb.tobytes()))


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return out, (time.perf_counter() - t0) * 1e3


def compare(one_call, uniform_calls, runs):
    """Warm-up, then `runs` alternating pairs; (medians ms of one call and of the uniform calls in all, one call's out)"""
    one_call()
    uniform_calls()
    t_one, t_uni = [], []
    for _ in range(runs):
        out, ms = timed(one_call)
        t_one.append(ms)
        t_uni.append(timed(uniform_calls)[1])
    return float(np.median(t_one)), float(np.median(t_uni)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--trials", type=int, default=512)
    ap.add_argument("--frames", type=int, default=256)
    args = ap.parse_args()
    import torch
    from dcreg_b200 import Context, default_params
    from dcreg_b200.scenes import g2_initial_pose, load_pcd_xyz, make_parking_sequence, trial_poses
    if not torch.cuda.is_available():
        raise SystemExit("bench_lane_params.py: no CUDA device - dcreg_b200 has no CPU fallback")
    line = {"metric": "lane_params_speedup", "workloads": {}, "card": card()}
    ok = True
    with Context(0) as ctx:
        # ---- methods x perturbations on the G2 cylinder
        pts = load_pcd_xyz(os.path.join(ROOT, "tests", "golden", "cylinder_7562.pcd"))
        ctx.set_source(pts)
        ctx.set_target(pts, 1.0)
        T = g2_initial_pose() @ trial_poses(args.trials, seed=45)
        n = len(T)
        prm = {m: default_params(search_radius=1.0, max_iterations=30, use_weight_derivative=1, conv_thresh_rot=1e-5,
                                 conv_thresh_trans=1e-3, kappa_target=10.0, detection=d, handling=h)
               for m, (d, h) in METHODS.items()}
        entries = [prm[m] for m in METHODS for _ in range(n)]
        T_all = np.concatenate([T] * len(METHODS))
        t_one, t_uni, out = compare(lambda: ctx.icp_run_batch(entries, T_all),
                                    lambda: [ctx.icp_run_batch(prm[m], T) for m in METHODS], args.runs)
        bad = 0
        for k, m in enumerate(METHODS):
            ref = ctx.icp_run_batch([prm[m]] * len(entries), T_all)
            bad += sum(not same(out[i], ref[i]) for i in range(k * n, (k + 1) * n))
        ok &= bad == 0
        line["workloads"]["methods"] = {
            "lanes": len(entries), "one_call_ms": round(t_one, 2), "uniform_calls_ms": round(t_uni, 2),
            "speedup": round(t_uni / t_one, 3), "trials_per_s_one_call": round(1e3 * len(entries) / t_one),
            "lanes_differing_from_uniform": bad}
        # ---- the kappa sweep on one odometry recording
        frames, _, _, deltas, _ = make_parking_sequence(args.frames, seed=47, n_scan=20_000, max_range=20.0)
        T0 = np.eye(4)[None]
        kp = [default_params(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                             cond_thresh=float(k), kappa_target=float(k), detection="SCHUR_CONDITION_NUMBER",
                             handling="PRECONDITIONED_CG") for k in KAPPAS]
        S = len(kp)
        seqs = [list(frames)] * S
        D_all = np.concatenate([deltas] * S)
        T0_all = np.repeat(T0, S, axis=0)

        def odo(p, sq, D, T_init):
            return ctx.icp_run_odometry(p, sq, T_init, D, map_frames=10, cell_size=0.5)
        t_one, t_uni, out = compare(lambda: odo(kp, seqs, D_all, T0_all),
                                    lambda: [odo(p, [list(frames)], deltas, T0) for p in kp], args.runs)
        bad = 0
        for s in range(S):
            ref = odo([kp[s]] * S, seqs, D_all, T0_all)
            bad += sum(not same(out[i], ref[i]) for i in range(s * len(frames), (s + 1) * len(frames)))
        ok &= bad == 0
        nf = S * len(frames)
        line["workloads"]["kappa"] = {
            "lanes": S, "frames": nf, "one_call_ms": round(t_one, 2), "uniform_calls_ms": round(t_uni, 2),
            "speedup": round(t_uni / t_one, 3), "frames_per_s_one_call": round(1e3 * nf / t_one),
            "frames_per_s_uniform_calls": round(1e3 * nf / t_uni), "frames_differing_from_uniform": bad}
    line["contract_ok"] = bool(ok)
    print(json.dumps(line))
    if not ok:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
