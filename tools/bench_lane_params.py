"""Per-lane solver settings (dcreg_set_lane_params): M settings as the lanes of one batched call against M uniform calls.

Workloads:
- "methods": the six SO(3) methods of the CLI x 512 perturbations (trial_poses, seed 45) of the shipped 7 562-point
  cylinder in the G2 setup (radius 1, weight derivative, ROT 1e-5 / TRANS 1e-3, kappa 10): one dcreg_icp_run_batch call
  of 3 072 lanes against six calls of 512.
- "kappa": Fig. 19's 15 values (cond_thresh = kappa_target = k, "Ours") on tools/bench_odometry.py's 256-frame sequence
  (make_parking_sequence seed 47, 20 k points per frame, map_frames 10, radius and cell 0.5): one dcreg_icp_run_odometry
  call of 15 sequences against 15 calls of one.
Both sides are timed as tools/bench_scans.py times its calls: host arrays in, results out, the max of CUDA events on
the context's stream and the host wall clock, after a warm-up of both; --runs alternating pairs, medians reported.

Contract (asserted; the tool exits non-zero if it fails): every lane of the per-lane call has the status, iterations and
converged flag of the same lane of the call whose entries all are that lane's, and the same T_out and T_prior bytes.
Logs, covariances and radii are not requested here; tests/test_gpu_lane_params.py compares those byte for byte.
Prints one JSON line with the card name and power limit; --dump-outputs DIR writes the per-lane calls' poses and
flags as float64 .npy files."""
import os

import numpy as np

import bench_harness as h

KAPPAS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 20, 30, 40, 50, 100]


def same(a, b):
    pa, pb = getattr(a, "T_prior", None), getattr(b, "T_prior", None)
    return ((a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged) and
            a.T.tobytes() == b.T.tobytes() and (pa is None) == (pb is None) and (pa is None or pa.tobytes() == pb.tobytes()))


def main():
    ap = h.parser()
    ap.add_argument("--trials", type=int, default=512)
    ap.add_argument("--frames", type=int, default=256)
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.scenes import g2_initial_pose, load_pcd_xyz, trial_poses
    line = {"metric": "lane_params_speedup", "workloads": {}, "card": h.card()}
    ok = True
    dumps = {}
    with Context(0) as ctx:
        # ---- methods x perturbations on the G2 cylinder
        pts = load_pcd_xyz(os.path.join(h.ROOT, "tests", "golden", "cylinder_7562.pcd"))
        ctx.set_source(pts)
        ctx.set_target(pts, 1.0)
        T = g2_initial_pose() @ trial_poses(args.trials, seed=45)
        n = len(T)
        prm = {m: h.c3_params(m, search_radius=1.0, use_weight_derivative=1) for m in h.METHODS}
        entries = [prm[m] for m in h.METHODS for _ in range(n)]
        T_all = np.concatenate([T] * len(h.METHODS))
        outs, _, med = h.run_arms(ctx, {"one": lambda: ctx.icp_run_batch(entries, T_all),
                                        "uniform": lambda: [ctx.icp_run_batch(prm[m], T) for m in h.METHODS]}, args.runs)
        t_one, t_uni, out = med["one"], med["uniform"], outs["one"]
        bad = 0
        for k, m in enumerate(h.METHODS):
            ref = ctx.icp_run_batch([prm[m]] * len(entries), T_all)
            bad += sum(not same(out[i], ref[i]) for i in range(k * n, (k + 1) * n))
        ok &= bad == 0
        line["workloads"]["methods"] = {
            "lanes": len(entries), "one_call_ms": round(t_one, 2), "uniform_calls_ms": round(t_uni, 2),
            "speedup": round(t_uni / t_one, 3), "trials_per_s_one_call": round(1e3 * len(entries) / t_one),
            "lanes_differing_from_uniform": bad}
        dumps.update(h.result_dumps("lane_params_methods", out, ("T", "iterations", "converged", "status")))
        # ---- the kappa sweep on one odometry recording
        (frames,), _, deltas, _ = h.parking_sequences([(args.frames, 47)], n_scan=20_000, max_range=20.0)
        T0 = np.eye(4)[None]
        kp = [h.c3_params(cond_thresh=float(k), kappa_target=float(k)) for k in KAPPAS]
        S = len(kp)
        seqs = [list(frames)] * S
        D_all = np.concatenate([deltas] * S)
        T0_all = np.repeat(T0, S, axis=0)

        def odo(p, sq, D, T_init):
            return ctx.icp_run_odometry(p, sq, T_init, D, map_frames=10, cell_size=0.5)
        outs, _, med = h.run_arms(ctx, {"one": lambda: odo(kp, seqs, D_all, T0_all),
                                        "uniform": lambda: [odo(p, [list(frames)], deltas, T0) for p in kp]}, args.runs)
        t_one, t_uni, out = med["one"], med["uniform"], outs["one"]
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
        dumps.update(h.result_dumps("lane_params_kappa", out))
    line["contract_ok"] = bool(ok)
    h.finish(args, line, dumps, ok, 1)


if __name__ == "__main__":
    main()
