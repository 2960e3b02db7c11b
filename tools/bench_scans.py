"""Frames/s of registering many C3-shaped LiDAR frames against one map: one dcreg_icp_run_scans call against the
per-frame dcreg_set_source + dcreg_icp_run loop a user runs without it.

Workload: --frames (64) frames of make_parking_frames (seed 47, ~6 k points each) against the 0.5 M-point parking map,
radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3 (icp_pk01.yaml), method Ours.  Both are timed the way bench.py times its
C5 batch: host arrays in, results out, the max of CUDA events on the context's stream and the host wall clock, after a
warm-up of both; --runs alternating pairs, medians reported.  Every frame of the batch is checked against its own
sequential run (status, iterations, converged identical, pose <= 1e-8 on the SE(3) log); the tool exits non-zero if that
fails.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes the batched poses and flags as
float64 .npy files."""
import numpy as np

import bench_harness as h


def main():
    ap = h.parser()
    ap.add_argument("--frames", type=int, default=64)
    args = ap.parse_args()
    h.require_gpu()
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context
    from dcreg_b200.scenes import make_parking_frames
    frames, _, T_init, park_map = make_parking_frames(args.frames, seed=47)
    prm = h.c3_params()
    with Context(0) as ctx:
        ctx.set_target(park_map, 0.5)

        def frame_loop():
            out = []
            for f, T in zip(frames, T_init):
                ctx.set_source(f)
                out.append(ctx.icp_run(prm, T, want_log=False))
            return out

        outs, ms, med = h.run_arms(ctx, {"batch": lambda: ctx.icp_run_scans(prm, frames, T_init), "seq": frame_loop},
                                   args.runs)
    batch, seq = outs["batch"], outs["seq"]
    same, worst = True, 0.0
    for b, s in zip(batch, seq):
        same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
        worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
    ok = same and worst <= 1e-8
    n = args.frames
    line = {"metric": "frames_per_s", "frames": n, **h.rate(n, med["batch"], ms["batch"]),
            **h.rate(n, med["seq"], ms["seq"], "sequential_"), "speedup_vs_sequential": med["seq"] / med["batch"],
            "mean_iterations": float(np.mean([b.iterations for b in batch])),
            "converged": int(sum(b.converged for b in batch)), "points_per_frame": h.spread([len(f) for f in frames]),
            "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8},
            "card": h.card()}
    h.finish(args, line, h.result_dumps("scans", batch, ("T", "iterations", "converged", "status")), ok,
             f"bench_scans.py: parity FAILED (status/iterations/converged identical: {same}, max pose err {worst:.3e})")


if __name__ == "__main__":
    main()
