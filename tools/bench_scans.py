"""Frames/s of registering many C3-shaped LiDAR frames against one map: one dcreg_icp_run_scans call against the
per-frame dcreg_set_source + dcreg_icp_run loop a user runs without it.

Workload: --frames (64) frames of make_parking_frames (seed 47, ~6 k points each) against the 0.5 M-point parking map,
radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3 (icp_pk01.yaml), method Ours.  Both are timed the way bench.py times its
C5 batch: host arrays in, results out, the max of CUDA events on the context's stream and the host wall clock, after a
warm-up of both; --runs alternating pairs, medians reported.  Every frame of the batch is checked against its own
sequential run (status, iterations, converged identical, pose <= 1e-8 on the SE(3) log); the tool exits non-zero if that
fails.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes the batched poses and flags as
float64 .npy files."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context, default_params
    from dcreg_b200.scenes import make_parking_frames
    if not torch.cuda.is_available():
        raise SystemExit("bench_scans.py: no CUDA device - dcreg_b200 has no CPU fallback")
    frames, _, T_init, park_map = make_parking_frames(args.frames, seed=47)
    prm = default_params(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    with Context(0) as ctx:
        ctx.set_target(park_map, 0.5)
        stream = torch.cuda.ExternalStream(ctx.stream)

        def frame_loop():
            out = []
            for f, T in zip(frames, T_init):
                ctx.set_source(f)
                out.append(ctx.icp_run(prm, T, want_log=False))
            return out

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w = time.perf_counter()
            e0.record(stream)
            out = fn()
            e1.record(stream)
            e1.synchronize()
            w = time.perf_counter() - w
            return out, max(e0.elapsed_time(e1), w * 1e3)

        ctx.icp_run_scans(prm, frames, T_init)                                 # warm-up of both shapes
        frame_loop()
        batch_ms, seq_ms = [], []
        for _ in range(max(1, args.runs)):
            batch, ms = timed(lambda: ctx.icp_run_scans(prm, frames, T_init))
            batch_ms.append(ms)
            seq, ms = timed(frame_loop)
            seq_ms.append(ms)
    same, worst = True, 0.0
    for b, s in zip(batch, seq):
        same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
        worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
    ok = same and worst <= 1e-8
    n = args.frames
    bm, sm = float(np.median(batch_ms)), float(np.median(seq_ms))
    sizes = [len(f) for f in frames]
    line = {"metric": "frames_per_s", "frames": n, "frames_per_s": n / (bm * 1e-3), "ms": bm,
            "runs_ms": batch_ms, "sequential_frames_per_s": n / (sm * 1e-3), "sequential_ms": sm, "sequential_runs_ms": seq_ms,
            "speedup_vs_sequential": sm / bm, "mean_iterations": float(np.mean([b.iterations for b in batch])),
            "converged": int(sum(b.converged for b in batch)),
            "points_per_frame": {"min": int(min(sizes)), "max": int(max(sizes)), "total": int(sum(sizes))},
            "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8},
            "card": card()}
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in {"scans_T": [b.T for b in batch], "scans_iterations": [b.iterations for b in batch],
                     "scans_converged": [b.converged for b in batch], "scans_status": [b.status for b in batch]}.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), np.asarray(v, dtype=np.float64))
    if not ok:
        raise SystemExit(f"bench_scans.py: parity FAILED (status/iterations/converged identical: {same}, max pose err {worst:.3e})")


if __name__ == "__main__":
    main()
