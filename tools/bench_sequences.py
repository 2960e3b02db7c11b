"""Frames/s of map-based localisation with chained priors: one dcreg_icp_run_sequences call against the per-frame host
loop a user runs without it (dcreg_set_source + dcreg_icp_run, then the next prior composed on the host from the result).

Workloads (make_parking_sequence: C3-shaped frames, ~6 k points each, against the 0.5 M-point parking map, odometry
increments perturbed by 3 cm / 0.3 deg per axis and step): "1x256", one sequence of 256 frames (seed 47), and "8x64",
eight sequences of 64 frames drawn with seeds 71..78.  Radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3
(icp_pk01.yaml), method Ours.  Both are timed the way tools/bench_scans.py times its batch: host arrays in, results out,
the max of CUDA events on the context's stream and the host wall clock, after a warm-up of both; --runs alternating
pairs, medians reported.  Every frame of the call is checked against the loop's own run of it (status, iterations,
converged identical, pose <= 1e-8 on the SE(3) log); the tool exits non-zero if that fails.  Also reported, not asserted:
the largest translation / rotation error against the true poses of the chained results and of the dead-reckoned priors
(T_init composed with the increments alone).  Prints one JSON line with the card name and power limit; --dump-outputs
DIR writes the chained poses, priors and flags as float64 .npy files."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_scans import card  # noqa: E402


def pose_errors(T_true, T):
    """Largest translation (m) and rotation (deg) error of the poses T against T_true."""
    import dcreg_oracle as o
    dt, dr = 0.0, 0.0
    for A, B in zip(T_true, T):
        E = np.linalg.inv(A) @ B
        dt = max(dt, float(np.linalg.norm(E[:3, 3])))
        dr = max(dr, float(np.degrees(np.linalg.norm(o.so3_log(E[:3, :3])))))
    return dt, dr


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import compose_prior
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_sequences.py: no CUDA device - dcreg_b200 has no CPU fallback")
    prm = default_params(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    workloads = {"1x256": [(256, 47)], "8x64": [(64, 71 + i) for i in range(8)]}
    line = {"metric": "frames_per_s", "workloads": {}, "card": card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream)
        park_map = None
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in spec:
                frames, Tt, Ti0, D, park_map = make_parking_sequence(n, seed=seed)
                seqs.append(frames); T0.append(Ti0); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            ctx.set_target(park_map, 0.5)
            n_frames = len(deltas)

            def call():
                return ctx.icp_run_sequences(prm, seqs, T0, deltas)

            def frame_loop():
                out, k = [], 0
                for s, frames in enumerate(seqs):
                    T = T0[s]
                    for f in frames:
                        ctx.set_source(f)
                        r = ctx.icp_run(prm, T, want_log=False)
                        r.T_prior = T
                        out.append(r)
                        T = compose_prior(r.T, deltas[k])
                        k += 1
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

            call()                                                             # warm-up of both shapes
            frame_loop()
            call_ms, loop_ms = [], []
            for _ in range(max(1, args.runs)):
                res, ms = timed(call)
                call_ms.append(ms)
                loop, ms = timed(frame_loop)
                loop_ms.append(ms)
            same, worst = True, 0.0
            for b, s in zip(res, loop):
                same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
                worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok
            T_dr, k = [], 0                                                    # dead reckoning: increments alone
            for s, frames in enumerate(seqs):
                T = T0[s]
                for _ in frames:
                    T_dr.append(T)
                    T = compose_prior(T, deltas[k])
                    k += 1
            chained = pose_errors(T_true, [r.T for r in res])
            dead = pose_errors(T_true, T_dr)
            cm, lm = float(np.median(call_ms)), float(np.median(loop_ms))
            sizes = [len(f) for frames in seqs for f in frames]
            line["workloads"][name] = {
                "sequences": len(seqs), "frames": n_frames, "frames_per_s": n_frames / (cm * 1e-3), "ms": cm,
                "runs_ms": call_ms, "loop_frames_per_s": n_frames / (lm * 1e-3), "loop_ms": lm, "loop_runs_ms": loop_ms,
                "speedup_vs_loop": lm / cm, "mean_iterations": float(np.mean([r.iterations for r in res])),
                "converged": int(sum(r.converged for r in res)),
                "points_per_frame": {"min": int(min(sizes)), "max": int(max(sizes)), "total": int(sum(sizes))},
                "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst,
                           "tolerance": 1e-8},
                "max_err_vs_truth": {"chained": {"trans_m": chained[0], "rot_deg": chained[1]},
                                     "dead_reckoned_prior": {"trans_m": dead[0], "rot_deg": dead[1]}}}
            dumps[name] = res
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, res in dumps.items():
            for k, v in {"T": [r.T for r in res], "T_prior": [r.T_prior for r in res],
                         "iterations": [r.iterations for r in res], "converged": [r.converged for r in res],
                         "status": [r.status for r in res]}.items():
                np.save(os.path.join(args.dump_outputs, f"sequences_{name}_{k}.npy"), np.asarray(v, dtype=np.float64))
    if not ok_all:
        bad = {n: w["parity"] for n, w in line["workloads"].items() if not w["parity"]["ok"]}
        raise SystemExit(f"bench_sequences.py: parity FAILED {bad}")


if __name__ == "__main__":
    main()
