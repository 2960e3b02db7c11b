"""Frames/s of scan-to-map odometry: one dcreg_icp_run_odometry call against the per-frame host loop a user runs without
it (build the local map from the loop's own previous results with map_points, then dcreg_set_target + dcreg_set_source
+ dcreg_icp_run from compose_prior of the previous result).

Workloads (make_parking_sequence with n_scan = 20 000 and max_range = 20 m: frames of about 20 k points, an estimated
16 points / m^2 of ground; odometry increments perturbed by 3 cm / 0.3 deg per axis and step): "1x256", one sequence of
256 frames (seed 47), and "8x64", eight sequences of 64 frames (seeds 71..78).  Each sequence is anchored at its first
true pose.  map_frames 10, radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3 (icp_pk01.yaml), method Ours,
motion "increments".  Timing as tools/bench_sequences.py: host arrays in, results out, the max of CUDA events on the
context's stream and the host wall clock, after a warm-up of both; --runs alternating pairs, medians reported.

Parity (asserted; the tool exits non-zero if it fails): every registered frame of the call against its single run
reconstructed from the call's own T_out / T_prior (status, iterations, converged identical, pose <= 1e-8 on the SE(3)
log).  Reported, not asserted: the largest pose difference between the call and the independent host-loop chain (its
maps come from its own rounding), the drift of T_out against the true poses, and a call with max_iterations = 1 (set-up,
map assembly and grid build of every step with one loop body each).  Prints one JSON line with the card name and power
limit; --dump-outputs DIR writes the poses, priors and flags as float64 .npy files."""
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
from bench_sequences import pose_errors  # noqa: E402

MAP_FRAMES = 10
CELL = 0.5


def local_map(frames, T, k):
    from dcreg_b200.api import map_points
    return np.concatenate([map_points(T[j], frames[j]) for j in range(max(0, k - MAP_FRAMES), k)])


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
        raise SystemExit("bench_odometry.py: no CUDA device - dcreg_b200 has no CPU fallback")
    kw = dict(search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0,
              detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    prm = default_params(max_iterations=30, **kw)
    prm1 = default_params(max_iterations=1, **kw)
    workloads = {"1x256": [(256, 47)], "8x64": [(64, 71 + i) for i in range(8)]}
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "workloads": {}, "card": card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream)
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in spec:
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_scan=20_000, max_range=20.0)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            n_frames = len(deltas)

            def call(p=prm):
                return ctx.icp_run_odometry(p, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL)

            def frame_loop():
                out, k = [], 0
                for s, frames in enumerate(seqs):
                    Ts = [T0[s]]
                    out.append(None)                                           # the anchor is not registered
                    k += 1
                    for j in range(1, len(frames)):
                        T = compose_prior(Ts[j - 1], deltas[k - 1])
                        ctx.set_target(local_map(frames, Ts, j), CELL)
                        ctx.set_source(frames[j])
                        r = ctx.icp_run(prm, T, want_log=False)
                        r.T_prior = T
                        out.append(r)
                        Ts.append(r.T)
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
            call(prm1)
            frame_loop()
            call_ms, loop_ms, one_ms = [], [], []
            for _ in range(max(1, args.runs)):
                res, ms = timed(call)
                call_ms.append(ms)
                loop, ms = timed(frame_loop)
                loop_ms.append(ms)
                _, ms = timed(lambda: call(prm1))
                one_ms.append(ms)
            # parity: every registered frame against its run on the map rebuilt from the call's own results
            same, worst, chain_diff, k = True, 0.0, 0.0, 0
            for s, frames in enumerate(seqs):
                rs = res[k:k + len(frames)]
                Ts = [r.T for r in rs]
                for j in range(1, len(frames)):
                    ctx.set_target(local_map(frames, Ts, j), CELL)
                    ctx.set_source(frames[j])
                    single = ctx.icp_run(prm, rs[j].T_prior, want_log=False)
                    b = rs[j]
                    same = same and (b.status, b.iterations, b.converged) == (single.status, single.iterations, single.converged)
                    worst = max(worst, float(o.se3_log_distance(single.T, b.T)))
                    chain_diff = max(chain_diff, float(o.se3_log_distance(loop[k + j].T, b.T)))
                k += len(frames)
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok
            drift = pose_errors(T_true, [r.T for r in res])
            reg = [r for r in res if r.iterations > 0]
            map_pts = []                                                       # map points of every step, over the sequences
            for i in range(1, max(len(f) for f in seqs)):
                map_pts.append(sum(sum(len(f[j]) for j in range(max(0, i - MAP_FRAMES), i)) for f in seqs if len(f) > i))
            cm, lm, om = float(np.median(call_ms)), float(np.median(loop_ms)), float(np.median(one_ms))
            sizes = [len(f) for frames in seqs for f in frames]
            line["workloads"][name] = {
                "sequences": len(seqs), "frames": n_frames, "registered": len(reg),
                "frames_per_s": n_frames / (cm * 1e-3), "ms": cm, "runs_ms": call_ms,
                "loop_frames_per_s": n_frames / (lm * 1e-3), "loop_ms": lm, "loop_runs_ms": loop_ms,
                "speedup_vs_loop": lm / cm, "one_iteration_call_ms": om, "one_iteration_runs_ms": one_ms,
                "mean_iterations": float(np.mean([r.iterations for r in reg])), "converged": int(sum(r.converged for r in reg)),
                "points_per_frame": {"min": int(min(sizes)), "max": int(max(sizes)), "total": int(sum(sizes))},
                "map_points_per_step": {"mean": float(np.mean(map_pts)), "max": int(max(map_pts))},
                "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst,
                           "tolerance": 1e-8},
                "host_loop_chain_max_pose_diff": chain_diff,
                "max_err_vs_truth": {"trans_m": drift[0], "rot_deg": drift[1]}}
            dumps[name] = res
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, res in dumps.items():
            for k, v in {"T": [r.T for r in res], "T_prior": [r.T_prior for r in res],
                         "iterations": [r.iterations for r in res], "converged": [r.converged for r in res],
                         "status": [r.status for r in res]}.items():
                np.save(os.path.join(args.dump_outputs, f"odometry_{name}_{k}.npy"), np.asarray(v, dtype=np.float64))
    if not ok_all:
        bad = {n: w["parity"] for n, w in line["workloads"].items() if not w["parity"]["ok"]}
        raise SystemExit(f"bench_odometry.py: parity FAILED {bad}")


if __name__ == "__main__":
    main()
