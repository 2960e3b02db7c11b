"""Scan-to-map odometry with the window map against the persistent voxel map (dcreg_icp_run_odometry_map), on the
workloads of tools/bench_odometry_voxel.py; the arms run alternately on the same frames, medians reported.

  window      dcreg_icp_run_odometry_voxel_n, map 0.25 m x 4 points per voxel over a window of map_frames 10
  vmap_0.25x4 dcreg_icp_run_odometry_map, map 0.25 m x 4, max_distance = the scene's sensor range (20 m)
  vmap_0.5x20 dcreg_icp_run_odometry_map, map 0.5 m x 20 (KISS-ICP's cap), max_distance 20 m
  inf         dcreg_icp_run_odometry_map, map 0.25 m x 4, max_distance = inf

Every arm filters the frames at --source-voxel (0.25 m, one point per voxel).  Workloads (make_parking_sequence with
n_map = 2 000 000, n_scan = 100 000, max_range = 20 m): "1x128", one sequence of 128 frames (seed 47), and "8x32", eight
sequences of 32 frames (seeds 71..78).  Radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours, motion
"increments".  Timing as tools/bench_odometry.py: host arrays in, results out, the max of CUDA events on the context's
stream and the host wall clock, after a warm-up.

Per arm: frames/s, mean iterations and converged frames of the registered frames, map points per step (over the
sequences: the window's from the twin, the voxel maps' from the twin's M_k), and the largest error against the true
poses.  Parity (exits non-zero on a mismatch): the inf arm is the window call with map_frames >= the longest sequence,
byte for byte in T_out, T_prior, status, iterations, converged and points; every registered frame of the two finite
voxel-map arms equals its reconstruction set_target(twin M_k) + set_source + icp_run(T_prior) (status, iterations and
converged identical, pose <= 1e-8 on the SE(3) log).  Prints one JSON line with the card name and power limit;
--dump-outputs DIR writes every arm's poses, priors, flags and kept points per frame as float64 .npy files."""
import argparse
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_scans import card  # noqa: E402
from bench_odometry_voxel import dump_results  # noqa: E402
from bench_sequences import pose_errors  # noqa: E402

MAP_FRAMES = 10
CELL = 0.5
RANGE = 20.0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import map_points, voxel_downsample, voxel_map_update
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_odometry_map.py: no CUDA device - dcreg_b200 has no CPU fallback")
    sv = args.source_voxel
    prm = default_params(max_iterations=30, search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan = 200_000, 10_000
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan = 2_000_000, 100_000
    vmaps = {"vmap_0.25x4": (0.25, 4, RANGE), "vmap_0.5x20": (0.5, 20, RANGE), "inf": (0.25, 4, math.inf)}
    line = {"metric": "frames_per_s", "source_voxel": sv, "window": {"map_frames": MAP_FRAMES, "map_voxel": 0.25,
            "map_max_points": 4}, "voxel_maps": {a: {"map_voxel": v, "map_max_points": c, "max_distance": d}
                                                 for a, (v, c, d) in vmaps.items()},
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "card": card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream)

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w = time.perf_counter()
            e0.record(stream)
            out = fn()
            e1.record(stream)
            e1.synchronize()
            w = time.perf_counter() - w
            return out, max(e0.elapsed_time(e1), w * 1e3)

        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in spec:
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_map=n_map, n_scan=n_scan, max_range=RANGE)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            n_frames = len(deltas)

            def window(frames=MAP_FRAMES):
                return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=frames, cell_size=CELL, source_voxel=sv,
                                            map_voxel=0.25, map_max_points=4)

            def vmap(v, c, d):
                return lambda: ctx.icp_run_odometry_map(prm, seqs, T0, deltas, map_voxel=v, max_distance=d,
                                                        cell_size=CELL, source_voxel=sv, map_max_points=c)

            arms = {"window": window}
            arms.update({a: vmap(*p) for a, p in vmaps.items()})
            for fn in arms.values():                                           # warm-up
                fn()
            ms = {a: [] for a in arms}
            res = {}
            for _ in range(max(1, args.runs)):
                for a, fn in arms.items():
                    res[a], t = timed(fn)
                    ms[a].append(t)
            # parity: inf against the long window, byte for byte
            long_w = window(max(len(s) for s in seqs) + 1)
            same_inf = all((a.T.tobytes(), a.T_prior.tobytes(), a.status, a.iterations, a.converged, a.n_points) ==
                           (b.T.tobytes(), b.T_prior.tobytes(), b.status, b.iterations, b.converged, b.n_points)
                           for a, b in zip(res["inf"], long_w))
            # the finite voxel maps against their reconstructions; every arm's map sizes per step from the twins
            filt = [[voxel_downsample(f, sv)[0] for f in s] for s in seqs]
            sizes = {a: {} for a in arms}
            worst, same = 0.0, True
            for a in arms:
                k = 0
                for s, frames in enumerate(seqs):
                    rs = res[a][k:k + len(frames)]
                    if a == "window":
                        for j in range(1, len(frames)):
                            M = np.concatenate([map_points(rs[w].T, filt[s][w]) for w in range(max(0, j - MAP_FRAMES), j)])
                            sizes[a][j] = sizes[a].get(j, 0) + len(voxel_downsample(M, 0.25, 4)[0])
                    else:
                        v, c, d = vmaps[a]
                        M = np.zeros((0, 3), np.float32)
                        for j in range(len(frames)):
                            if j > 0:
                                sizes[a][j] = sizes[a].get(j, 0) + len(M)
                                if a != "inf":
                                    ctx.set_target(M, CELL)
                                    ctx.set_source(filt[s][j])
                                    single = ctx.icp_run(prm, rs[j].T_prior, want_log=False)
                                    b = rs[j]
                                    same = same and (b.status, b.iterations, b.converged) == (
                                        single.status, single.iterations, single.converged)
                                    worst = max(worst, float(o.se3_log_distance(single.T, b.T)))
                            M = voxel_map_update(M, filt[s][j], rs[j].T, v, c, d)
                    k += len(frames)
            ok = same_inf and same and worst <= 1e-8
            ok_all = ok_all and ok
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "inf_equals_long_window": same_inf,
                            "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8}}
            for a in arms:
                m = float(np.median(ms[a]))
                reg = [r for r in res[a] if r.iterations > 0]
                drift = pose_errors(T_true, [r.T for r in res[a]])
                per_step = [sizes[a][j] for j in sorted(sizes[a])]
                w[a] = {"frames_per_s": n_frames / (m * 1e-3), "ms": m, "runs_ms": ms[a],
                        "mean_iterations": float(np.mean([r.iterations for r in reg])),
                        "converged": int(sum(r.converged for r in reg)), "registered": len(reg),
                        "map_points_per_step": {"mean": float(np.mean(per_step)), "max": int(max(per_step))},
                        "max_err_vs_truth": {"trans_m": drift[0], "rot_deg": drift[1]}}
            line["workloads"][name] = w
            dumps.update({f"{name}_{a}": res[a] for a in arms})
    print(json.dumps(line))
    if args.dump_outputs:
        dump_results(args.dump_outputs, "odometry_map", dumps)
    if not ok_all:
        raise SystemExit("bench_odometry_map.py: parity FAILED")


if __name__ == "__main__":
    main()
