"""Scan-to-map odometry with capped map filters: where between the raw call and the one-point-per-voxel map filter does
a map that keeps up to N points per voxel land?  All arms run alternately on the same frames, medians reported.

  raw         dcreg_icp_run_odometry on the full frames (maps of full frames)
  m<v>x<N>    dcreg_icp_run_odometry_voxel_n: frames filtered at --source-voxel (one point per voxel), every step's
              local map at map_voxel v keeping up to N points per voxel; v 0.25 with N in 1, 2, 4, 8, 20, and v 0.5
              with N 20.  m0.25x1 is dcreg_icp_run_odometry_voxel(0.25, 0.25)

Workloads as tools/bench_odometry_voxel.py (make_parking_sequence with n_map = 2 000 000, n_scan = 100 000, max_range
= 20 m): "1x128", one sequence of 128 frames (seed 47), and "8x32", eight sequences of 32 frames (seeds 71..78), each
anchored at its first true pose.  map_frames 10, radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method
Ours, motion "increments".  Timing: host arrays in, results out, the max of CUDA events on the context's stream and the
host wall clock, after a warm-up; one run of every arm per round, --runs rounds.

Per arm: frames/s, mean iterations and converged count of the registered frames, map points per step (over the
sequences: the twin's kept maps for the filtered arms, the frames' sizes for the raw call), and the largest error
against the true poses.  Also the standalone filter: Context.voxel_downsample of 64 clouds of 100 000 points in one
call at max_points 1 and 20, against the twin on each cloud.

Parity (asserted; exits non-zero on a mismatch): every registered frame of every filtered arm against its
reconstruction with the twin (set_target(filtered map, cell) + set_source(filtered frame) + icp_run(T_prior)): status,
iterations and converged identical, pose <= 1e-8 on the SE(3) log, n_points the twin's; and the standalone filter's
output equal to the twin's bit for bit.  Prints one JSON line with the card name and power limit."""
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

from bench_odometry_voxel import map_sizes  # noqa: E402
from bench_scans import card  # noqa: E402
from bench_sequences import pose_errors  # noqa: E402

MAP_FRAMES = 10
CELL = 0.5
ARMS = [("raw", None, None), ("m0.25x1", 0.25, 1), ("m0.25x2", 0.25, 2), ("m0.25x4", 0.25, 4), ("m0.25x8", 0.25, 8),
        ("m0.25x20", 0.25, 20), ("m0.5x20", 0.5, 20)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import map_points, voxel_downsample
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("sweep_odometry_voxel.py: no CUDA device - dcreg_b200 has no CPU fallback")
    sv = args.source_voxel
    prm = default_params(max_iterations=30, search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan, n_clouds = 200_000, 10_000, 4
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan, n_clouds = 2_000_000, 100_000, 64
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "source_voxel": sv, "n_scan": n_scan, "n_map": n_map,
            "workloads": {}, "card": card()}
    ok_all = True
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
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_map=n_map, n_scan=n_scan, max_range=20.0)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            n_frames = len(deltas)

            def arm(mv, cap):
                if mv is None:
                    return lambda: ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL)
                return lambda: ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL,
                                                    source_voxel=sv, map_voxel=mv, map_max_points=cap)
            arms = {a: arm(mv, cap) for a, mv, cap in ARMS}
            for fn in arms.values():                                           # warm-up
                fn()
            ms = {a: [] for a in arms}
            res = {}
            for _ in range(max(1, args.runs)):
                for a, fn in arms.items():
                    res[a], t = timed(fn)
                    ms[a].append(t)
            filt = [[voxel_downsample(f, sv)[0] for f in frames] for frames in seqs]
            w = {"sequences": len(seqs), "frames": n_frames, "tolerance": 1e-8}
            for a, mv, cap in ARMS:
                # parity of a filtered arm, and its kept map sizes
                same, worst, k, maps = True, 0.0, 0, {}
                if mv is not None:
                    for s, frames in enumerate(seqs):
                        rs = res[a][k:k + len(frames)]
                        placed = [map_points(rs[j].T, filt[s][j]) for j in range(len(frames))]
                        for j in range(1, len(frames)):
                            M = voxel_downsample(np.concatenate(placed[max(0, j - MAP_FRAMES):j]), mv, cap)[0]
                            maps[j] = maps.get(j, 0) + len(M)
                            ctx.set_target(M, CELL)
                            ctx.set_source(filt[s][j])
                            single = ctx.icp_run(prm, rs[j].T_prior, want_log=False)
                            b = rs[j]
                            same = same and (b.status, b.iterations, b.converged) == (single.status, single.iterations,
                                                                                       single.converged)
                            same = same and b.n_points == len(filt[s][j])
                            worst = max(worst, float(o.se3_log_distance(single.T, b.T)))
                        k += len(frames)
                    ok = same and worst <= 1e-8
                    ok_all = ok_all and ok
                    step_maps = [maps[j] for j in sorted(maps)]
                    parity = {"ok": ok, "identical_status_iterations_converged_points": same, "max_pose_err": worst}
                else:
                    step_maps = map_sizes([[len(f) for f in frames] for frames in seqs])
                    parity = None
                m = float(np.median(ms[a]))
                reg = [r for r in res[a] if r.iterations > 0]
                drift = pose_errors(T_true, [r.T for r in res[a]])
                w[a] = {"map_voxel": mv, "map_max_points": cap, "frames_per_s": n_frames / (m * 1e-3), "ms": m,
                        "runs_ms": ms[a], "mean_iterations": float(np.mean([r.iterations for r in reg])),
                        "converged": int(sum(r.converged for r in reg)), "registered": len(reg),
                        "map_points_per_step": {"mean": float(np.mean(step_maps)), "max": int(max(step_maps))},
                        "max_err_vs_truth": {"trans_m": drift[0], "rot_deg": drift[1]}, "parity": parity}
            line["workloads"][name] = w
        # the standalone filter: one device call over n_clouds clouds against the twin on each, at 1 and 20 points a voxel
        frames, _, _, _, _ = make_parking_sequence(n_clouds, seed=90, n_map=n_map, n_scan=n_scan, max_range=20.0)
        clouds = [f[:n_scan] for f in frames]
        n_pts = sum(len(c) for c in clouds)
        line["filter"] = {"clouds": len(clouds), "points": n_pts, "voxel": sv}
        for cap in (1, 20):
            ctx.voxel_downsample(clouds, sv, cap)
            dev_ms, twin_ms = [], []
            for _ in range(max(1, args.runs)):
                got, t = timed(lambda: ctx.voxel_downsample(clouds, sv, cap))
                dev_ms.append(t)
                t0 = time.perf_counter()
                twin = [voxel_downsample(c, sv, cap) for c in clouds]
                twin_ms.append((time.perf_counter() - t0) * 1e3)
            equal = all(p.tobytes() == tp.tobytes() and np.array_equal(i, ti) for (p, i), (tp, ti) in zip(got, twin))
            ok_all = ok_all and equal
            dm, tm = float(np.median(dev_ms)), float(np.median(twin_ms))
            line["filter"][f"max_points_{cap}"] = {
                "kept": int(sum(len(i) for _, i in got)), "device_ms": dm, "device_points_per_s": n_pts / (dm * 1e-3),
                "device_runs_ms": dev_ms, "twin_ms": tm, "twin_points_per_s": n_pts / (tm * 1e-3), "twin_runs_ms": twin_ms,
                "equal_to_twin": equal}
    print(json.dumps(line))
    if not ok_all:
        raise SystemExit("sweep_odometry_voxel.py: parity FAILED")


if __name__ == "__main__":
    main()
