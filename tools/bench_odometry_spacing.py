"""The minimum point spacing of odometry's map filter (dcreg_set_map_spacing, KISS-ICP's AddPoints) on the workloads of
tools/bench_odometry_map.py; every arm runs with the spacing off and at map_voxel / sqrt(map_max_points), alternately on
the same frames, medians reported.

  window_0.25x4  dcreg_icp_run_odometry_voxel_n, map 0.25 m x 4 points per voxel over a window of map_frames 10
  vmap_0.25x4    dcreg_icp_run_odometry_map, map 0.25 m x 4, max_distance 20 m (the scene's sensor range)
  vmap_0.5x20    dcreg_icp_run_odometry_map, map 0.5 m x 20 (KISS-ICP's cap), max_distance 20 m

Frames are filtered at --source-voxel (0.25 m, one point per voxel); workloads, parameters and timing as in
tools/bench_odometry_map.py ("1x128": one sequence of 128 frames, seed 47; "8x32": eight of 32, seeds 71..78).

Per arm and setting: frames/s, mean iterations and converged frames of the registered frames, map points per step (from
the twins), and the largest error against the true poses.  The standalone filter: dcreg_voxel_downsample_spaced against
dcreg_voxel_downsample_n on a window of the first 10 filtered frames at their true poses (about 0.2 M points) and on one
of the first 5 unfiltered frames (about 0.5 M points), at 0.25 m x 4 and 0.5 m x 20, median ms per call (host arrays in
and out, one host sync each).  Parity (exits non-zero on a mismatch): every registered frame of every spaced arm equals
set_target(its twin map) + set_source + icp_run(T_prior) (status, iterations and converged identical, pose <= 1e-8 on
the SE(3) log), and the spaced voxel map at max_distance = inf is the spaced window with map_frames >= the longest
sequence, byte for byte.  Prints one JSON line with the card name and power limit."""
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
from bench_sequences import pose_errors  # noqa: E402

MAP_FRAMES = 10
CELL = 0.5
RANGE = 20.0
ARMS = {"window_0.25x4": (0.25, 4, None), "vmap_0.25x4": (0.25, 4, RANGE), "vmap_0.5x20": (0.5, 20, RANGE)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    ap.add_argument("--workload", default=None, help="run only this workload (e.g. 8x32)")
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import map_points, voxel_downsample, voxel_map_update
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_odometry_spacing.py: no CUDA device - dcreg_b200 has no CPU fallback")
    sv = args.source_voxel
    prm = default_params(max_iterations=30, search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan = 200_000, 10_000
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan = 2_000_000, 100_000
    if args.workload:
        workloads = {args.workload: workloads[args.workload]}
    line = {"metric": "frames_per_s", "source_voxel": sv, "map_frames": MAP_FRAMES,
            "arms": {a: {"map_voxel": v, "map_max_points": c, "max_distance": d, "spacing": v / math.sqrt(c)}
                     for a, (v, c, d) in ARMS.items()},
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "filter_ms": {}, "card": card()}
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
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_map=n_map, n_scan=n_scan, max_range=RANGE)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            n_frames = len(deltas)

            def run(v, c, d, s, frames=MAP_FRAMES):
                ctx.set_map_spacing(s)
                try:
                    if d is None:
                        return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=frames, cell_size=CELL,
                                                    source_voxel=sv, map_voxel=v, map_max_points=c)
                    return ctx.icp_run_odometry_map(prm, seqs, T0, deltas, map_voxel=v, max_distance=d, cell_size=CELL,
                                                    source_voxel=sv, map_max_points=c)
                finally:
                    ctx.set_map_spacing(0.0)

            arms = {}
            for a, (v, c, d) in ARMS.items():
                for tag, s in (("off", 0.0), ("on", v / math.sqrt(c))):
                    arms[a, tag] = (lambda v=v, c=c, d=d, s=s: run(v, c, d, s)), (v, c, d, s)
            for fn, _ in arms.values():                                        # warm-up
                fn()
            ms = {k: [] for k in arms}
            res = {}
            for _ in range(max(1, args.runs)):
                for k, (fn, _) in arms.items():
                    res[k], t = timed(fn)
                    ms[k].append(t)
            # parity: the spaced voxel map at inf against the spaced long window, byte for byte
            s0 = 0.25 / 2.0
            inf_map = run(0.25, 4, math.inf, s0)
            long_w = run(0.25, 4, None, s0, max(len(q) for q in seqs) + 1)
            same_inf = all((a.T.tobytes(), a.T_prior.tobytes(), a.status, a.iterations, a.converged, a.n_points) ==
                           (b.T.tobytes(), b.T_prior.tobytes(), b.status, b.iterations, b.converged, b.n_points)
                           for a, b in zip(inf_map, long_w))
            # every arm's map sizes per step from the twins; every spaced frame against its reconstruction
            filt = [[voxel_downsample(f, sv)[0] for f in q] for q in seqs]
            sizes = {k: {} for k in arms}
            worst, same = 0.0, True
            for k, (_, (v, c, d, s)) in arms.items():
                at = 0
                for q, frames in enumerate(seqs):
                    rs = res[k][at:at + len(frames)]
                    M = np.zeros((0, 3), np.float32)
                    for j in range(len(frames)):
                        if d is None and j > 0:
                            W = np.concatenate([map_points(rs[w].T, filt[q][w]) for w in range(max(0, j - MAP_FRAMES), j)])
                            M = voxel_downsample(W, v, c, s)[0]
                        if j > 0:
                            sizes[k][j] = sizes[k].get(j, 0) + len(M)
                            if s > 0.0:
                                ctx.set_target(M, CELL)
                                ctx.set_source(filt[q][j])
                                single = ctx.icp_run(prm, rs[j].T_prior, want_log=False)
                                b = rs[j]
                                same = same and (b.status, b.iterations, b.converged) == (
                                    single.status, single.iterations, single.converged)
                                worst = max(worst, float(o.se3_log_distance(single.T, b.T)))
                        if d is not None:
                            M = voxel_map_update(M, filt[q][j], rs[j].T, v, c, d, s)
                    at += len(frames)
            ok = same_inf and same and worst <= 1e-8
            ok_all = ok_all and ok
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "inf_equals_long_window": same_inf,
                            "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8}}
            for (a, tag) in arms:
                m = float(np.median(ms[a, tag]))
                reg = [r for r in res[a, tag] if r.iterations > 0]
                drift = pose_errors(T_true, [r.T for r in res[a, tag]])
                per_step = [sizes[a, tag][j] for j in sorted(sizes[a, tag])]
                w.setdefault(a, {})[tag] = {
                    "frames_per_s": n_frames / (m * 1e-3), "ms": m, "runs_ms": ms[a, tag],
                    "mean_iterations": float(np.mean([r.iterations for r in reg])),
                    "converged": int(sum(r.converged for r in reg)), "registered": len(reg),
                    "map_points_per_step": {"mean": float(np.mean(per_step)), "max": int(max(per_step))},
                    "max_err_vs_truth": {"trans_m": drift[0], "rot_deg": drift[1]}}
            line["workloads"][name] = w
            if name == next(iter(workloads)):
                Tt = T_true[:len(seqs[0])]
                windows = {
                    "filtered_10": np.concatenate([map_points(Tt[j], filt[0][j]) for j in range(min(10, len(Tt)))]),
                    "unfiltered_5": np.concatenate([map_points(Tt[j], seqs[0][j]) for j in range(min(5, len(Tt)))])}
                for wn, X in windows.items():
                    for v, c in ((0.25, 4), (0.5, 20)):
                        s = v / math.sqrt(c)
                        calls = {"n": lambda: ctx.voxel_downsample([X], v, c),
                                 "spaced": lambda: ctx.voxel_downsample([X], v, c, s)}
                        for fn in calls.values():
                            fn()
                        t = {k: [] for k in calls}
                        for _ in range(5):
                            for k, fn in calls.items():
                                t0 = time.perf_counter()
                                for _ in range(10):
                                    fn()
                                t[k].append((time.perf_counter() - t0) * 100.0)
                        kept = {k: len(fn()[0][0]) for k, fn in calls.items()}
                        line["filter_ms"][f"{wn}_{v}x{c}"] = {"points": len(X), "kept": kept,
                                                             **{k: float(np.median(x)) for k, x in t.items()}}
    print(json.dumps(line))
    if not ok_all:
        raise SystemExit("bench_odometry_spacing.py: parity FAILED")


if __name__ == "__main__":
    main()
