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
sequence, byte for byte.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes every arm's
poses, priors, flags and kept points per frame as float64 .npy files."""
import math

import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
RANGE = 20.0
ARMS = {"window_0.25x4": (0.25, 4, None), "vmap_0.25x4": (0.25, 4, RANGE), "vmap_0.5x20": (0.5, 20, RANGE)}


def main():
    ap = h.parser()
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    ap.add_argument("--workload", default=None, help="run only this workload (e.g. 8x32)")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import map_points, voxel_downsample, voxel_map_update
    sv = args.source_voxel
    prm = h.c3_params()
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
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "filter_ms": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_map=n_map, n_scan=n_scan, max_range=RANGE)
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

            settings = {(a, tag): (v, c, d, s) for a, (v, c, d) in ARMS.items()
                        for tag, s in (("off", 0.0), ("on", v / math.sqrt(c)))}
            outs, ms, med = h.run_arms(ctx, {k: lambda p=p: run(*p) for k, p in settings.items()}, args.runs)
            res = outs
            # parity: the spaced voxel map at inf against the spaced long window, byte for byte
            s0 = 0.25 / 2.0
            inf_map = run(0.25, 4, math.inf, s0)
            long_w = run(0.25, 4, None, s0, max(len(q) for q in seqs) + 1)
            same_inf = all(h.same_bytes(a, b) for a, b in zip(inf_map, long_w))
            # every arm's map sizes per step from the twins; every spaced frame against its reconstruction
            filt = [[voxel_downsample(f, sv)[0] for f in q] for q in seqs]
            sizes = {}
            worst, same = 0.0, True
            for k, (v, c, d, s) in settings.items():
                def target(q, j, rs, M):
                    if d is None:
                        return voxel_downsample(h.window_map(filt[q], [r.T for r in rs], j, MAP_FRAMES), v, c, s)[0]
                    return voxel_map_update(M, filt[q][j - 1], rs[j - 1].T, v, c, d, s)
                sk, wk, sizes[k] = h.replay(ctx, prm if s > 0.0 else None, filt, res[k], target, CELL)
                same, worst = same and sk, max(worst, wk)
            ok = same_inf and same and worst <= 1e-8
            ok_all = ok_all and ok
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "inf_equals_long_window": same_inf,
                            "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8}}
            for (a, tag) in settings:
                w.setdefault(a, {})[tag] = {
                    **h.arm_block(n_frames, med[a, tag], ms[a, tag], res[a, tag], T_true),
                    "map_points_per_step": {"mean": float(np.mean(sizes[a, tag])), "max": int(max(sizes[a, tag]))}}
                dumps.update(h.result_dumps(f"spacing_{name}_{a}_{tag}", res[a, tag], h.FIELDS + ("n_points",)))
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

                        def ten(fn):                            # ten calls per timed run, each output dropped at once
                            for _ in range(10):
                                fn()
                        _, _, med = h.run_arms(ctx, {k: lambda fn=fn: ten(fn) for k, fn in calls.items()}, 5)
                        kept = {k: len(fn()[0][0]) for k, fn in calls.items()}
                        line["filter_ms"][f"{wn}_{v}x{c}"] = {"points": len(X), "kept": kept,
                                                             **{k: t / 10.0 for k, t in med.items()}}
    h.finish(args, line, dumps, ok_all, "bench_odometry_spacing.py: parity FAILED")


if __name__ == "__main__":
    main()
