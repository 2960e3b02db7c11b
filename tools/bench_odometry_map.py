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
import math

import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
RANGE = 20.0


def main():
    ap = h.parser()
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import voxel_downsample, voxel_map_update
    sv = args.source_voxel
    prm = h.c3_params()
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
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_map=n_map, n_scan=n_scan, max_range=RANGE)
            n_frames = len(deltas)

            def window(frames=MAP_FRAMES):
                return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=frames, cell_size=CELL, source_voxel=sv,
                                            map_voxel=0.25, map_max_points=4)

            def vmap(v, c, d):
                return lambda: ctx.icp_run_odometry_map(prm, seqs, T0, deltas, map_voxel=v, max_distance=d,
                                                        cell_size=CELL, source_voxel=sv, map_max_points=c)

            arms = {"window": window}
            arms.update({a: vmap(*p) for a, p in vmaps.items()})
            outs, ms, med = h.run_arms(ctx, arms, args.runs)
            res = outs
            # parity: inf against the long window, byte for byte
            long_w = window(max(len(s) for s in seqs) + 1)
            same_inf = all(h.same_bytes(a, b) for a, b in zip(res["inf"], long_w))
            # the finite voxel maps against their reconstructions; every arm's map sizes per step from the twins
            filt = [[voxel_downsample(f, sv)[0] for f in s] for s in seqs]
            _, _, sizes = h.replay(ctx, None, filt, res["window"], lambda s, j, rs, M: voxel_downsample(
                h.window_map(filt[s], [r.T for r in rs], j, MAP_FRAMES), 0.25, 4)[0], CELL)
            sizes = {"window": sizes}
            worst, same = 0.0, True
            for a, (v, c, d) in vmaps.items():
                def target(s, j, rs, M):
                    return voxel_map_update(M, filt[s][j - 1], rs[j - 1].T, v, c, d)
                sa, wa, sizes[a] = h.replay(ctx, None if a == "inf" else prm, filt, res[a], target, CELL)
                same, worst = same and sa, max(worst, wa)
            ok = same_inf and same and worst <= 1e-8
            ok_all = ok_all and ok
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "inf_equals_long_window": same_inf,
                            "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8}}
            for a in arms:
                w[a] = {**h.arm_block(n_frames, med[a], ms[a], res[a], T_true),
                        "map_points_per_step": {"mean": float(np.mean(sizes[a])), "max": int(max(sizes[a]))}}
            line["workloads"][name] = w
            for a in arms:
                dumps.update(h.result_dumps(f"odometry_map_{name}_{a}", res[a], h.FIELDS + ("n_points",)))
    h.finish(args, line, dumps, ok_all, "bench_odometry_map.py: parity FAILED")


if __name__ == "__main__":
    main()
