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
output equal to the twin's bit for bit.  Prints one JSON line with the card name and power limit; --dump-outputs DIR
writes every arm's poses, priors, flags and kept points per frame, and the filter's kept points and indices, as float64
.npy files."""
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
ARMS = [("raw", None, None), ("m0.25x1", 0.25, 1), ("m0.25x2", 0.25, 2), ("m0.25x4", 0.25, 4), ("m0.25x8", 0.25, 8),
        ("m0.25x20", 0.25, 20), ("m0.5x20", 0.5, 20)]


def main():
    ap = h.parser()
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import voxel_downsample
    from dcreg_b200.scenes import make_parking_sequence
    sv = args.source_voxel
    prm = h.c3_params()
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan, n_clouds = 200_000, 10_000, 4
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan, n_clouds = 2_000_000, 100_000, 64
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "source_voxel": sv, "n_scan": n_scan, "n_map": n_map,
            "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_map=n_map, n_scan=n_scan, max_range=20.0)
            n_frames = len(deltas)

            def arm(mv, cap):
                if mv is None:
                    return lambda: ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL)
                return lambda: ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL,
                                                    source_voxel=sv, map_voxel=mv, map_max_points=cap)
            outs, ms, med = h.run_arms(ctx, {a: arm(mv, cap) for a, mv, cap in ARMS}, args.runs)
            filt = [[voxel_downsample(f, sv)[0] for f in frames] for frames in seqs]
            w = {"sequences": len(seqs), "frames": n_frames, "tolerance": 1e-8}
            for a, mv, cap in ARMS:
                res = outs[a]
                # parity of a filtered arm, and its kept map sizes
                if mv is not None:
                    same, worst, step_maps = h.replay(ctx, prm, filt, res, lambda s, j, rs, M: voxel_downsample(
                        h.window_map(filt[s], [r.T for r in rs], j, MAP_FRAMES), mv, cap)[0], CELL, points=True)
                    ok = same and worst <= 1e-8
                    ok_all = ok_all and ok
                    parity = {"ok": ok, "identical_status_iterations_converged_points": same, "max_pose_err": worst}
                else:
                    step_maps = h.map_sizes([[len(f) for f in frames] for frames in seqs], MAP_FRAMES)
                    parity = None
                w[a] = {"map_voxel": mv, "map_max_points": cap, **h.arm_block(n_frames, med[a], ms[a], res, T_true),
                        "map_points_per_step": {"mean": float(np.mean(step_maps)), "max": int(max(step_maps))},
                        "parity": parity}
                dumps.update(h.result_dumps(f"sweep_{name}_{a}", res, h.FIELDS + ("n_points",)))
            line["workloads"][name] = w
        # the standalone filter: one device call over n_clouds clouds against the twin on each, at 1 and 20 points a voxel
        frames, _, _, _, _ = make_parking_sequence(n_clouds, seed=90, n_map=n_map, n_scan=n_scan, max_range=20.0)
        clouds = [f[:n_scan] for f in frames]
        n_pts = sum(len(c) for c in clouds)
        line["filter"] = {"clouds": len(clouds), "points": n_pts, "voxel": sv}
        for cap in (1, 20):
            outs, ms, med = h.run_arms(ctx, {"device": lambda: ctx.voxel_downsample(clouds, sv, cap),
                                             "twin": lambda: [voxel_downsample(c, sv, cap) for c in clouds]}, args.runs)
            got, twin = outs["device"], outs["twin"]
            equal = all(p.tobytes() == tp.tobytes() and np.array_equal(i, ti) for (p, i), (tp, ti) in zip(got, twin))
            ok_all = ok_all and equal
            line["filter"][f"max_points_{cap}"] = {
                "kept": int(sum(len(i) for _, i in got)), **h.rate(n_pts, med["device"], ms["device"], "device_", "points"),
                **h.rate(n_pts, med["twin"], ms["twin"], "twin_", "points"), "equal_to_twin": equal}
            for c, (p, i) in enumerate(got):
                dumps[f"sweep_filter_{cap}_{c}_xyz"], dumps[f"sweep_filter_{cap}_{c}_index"] = p, i
    h.finish(args, line, dumps, ok_all, "sweep_odometry_voxel.py: parity FAILED")


if __name__ == "__main__":
    main()
