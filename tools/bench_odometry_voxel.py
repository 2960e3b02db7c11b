"""Scan-to-map odometry on LiDAR-sized frames, with and without voxel filters: three arms run alternately on the same
frames, medians reported.

  raw     dcreg_icp_run_odometry on the full frames (maps of full frames)
  host    the NumPy twin api.voxel_downsample on every frame on the host (timed), then dcreg_icp_run_odometry on the
          filtered frames (maps of filtered frames, not filtered themselves)
  device  dcreg_icp_run_odometry_voxel(source_voxel, map_voxel): frames and every step's local maps filtered on the device

Workloads (make_parking_sequence with n_map = 2 000 000, n_scan = 100 000, max_range = 20 m): "1x128", one sequence of
128 frames (seed 47), and "8x32", eight sequences of 32 frames (seeds 71..78), each anchored at its first true pose.
map_frames 10, radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours, motion "increments", voxel sizes
--source-voxel / --map-voxel (0.25 / 0.25).  Timing as tools/bench_odometry.py: host arrays in, results out, the max of
CUDA events on the context's stream and the host wall clock, after a warm-up.

Per arm: frames/s, mean iterations of the registered frames, points per frame, map points per step (over the
sequences), and the largest error against the true poses.  Also the standalone filter: Context.voxel_downsample of 64
clouds of 100 000 points in one call (host arrays in and out) against the twin on each cloud, in points/s.

Parity (asserted; exits non-zero on a mismatch): every registered frame of the device arm against its reconstruction
with the twin (set_target(filtered map, cell) + set_source(filtered frame) + icp_run(T_prior)): status, iterations and
converged identical, pose <= 1e-8 on the SE(3) log; and the device filter's output equal to the twin's bit for bit.
Prints one JSON line with the card name and power limit; --dump-outputs DIR writes every arm's poses, priors, flags and
kept points per frame, and the filter's kept points and indices, as float64 .npy files."""
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5


def main():
    ap = h.parser()
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--map-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import voxel_downsample
    from dcreg_b200.scenes import make_parking_sequence
    sv, mv = args.source_voxel, args.map_voxel
    prm = h.c3_params()
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan, n_clouds = 200_000, 10_000, 4
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan, n_clouds = 2_000_000, 100_000, 64
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "source_voxel": sv, "map_voxel": mv,
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_map=n_map, n_scan=n_scan, max_range=20.0)
            n_frames = len(deltas)

            def raw():
                return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL)

            def host():
                filt = [[voxel_downsample(f, sv)[0] for f in s] for s in seqs]
                return ctx.icp_run_odometry(prm, filt, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL)

            def device():
                return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=MAP_FRAMES, cell_size=CELL,
                                            source_voxel=sv, map_voxel=mv)

            arms = {"raw": raw, "host": host, "device": device}
            outs, ms, med = h.run_arms(ctx, arms, args.runs)
            res = outs
            # parity of the device arm, and its filtered map sizes
            filt = [[voxel_downsample(f, sv)[0] for f in s] for s in seqs]
            same, worst, dev_maps = h.replay(ctx, prm, filt, res["device"], lambda s, j, rs, M: voxel_downsample(
                h.window_map(filt[s], [r.T for r in rs], j, MAP_FRAMES), mv)[0], CELL, points=True)
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok
            maps = {a: h.map_sizes([[r.n_points for r in rs] for rs in h.per_sequence(seqs, res[a])], MAP_FRAMES)
                    for a in ("raw", "host")}
            maps["device"] = dev_maps
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "identical_status_iterations_converged_points": same, "max_pose_err": worst,
                            "tolerance": 1e-8}}
            for a in arms:
                w[a] = {**h.arm_block(n_frames, med[a], ms[a], res[a], T_true),
                        "points_per_frame_mean": float(np.mean([r.n_points for r in res[a]])),
                        "map_points_per_step": {"mean": float(np.mean(maps[a])), "max": int(max(maps[a]))}}
            line["workloads"][name] = w
            for a in arms:
                dumps.update(h.result_dumps(f"odometry_voxel_{name}_{a}", res[a], h.FIELDS + ("n_points",)))
        # the standalone filter: one device call over n_clouds clouds against the twin on each
        frames, _, _, _, _ = make_parking_sequence(n_clouds, seed=90, n_map=n_map, n_scan=n_scan, max_range=20.0)
        clouds = [f[:n_scan] for f in frames]
        n_pts = sum(len(c) for c in clouds)
        outs, ms, med = h.run_arms(ctx, {"device": lambda: ctx.voxel_downsample(clouds, sv),
                                         "twin": lambda: [voxel_downsample(c, sv) for c in clouds]}, args.runs)
        got, twin = outs["device"], outs["twin"]
        equal = all(p.tobytes() == tp.tobytes() and np.array_equal(i, ti) for (p, i), (tp, ti) in zip(got, twin))
        ok_all = ok_all and equal
        line["filter"] = {"clouds": len(clouds), "points": n_pts, "voxel": sv, "kept": int(sum(len(i) for _, i in got)),
                          **h.rate(n_pts, med["device"], ms["device"], "device_", "points"),
                          **h.rate(n_pts, med["twin"], ms["twin"], "twin_", "points"), "equal_to_twin": equal}
        for c, (p, i) in enumerate(got):
            dumps[f"voxel_filter_{c}_xyz"], dumps[f"voxel_filter_{c}_index"] = p, i
    h.finish(args, line, dumps, ok_all, "bench_odometry_voxel.py: parity FAILED")


if __name__ == "__main__":
    main()
