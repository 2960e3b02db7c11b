"""The map-input filter of scan-to-map odometry (dcreg_set_map_input_voxel, KISS-ICP's Voxelize) on the workloads of
tools/bench_odometry_map.py; the arms run alternately on the same frames, medians reported.

  kiss_split   KISS-ICP's recipe at v = 0.2 m (its default, max_range / 100): map input 0.5 v = 0.1 m, source 1.5 v =
               0.3 m, voxel map v = 0.2 m x 20 points per voxel pruned at 20 m
  kiss_joined  the same without the split: the 0.3 m source feeds the maps
  design_best  DESIGN.md's best arm before the split: source 0.25 m, voxel map 0.5 m x 20 pruned at 20 m

Workloads (make_parking_sequence with n_map = 2 000 000, n_scan = 100 000, max_range = 20 m): "1x128", one sequence of
128 frames (seed 47), and "8x32", eight sequences of 32 frames (seeds 71..78).  Radius and cell 0.5, 30 iterations,
ROT 1e-5 / TRANS 1e-3, method Ours, motion "increments".  Timing as tools/bench_odometry.py: host arrays in, results
out, the max of CUDA events on the context's stream and the host wall clock, after a warm-up.

Per arm: frames/s, mean iterations and converged frames of the registered frames, source points per frame and map
points per step (over the sequences, from the twin's M_k), and the largest error against the true poses.  Checks
(exits non-zero on a failure): every registered frame of kiss_split equals its reconstruction set_target(twin M_k of
F_in points) + set_source(F_s(F_in(frame))) + icp_run(T_prior) (status, iterations and converged identical, pose <=
1e-8 on the SE(3) log, n_points the twin's); and the identity case: map input 0.1 m with no source filter is byte for
byte the call with a 0.1 m source filter and no map-input filter.  Prints one JSON line with the card name and power
limit; --dump-outputs DIR writes every arm's poses, priors, flags and source points per frame as float64 .npy files."""
import numpy as np

import bench_harness as h

CELL = 0.5
RANGE = 20.0
V = 0.2                                   # KISS-ICP's voxel size at a 20 m range
ARMS = {"kiss_split": dict(map_input=0.5 * V, source_voxel=1.5 * V, map_voxel=V),
        "kiss_joined": dict(map_input=0.0, source_voxel=1.5 * V, map_voxel=V),
        "design_best": dict(map_input=0.0, source_voxel=0.25, map_voxel=0.5)}
CAP = 20


def main():
    ap = h.parser()
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import voxel_downsample, voxel_map_update
    prm = h.c3_params()
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan = 200_000, 10_000
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan = 2_000_000, 100_000
    line = {"metric": "frames_per_s", "arms": {a: {**p, "map_max_points": CAP, "max_distance": RANGE}
                                               for a, p in ARMS.items()},
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_map=n_map, n_scan=n_scan, max_range=RANGE)
            n_frames = len(deltas)

            def call(map_input, source_voxel, map_voxel):
                ctx.set_map_input_voxel(map_input)
                try:
                    return ctx.icp_run_odometry_map(prm, seqs, T0, deltas, map_voxel=map_voxel, max_distance=RANGE,
                                                    cell_size=CELL, source_voxel=source_voxel, map_max_points=CAP)
                finally:
                    ctx.set_map_input_voxel(0.0)

            arms = {a: (lambda p=p: call(**p)) for a, p in ARMS.items()}
            res, ms, med = h.run_arms(ctx, arms, args.runs)
            # the identity case, byte for byte
            a = call(0.5 * V, 0.0, V)
            b = call(0.0, 0.5 * V, V)
            identity = all(h.same_bytes(x, y) for x, y in zip(a, b))
            w = {"sequences": len(seqs), "frames": n_frames, "identity_ok": identity}
            ok = identity
            for arm, p in ARMS.items():
                fin = [[voxel_downsample(f, p["map_input"])[0] if p["map_input"] else f for f in s] for s in seqs]
                src = [[voxel_downsample(f, p["source_voxel"])[0] for f in s] for s in fin]
                ins = fin if p["map_input"] else src

                def target(s, j, rs, M, ins=ins, mv=p["map_voxel"]):
                    return voxel_map_update(M, ins[s][j - 1], rs[j - 1].T, mv, CAP, RANGE)
                same, worst, sizes = h.replay(ctx, prm if arm == "kiss_split" else None, src, res[arm], target, CELL,
                                              points=True)
                w[arm] = {**h.arm_block(n_frames, med[arm], ms[arm], res[arm], T_true),
                          "source_points_per_frame": float(np.mean([r.n_points for r in res[arm]])),
                          "map_points_per_step": {"mean": float(np.mean(sizes)), "max": int(max(sizes))}}
                if arm == "kiss_split":
                    twin_ok = same and worst <= 1e-8 and all(
                        r.n_points == len(f) for r, f in zip(res[arm], [f for s in src for f in s]))
                    w["twin"] = {"ok": twin_ok, "identical_status_iterations_converged": same,
                                 "max_pose_err": worst, "tolerance": 1e-8}
                    ok = ok and twin_ok
                dumps.update(h.result_dumps(f"odometry_map_input_{name}_{arm}", res[arm], h.FIELDS + ("n_points",)))
            ok_all = ok_all and ok
            line["workloads"][name] = w
    h.finish(args, line, dumps, ok_all, "measure_odometry_map_input.py: twin or identity check FAILED")


if __name__ == "__main__":
    main()
