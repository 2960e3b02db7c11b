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
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5


def main():
    args = h.parser().parse_args()
    h.require_gpu()
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context
    from dcreg_b200.api import compose_prior
    prm = h.c3_params()
    prm1 = h.c3_params(max_iterations=1)
    workloads = {"1x256": [(256, 47)], "8x64": [(64, 71 + i) for i in range(8)]}
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = h.parking_sequences(spec, n_scan=20_000, max_range=20.0)
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
                        ctx.set_target(h.window_map(frames, Ts, j, MAP_FRAMES), CELL)
                        ctx.set_source(frames[j])
                        r = ctx.icp_run(prm, T, want_log=False)
                        r.T_prior = T
                        out.append(r)
                        Ts.append(r.T)
                        k += 1
                return out

            outs, ms, med = h.run_arms(ctx, {"call": call, "loop": frame_loop, "one": lambda: call(prm1)}, args.runs)
            res, loop = outs["call"], outs["loop"]
            # parity: every registered frame against its run on the map rebuilt from the call's own results
            same, worst, _ = h.replay(ctx, prm, seqs, res,
                                      lambda s, j, rs, M: h.window_map(seqs[s], [r.T for r in rs], j, MAP_FRAMES), CELL)
            chain_diff = max([0.0] + [float(o.se3_log_distance(l.T, r.T)) for l, r in zip(loop, res) if l is not None])
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok
            map_pts = h.map_sizes([[len(f) for f in frames] for frames in seqs], MAP_FRAMES)
            line["workloads"][name] = {
                "sequences": len(seqs), "frames": n_frames, **h.arm_block(n_frames, med["call"], ms["call"], res, T_true),
                **h.rate(n_frames, med["loop"], ms["loop"], "loop_"), "speedup_vs_loop": med["loop"] / med["call"],
                "one_iteration_call_ms": med["one"], "one_iteration_runs_ms": ms["one"],
                "points_per_frame": h.spread([len(f) for frames in seqs for f in frames]),
                "map_points_per_step": {"mean": float(np.mean(map_pts)), "max": int(max(map_pts))},
                "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst,
                           "tolerance": 1e-8},
                "host_loop_chain_max_pose_diff": chain_diff}
            dumps.update(h.result_dumps(f"odometry_{name}", res))
    bad = {n: w["parity"] for n, w in line["workloads"].items() if not w["parity"]["ok"]}
    h.finish(args, line, dumps, ok_all, f"bench_odometry.py: parity FAILED {bad}")


if __name__ == "__main__":
    main()
