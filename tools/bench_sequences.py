"""Frames/s of map-based localisation with chained priors: one dcreg_icp_run_sequences call against the per-frame host
loop a user runs without it (dcreg_set_source + dcreg_icp_run, then the next prior composed on the host from the result).

Workloads (make_parking_sequence: C3-shaped frames, ~6 k points each, against the 0.5 M-point parking map, odometry
increments perturbed by 3 cm / 0.3 deg per axis and step): "1x256", one sequence of 256 frames (seed 47), and "8x64",
eight sequences of 64 frames drawn with seeds 71..78.  Radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3
(icp_pk01.yaml), method Ours.  Both are timed the way tools/bench_scans.py times its batch: host arrays in, results out,
the max of CUDA events on the context's stream and the host wall clock, after a warm-up of both; --runs alternating
pairs, medians reported.  Every frame of the call is checked against the loop's own run of it (status, iterations,
converged identical, pose <= 1e-8 on the SE(3) log); the tool exits non-zero if that fails.  Also reported, not asserted:
the largest translation / rotation error against the true poses of the chained results and of the dead-reckoned priors
(T_init composed with the increments alone).  Prints one JSON line with the card name and power limit; --dump-outputs
DIR writes the chained poses, priors and flags as float64 .npy files."""
import numpy as np

import bench_harness as h


def main():
    args = h.parser().parse_args()
    h.require_gpu()
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context
    from dcreg_b200.api import compose_prior
    from dcreg_b200.scenes import make_parking_sequence
    prm = h.c3_params()
    workloads = {"1x256": [(256, 47)], "8x64": [(64, 71 + i) for i in range(8)]}
    line = {"metric": "frames_per_s", "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name, spec in workloads.items():
            # localisation starts from the scene's perturbed initial pose, against the scene's map
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in spec:
                frames, Tt, Ti0, D, park_map = make_parking_sequence(n, seed=seed)
                seqs.append(frames); T0.append(Ti0); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
            ctx.set_target(park_map, 0.5)
            n_frames = len(deltas)

            def frame_loop():
                out, k = [], 0
                for s, frames in enumerate(seqs):
                    T = T0[s]
                    for f in frames:
                        ctx.set_source(f)
                        r = ctx.icp_run(prm, T, want_log=False)
                        r.T_prior = T
                        out.append(r)
                        T = compose_prior(r.T, deltas[k])
                        k += 1
                return out

            outs, ms, med = h.run_arms(ctx, {"call": lambda: ctx.icp_run_sequences(prm, seqs, T0, deltas),
                                             "loop": frame_loop}, args.runs)
            res, loop = outs["call"], outs["loop"]
            same, worst = True, 0.0
            for b, s in zip(res, loop):
                same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
                worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok
            T_dr, k = [], 0                                                    # dead reckoning: increments alone
            for s, frames in enumerate(seqs):
                T = T0[s]
                for _ in frames:
                    T_dr.append(T)
                    T = compose_prior(T, deltas[k])
                    k += 1
            chained = h.pose_errors(T_true, [r.T for r in res])
            dead = h.pose_errors(T_true, T_dr)
            line["workloads"][name] = {
                "sequences": len(seqs), "frames": n_frames, **h.rate(n_frames, med["call"], ms["call"]),
                **h.rate(n_frames, med["loop"], ms["loop"], "loop_"), "speedup_vs_loop": med["loop"] / med["call"],
                "mean_iterations": float(np.mean([r.iterations for r in res])),
                "converged": int(sum(r.converged for r in res)),
                "points_per_frame": h.spread([len(f) for frames in seqs for f in frames]),
                "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst,
                           "tolerance": 1e-8},
                "max_err_vs_truth": {"chained": {"trans_m": chained[0], "rot_deg": chained[1]},
                                     "dead_reckoned_prior": {"trans_m": dead[0], "rot_deg": dead[1]}}}
            dumps.update(h.result_dumps(f"sequences_{name}", res))
    bad = {n: w["parity"] for n, w in line["workloads"].items() if not w["parity"]["ok"]}
    h.finish(args, line, dumps, ok_all, f"bench_sequences.py: parity FAILED {bad}")


if __name__ == "__main__":
    main()
