"""Pairs/s of registering many scan/target pairs, each source against its own target: one dcreg_icp_run_pairs call
against the per-pair dcreg_set_target + dcreg_set_source + dcreg_icp_run loop a user runs without it.

Workload: --pairs (64) pairs of make_parking_pairs (seed 53): frame k + 1 (~6 k points) against the ~100 k-point local
submap around pose k, radius 0.5 (also the targets' cell size), 30 iterations, ROT 1e-5 / TRANS 1e-3 (icp_pk01.yaml),
method Ours.  Both are timed as tools/bench_scans.py times them: host arrays in, results out, the max of CUDA events on
the context's stream and the host wall clock, after a warm-up of both; --runs alternating pairs, medians reported.
The set-up alone (host concatenation and upload of sources and targets, the targets' grid build, the sources' pack and sort, state read-back)
is a call with max_iterations = 0, which runs no iteration and does nothing else.  Every pair of the batch is checked
against its own sequential run (status, iterations, converged identical, pose <= 1e-8 on the SE(3) log); the tool exits
non-zero if that fails.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes the batched
poses and flags as float64 .npy files."""
import numpy as np

import bench_harness as h


def main():
    ap = h.parser()
    ap.add_argument("--pairs", type=int, default=64)
    args = ap.parse_args()
    h.require_gpu()
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context
    from dcreg_b200.scenes import make_parking_pairs
    sources, targets, _, T_init = make_parking_pairs(args.pairs, seed=53)
    radius = 0.5
    prm = h.c3_params(search_radius=radius)
    prm0 = h.c3_params(search_radius=radius, max_iterations=0)
    with Context(0) as ctx:

        def pair_loop():
            out = []
            for s, t, T in zip(sources, targets, T_init):
                ctx.set_target(t, radius)
                ctx.set_source(s)
                out.append(ctx.icp_run(prm, T, want_log=False))
            return out

        outs, ms, med = h.run_arms(ctx, {"batch": lambda: ctx.icp_run_pairs(prm, sources, targets, T_init),
                                         "setup": lambda: ctx.icp_run_pairs(prm0, sources, targets, T_init),
                                         "seq": pair_loop}, args.runs)
    batch, seq = outs["batch"], outs["seq"]
    same, worst = True, 0.0
    for b, s in zip(batch, seq):
        same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
        worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
    ok = same and worst <= 1e-8
    n = args.pairs
    line = {"metric": "pairs_per_s", "pairs": n, **h.rate(n, med["batch"], ms["batch"], unit="pairs"),
            "setup_ms": med["setup"], "setup_runs_ms": ms["setup"],
            **h.rate(n, med["seq"], ms["seq"], "sequential_", "pairs"), "speedup_vs_sequential": med["seq"] / med["batch"],
            "mean_iterations": float(np.mean([b.iterations for b in batch])),
            "converged": int(sum(b.converged for b in batch)),
            "source_points": h.spread([len(s) for s in sources]), "target_points": h.spread([len(t) for t in targets]),
            "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8},
            "card": h.card()}
    h.finish(args, line, h.result_dumps("pairs", batch, ("T", "iterations", "converged", "status")), ok,
             f"bench_pairs.py: parity FAILED (status/iterations/converged identical: {same}, max pose err {worst:.3e})")


if __name__ == "__main__":
    main()
