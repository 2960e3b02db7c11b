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

from bench_scans import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o                                                   # se3 log distance (NumPy), checker only
    from dcreg_b200 import Context, default_params
    from dcreg_b200.scenes import make_parking_pairs
    if not torch.cuda.is_available():
        raise SystemExit("bench_pairs.py: no CUDA device - dcreg_b200 has no CPU fallback")
    sources, targets, _, T_init = make_parking_pairs(args.pairs, seed=53)
    radius = 0.5
    kw = dict(search_radius=radius, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0,
              detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    prm = default_params(max_iterations=30, **kw)
    prm0 = default_params(max_iterations=0, **kw)
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream)

        def pair_loop():
            out = []
            for s, t, T in zip(sources, targets, T_init):
                ctx.set_target(t, radius)
                ctx.set_source(s)
                out.append(ctx.icp_run(prm, T, want_log=False))
            return out

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w = time.perf_counter()
            e0.record(stream)
            out = fn()
            e1.record(stream)
            e1.synchronize()
            w = time.perf_counter() - w
            return out, max(e0.elapsed_time(e1), w * 1e3)

        ctx.icp_run_pairs(prm, sources, targets, T_init)                        # warm-up of all shapes
        ctx.icp_run_pairs(prm0, sources, targets, T_init)
        pair_loop()
        batch_ms, seq_ms, setup_ms = [], [], []
        for _ in range(max(1, args.runs)):
            batch, ms = timed(lambda: ctx.icp_run_pairs(prm, sources, targets, T_init))
            batch_ms.append(ms)
            _, ms = timed(lambda: ctx.icp_run_pairs(prm0, sources, targets, T_init))
            setup_ms.append(ms)
            seq, ms = timed(pair_loop)
            seq_ms.append(ms)
    same, worst = True, 0.0
    for b, s in zip(batch, seq):
        same = same and (b.status, b.iterations, b.converged) == (s.status, s.iterations, s.converged)
        worst = max(worst, float(o.se3_log_distance(s.T, b.T)))
    ok = same and worst <= 1e-8
    n = args.pairs
    bm, sm, um = float(np.median(batch_ms)), float(np.median(seq_ms)), float(np.median(setup_ms))
    ss, ts = [len(s) for s in sources], [len(t) for t in targets]
    line = {"metric": "pairs_per_s", "pairs": n, "pairs_per_s": n / (bm * 1e-3), "ms": bm, "runs_ms": batch_ms,
            "setup_ms": um, "setup_runs_ms": setup_ms,
            "sequential_pairs_per_s": n / (sm * 1e-3), "sequential_ms": sm, "sequential_runs_ms": seq_ms,
            "speedup_vs_sequential": sm / bm, "mean_iterations": float(np.mean([b.iterations for b in batch])),
            "converged": int(sum(b.converged for b in batch)),
            "source_points": {"min": int(min(ss)), "max": int(max(ss)), "total": int(sum(ss))},
            "target_points": {"min": int(min(ts)), "max": int(max(ts)), "total": int(sum(ts))},
            "parity": {"ok": ok, "identical_status_iterations_converged": same, "max_pose_err": worst, "tolerance": 1e-8},
            "card": card()}
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in {"pairs_T": [b.T for b in batch], "pairs_iterations": [b.iterations for b in batch],
                     "pairs_converged": [b.converged for b in batch], "pairs_status": [b.status for b in batch]}.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), np.asarray(v, dtype=np.float64))
    if not ok:
        raise SystemExit(f"bench_pairs.py: parity FAILED (status/iterations/converged identical: {same}, max pose err {worst:.3e})")


if __name__ == "__main__":
    main()
