"""The adaptive threshold of scan-to-map odometry (dcreg_icp_run_odometry_adaptive): what it costs and what it changes.

Workloads: make_parking_sequence(n, n_scan = 20 000, max_range = 20 m), "1x128" (one sequence of 128 frames, seed 47) and
"8x32" (eight sequences of 32 frames, seeds 71..78), every sequence anchored at its first true pose.  Window of 10 frames
(--map window) or the voxel map (--map voxel: source voxel 0.25, map voxel 0.25 keeping 4 points, pruned at 20 m), cell
0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours.

Arms, each with the true increments (`_true`) and with the constant-velocity model (`_cv`):
  fixed05    search radius 0.5 m for every frame
  ceiling    search radius 2.0 m for every frame (four rings of cells)
  adaptive   KISS-ICP's defaults (initial 2.0, min_motion 0.1, max_range 100) under the ceiling of 2.0 m
  pinned05   (true increments only) the threshold with initial_threshold = min_motion = 0.5 under a ceiling of 0.5: every
             radius is 0.5 and the bytes are fixed05's, so its time against fixed05 is the feature's own cost, one launch
             per step and the table reads (pinned_overhead_pct)
An arm whose odometry fails reports its message, the frame the failure names and the radii and iteration counts of that
sequence's frames of a rerun that stops short of it (`before_failure`).
Reported per arm: frames/s (median of --runs rounds of the arms in turn after a warm-up; CUDA events on the context's
stream and the host clock, the larger), mean iterations per registered frame, converged frames, the largest translation
error against the true poses (drift), and the min / median / max returned radius.  Parity (the tool exits non-zero if it
fails): every registered frame of the adaptive arms equals set_target(its map) + set_source + icp_run at its returned
radius (status, iterations, converged, pose to 1e-8), pinned05 equals fixed05 byte for byte, and repeated runs give the
same bytes.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes every arm's poses and
radii as float64 .npy files."""
import argparse
import json
import os
import re
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
CEILING = 2.0
VOXEL = dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)
MAX_DISTANCE = 20.0
WORKLOADS = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}


def same_bytes(a, b):
    return ((a.status, a.iterations, a.converged, a.n_points) == (b.status, b.iterations, b.converged, b.n_points)
            and a.T.tobytes() == b.T.tobytes() and a.T_prior.tobytes() == b.T_prior.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    ap.add_argument("--map", choices=["window", "voxel"], default="window")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import AdaptiveThreshold, DcregError, map_points, voxel_downsample, voxel_map_update
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_odometry_adaptive.py: no CUDA device - dcreg_b200 has no CPU fallback")

    def params(radius):
        return default_params(max_iterations=30, search_radius=radius, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                              kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    voxel = args.map == "voxel"
    line = {"metric": "frames_per_s", "map": args.map, "cell": CELL, "ceiling": CEILING, "workloads": {}, "card": card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream)

        def timed(fn):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            w = time.perf_counter()
            e0.record(stream)
            out = fn()
            e1.record(stream)
            e1.synchronize()
            return out, max(e0.elapsed_time(e1) / 1e3, time.perf_counter() - w)

        def call(seqs, T_init, deltas, radius, thr, cv):
            kw = dict(motion="constant_velocity" if cv else "increments", cell_size=CELL, adaptive=thr, want_radius=True)
            D = None if cv else deltas
            if voxel:
                return ctx.icp_run_odometry_map(params(radius), seqs, T_init, D, max_distance=MAX_DISTANCE, **VOXEL, **kw)
            return ctx.icp_run_odometry(params(radius), seqs, T_init, D, map_frames=MAP_FRAMES, **kw)

        def reconstructed(seqs, res):
            """every registered frame against its single run at the radius the call returned"""
            k, ok = 0, True
            for seq in seqs:
                rs = res[k:k + len(seq)]
                src = [voxel_downsample(f, VOXEL["source_voxel"], 1)[0] for f in seq] if voxel else seq
                M = np.zeros((0, 3), np.float32)
                for j in range(1, len(seq)):
                    if voxel:
                        M = voxel_map_update(M, src[j - 1], rs[j - 1].T, VOXEL["map_voxel"], VOXEL["map_max_points"],
                                             MAX_DISTANCE)
                    else:
                        M = np.concatenate([map_points(rs[i].T, seq[i]) for i in range(max(0, j - MAP_FRAMES), j)])
                    ctx.set_target(M, CELL)
                    ctx.set_source(src[j])
                    one = ctx.icp_run(params(rs[j].search_radius), rs[j].T_prior, want_log=False)
                    ok &= ((one.status, one.iterations, one.converged) == (rs[j].status, rs[j].iterations, rs[j].converged)
                           and o.se3_log_distance(one.T, rs[j].T) < 1e-8)
                k += len(seq)
            return bool(ok)

        for name in args.workloads.split(","):
            seqs, T_true, T_init, deltas = [], [], [], []
            for n, seed in WORKLOADS[name]:
                frames, Tt, _, _, _ = make_parking_sequence(n, seed=seed, n_scan=20_000, max_range=20.0)
                seqs.append(list(frames)); T_true.append(Tt); T_init.append(Tt[0])
                D = np.array([np.linalg.inv(Tt[i]) @ Tt[min(i + 1, n - 1)] for i in range(n)])
                deltas.append(D)
            T_true, T_init, deltas = np.concatenate(T_true), np.array(T_init), np.concatenate(deltas)
            n_frames, n_reg = len(T_true), len(T_true) - len(seqs)
            first = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
            kiss = AdaptiveThreshold(2.0, 0.1, 100.0)
            arms = {}
            for cv in (False, True):
                tag = "_cv" if cv else "_true"
                arms["fixed05" + tag] = lambda cv=cv: call(seqs, T_init, deltas, 0.5, None, cv)
                arms["ceiling" + tag] = lambda cv=cv: call(seqs, T_init, deltas, CEILING, None, cv)
                arms["adaptive" + tag] = lambda cv=cv: call(seqs, T_init, deltas, CEILING, kiss, cv)
            arms["pinned05_true"] = lambda: call(seqs, T_init, deltas, 0.5, AdaptiveThreshold(0.5, 0.5, 100.0), False)
            res = {}
            for a in arms:
                try:
                    res[a] = arms[a]()
                except DcregError as e:
                    res[a] = str(e)
            live = [a for a in arms if not isinstance(res[a], str)]
            times = {a: [] for a in live}
            for _ in range(args.runs):
                for a in live:
                    r, dt = timed(arms[a])
                    times[a].append(dt)
                    ok_all &= all(same_bytes(x, y) for x, y in zip(r, res[a]))
            out = {"frames": n_frames, "arms": {}}
            for a in arms:
                if isinstance(res[a], str):
                    # the frames of the failing sequence before the frame the message names, from a shorter rerun
                    rec = {"error": res[a]}
                    m = re.search(r"sequence (\d+), frame (\d+) \(frame (\d+) of the sequence\)", res[a])
                    if m:
                        s, j = int(m.group(1)), int(m.group(3))
                        cv, kind = a.endswith("_cv"), a.split("_")[0]
                        radius, thr = {"fixed05": (0.5, None), "ceiling": (CEILING, None), "adaptive": (CEILING, kiss),
                                       "pinned05": (0.5, AdaptiveThreshold(0.5, 0.5, 100.0))}[kind]
                        try:
                            short = call([seqs[s][:j]], T_init[s:s + 1], deltas[first[s]:first[s] + j], radius, thr, cv)
                            dt, _ = pose_errors(T_true[first[s]:first[s] + j], [r.T for r in short])
                            rec["before_failure"] = {
                                "sequence": s, "frames": j, "max_trans_err_m": round(dt, 4),
                                "last_radii": [round(r.search_radius, 4) for r in short[-8:]],
                                "last_iterations": [r.iterations for r in short[-8:]],
                                "last_converged": [int(r.converged) for r in short[-8:]],
                                "last_trans_err_m": [round(float(np.linalg.norm(r.T[:3, 3] - T[:3, 3])), 3)
                                                     for r, T in zip(short[-8:], T_true[first[s] + j - 8:first[s] + j])]}
                        except DcregError as e:
                            rec["before_failure"] = str(e)
                    out["arms"][a] = rec
                    continue
                dt, dr = pose_errors(T_true, [r.T for r in res[a]])
                rad = np.array([r.search_radius for r in res[a] if r.search_radius > 0.0])
                rec = {"frames_per_s": round(n_frames / float(np.median(times[a])), 1),
                       "mean_iterations": round(sum(r.iterations for r in res[a]) / n_reg, 2),
                       "converged": int(sum(r.converged for r in res[a])),
                       "max_trans_err_m": round(dt, 4), "max_rot_err_deg": round(dr, 4),
                       "radius_min_med_max": [round(float(x), 4) for x in (rad.min(), np.median(rad), rad.max())]}
                if a.startswith("adaptive"):
                    rec["reconstruction"] = reconstructed(seqs, res[a])
                    ok_all &= rec["reconstruction"]
                out["arms"][a] = rec
                dumps[f"{name}_{a}_T"] = np.array([r.T for r in res[a]])
                dumps[f"{name}_{a}_radius"] = np.array([r.search_radius for r in res[a]])
            if "pinned05_true" in live and "fixed05_true" in live:
                same = all(same_bytes(x, y) for x, y in zip(res["pinned05_true"], res["fixed05_true"]))
                out["pinned_equals_fixed"] = bool(same)
                ok_all &= same
                out["pinned_overhead_pct"] = round(
                    100.0 * (np.median(times["pinned05_true"]) / np.median(times["fixed05_true"]) - 1.0), 2)
            line["workloads"][name] = out
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in dumps.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), v)
    line["parity"] = bool(ok_all)
    print(json.dumps(line))
    if not ok_all:
        sys.exit(1)


if __name__ == "__main__":
    main()
