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
import re

import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
CEILING = 2.0
VOXEL = dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)
MAX_DISTANCE = 20.0
WORKLOADS = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    ap.add_argument("--map", choices=["window", "voxel"], default="window")
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import AdaptiveThreshold, DcregError, voxel_downsample, voxel_map_update

    def params(radius):
        return h.c3_params(search_radius=radius)
    voxel = args.map == "voxel"
    line = {"metric": "frames_per_s", "map": args.map, "cell": CELL, "ceiling": CEILING, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:

        def call(seqs, T_init, deltas, radius, thr, cv):
            kw = dict(motion="constant_velocity" if cv else "increments", cell_size=CELL, adaptive=thr, want_radius=True)
            D = None if cv else deltas
            if voxel:
                return ctx.icp_run_odometry_map(params(radius), seqs, T_init, D, max_distance=MAX_DISTANCE, **VOXEL, **kw)
            return ctx.icp_run_odometry(params(radius), seqs, T_init, D, map_frames=MAP_FRAMES, **kw)

        def reconstructed(seqs, res):
            """every registered frame against its single run at the radius the call returned"""
            src = [[voxel_downsample(f, VOXEL["source_voxel"], 1)[0] for f in seq] for seq in seqs] if voxel else seqs

            def target(s, j, rs, M):
                if voxel:
                    return voxel_map_update(M, src[s][j - 1], rs[j - 1].T, VOXEL["map_voxel"], VOXEL["map_max_points"],
                                            MAX_DISTANCE)
                return h.window_map(seqs[s], [r.T for r in rs], j, MAP_FRAMES)
            same, worst, _ = h.replay(ctx, lambda r: params(r.search_radius), src, res, target, CELL)
            return bool(same and worst < 1e-8)

        for name in args.workloads.split(","):
            seqs, T0, _, T_true = h.parking_sequences(WORKLOADS[name], n_scan=20_000, max_range=20.0)
            seqs = [list(frames) for frames in seqs]
            # the true increments, not the scene's perturbed ones
            deltas = np.concatenate([[np.linalg.inv(Tt[i]) @ Tt[min(i + 1, len(Tt) - 1)] for i in range(len(Tt))]
                                     for Tt in h.per_sequence(seqs, T_true)])
            n_frames, n_reg = len(T_true), len(T_true) - len(seqs)
            first = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
            kiss = AdaptiveThreshold(2.0, 0.1, 100.0)
            arms = {}
            for cv in (False, True):
                tag = "_cv" if cv else "_true"
                arms["fixed05" + tag] = lambda cv=cv: call(seqs, T0, deltas, 0.5, None, cv)
                arms["ceiling" + tag] = lambda cv=cv: call(seqs, T0, deltas, CEILING, None, cv)
                arms["adaptive" + tag] = lambda cv=cv: call(seqs, T0, deltas, CEILING, kiss, cv)
            arms["pinned05_true"] = lambda: call(seqs, T0, deltas, 0.5, AdaptiveThreshold(0.5, 0.5, 100.0), False)
            warm, repeats = {}, []

            def check(a, out):                          # the warm-up's outputs are reported; every round repeats them
                if a in warm:
                    repeats.append(all(h.same_bytes(x, y) for x, y in zip(out, warm[a])))
                else:
                    warm[a] = out
            outs, _, med = h.run_arms(ctx, arms, args.runs, DcregError, check)
            res = {a: warm.get(a, o) for a, o in outs.items()}
            ok_all &= all(repeats)
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
                            short = call([seqs[s][:j]], T0[s:s + 1], deltas[first[s]:first[s] + j], radius, thr, cv)
                            dt, _ = h.pose_errors(T_true[first[s]:first[s] + j], [r.T for r in short])
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
                dt, dr = h.pose_errors(T_true, [r.T for r in res[a]])
                rad = np.array([r.search_radius for r in res[a] if r.search_radius > 0.0])
                rec = {"frames_per_s": round(n_frames / (med[a] * 1e-3), 1),
                       "mean_iterations": round(sum(r.iterations for r in res[a]) / n_reg, 2),
                       "converged": int(sum(r.converged for r in res[a])),
                       "max_trans_err_m": round(dt, 4), "max_rot_err_deg": round(dr, 4),
                       "radius_min_med_max": [round(float(x), 4) for x in (rad.min(), np.median(rad), rad.max())]}
                if a.startswith("adaptive"):
                    rec["reconstruction"] = reconstructed(seqs, res[a])
                    ok_all &= rec["reconstruction"]
                out["arms"][a] = rec
                dumps.update(h.result_dumps(f"{name}_{a}", res[a], ("T",)))
                dumps[f"{name}_{a}_radius"] = [r.search_radius for r in res[a]]
            if "pinned05_true" in med and "fixed05_true" in med:
                same = all(h.same_bytes(x, y) for x, y in zip(res["pinned05_true"], res["fixed05_true"]))
                out["pinned_equals_fixed"] = bool(same)
                ok_all &= same
                out["pinned_overhead_pct"] = round(100.0 * (med["pinned05_true"] / med["fixed05_true"] - 1.0), 2)
            line["workloads"][name] = out
    line["parity"] = bool(ok_all)
    h.finish(args, line, dumps, ok_all, 1)


if __name__ == "__main__":
    main()
