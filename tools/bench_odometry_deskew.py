"""Motion compensation inside scan-to-map odometry (dcreg_icp_run_odometry_deskew) on skewed LiDAR sweeps.

Workloads: make_parking_sweeps(n, n_scan = 20 000, max_range = 20 m), "1x128" (one sequence of 128 frames, seed 47)
and "8x32" (eight sequences of 32 frames, seeds 71..78), and the filtered "1x128v" (n_map = 2 000 000, n_scan =
100 000: about 94 k points a frame, seed 47) with source voxel 0.25 and map voxel 0.25 keeping 4 points per voxel.
Every sequence is anchored at its first true pose with its first frame unskewed (an anchor is never deskewed).
map_frames 10, radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours.

Arms, on the same frames:
  skewed       the skewed sweeps, no timestamps, the true increments as deltas
  deskew_cv    the skewed sweeps with their timestamps, constant velocity: the increment is the previous two results'
  deskew_true  the skewed sweeps with their timestamps, the true increments as deltas
  unskewed     the unskewed frames, the true increments as deltas: the bound deskewing can reach
  mid          the unskewed frames with every tau = 0.5, the true increments: the same bytes as `unskewed`, so its time
               against `unskewed` is the deskew path's own cost (mid_overhead_pct)
An arm whose odometry fails (a local map too large for a dense grid once the registration has diverged) is reported
with its error message instead of numbers.
Reported per arm: frames/s (median over --runs rounds of the arms in turn, after a warm-up; CUDA events on the context's
stream and the host clock, the larger), iterations, converged frames, and the largest translation / rotation error
against the true mid-sweep poses.  Parity (asserted; the tool exits non-zero if it fails): `mid` equals `unskewed` byte
for byte, and deskew_true's deskewed points of every frame lie within one float32 ulp (or 1e-12 m) of
api.deskew_points with the true increment.  Prints one JSON line with the card name and power limit; --dump-outputs DIR
writes every arm's poses as float64 .npy files."""
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
WORKLOADS = {
    "1x128": dict(spec=[(128, 47)], n_scan=20_000, n_map=500_000, filters={}),
    "8x32": dict(spec=[(32, 71 + i) for i in range(8)], n_scan=20_000, n_map=500_000, filters={}),
    "1x128v": dict(spec=[(128, 47)], n_scan=100_000, n_map=2_000_000,
                   filters=dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)),
}
ARMS = ["skewed", "deskew_cv", "deskew_true", "unskewed", "mid"]


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import DcregError, deskew_points, voxel_downsample
    from dcreg_b200.scenes import make_parking_sweeps
    prm = h.c3_params()
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name in args.workloads.split(","):
            wl = WORKLOADS[name]
            seqs = {"skewed": [], "unskewed": [], "stamps": [], "mid": []}
            T_true, T_init, deltas = [], [], []
            for n, seed in wl["spec"]:
                sk, ts, Tt, D, un = make_parking_sweeps(n, seed=seed, n_scan=wl["n_scan"], n_map=wl["n_map"],
                                                        max_range=20.0)
                sk[0] = un[0]
                seqs["skewed"].append(sk); seqs["unskewed"].append(un); seqs["stamps"].append(ts)
                seqs["mid"].append([np.full(len(t), 0.5, np.float32) for t in ts])
                T_true.append(Tt); T_init.append(Tt[0]); deltas.append(D)
            T_true = np.concatenate(T_true)
            T_init = np.array(T_init)
            deltas = np.concatenate(deltas)
            n_frames = len(T_true)
            f = wl["filters"]
            arms = {
                "skewed": lambda: ctx.icp_run_odometry(prm, seqs["skewed"], T_init, deltas, map_frames=MAP_FRAMES,
                                                       cell_size=CELL, **f),
                "deskew_cv": lambda: ctx.icp_run_odometry(prm, seqs["skewed"], T_init, motion="constant_velocity",
                                                          map_frames=MAP_FRAMES, cell_size=CELL,
                                                          timestamps=seqs["stamps"], **f),
                "deskew_true": lambda: ctx.icp_run_odometry(prm, seqs["skewed"], T_init, deltas, map_frames=MAP_FRAMES,
                                                            cell_size=CELL, timestamps=seqs["stamps"],
                                                            want_deskewed=True, **f),
                "unskewed": lambda: ctx.icp_run_odometry(prm, seqs["unskewed"], T_init, deltas, map_frames=MAP_FRAMES,
                                                         cell_size=CELL, **f),
                "mid": lambda: ctx.icp_run_odometry(prm, seqs["unskewed"], T_init, deltas, map_frames=MAP_FRAMES,
                                                    cell_size=CELL, timestamps=seqs["mid"], **f),
            }
            warm, repeats = {}, []

            def check(a, out):                          # the warm-up's outputs are checked below; every round repeats them
                if a in warm:
                    repeats.append(all(h.same_bytes(x, y) for x, y in zip(out, warm[a])))
                else:
                    warm[a] = out
            # an arm whose odometry diverged keeps its message
            outs, _, med = h.run_arms(ctx, arms, args.runs, DcregError, check)
            res = {a: warm.get(a, o) for a, o in outs.items()}
            ok_all &= all(repeats)
            for a in ("deskew_true", "unskewed", "mid"):
                if isinstance(res[a], str):
                    raise SystemExit(f"bench_odometry_deskew.py: {name}: {a} failed: {res[a]}")
            parity = all(h.same_bytes(x, y) for x, y in zip(res["mid"], res["unskewed"]))
            k = 0
            for s, (sk, ts) in enumerate(zip(seqs["skewed"], seqs["stamps"])):
                for j in range(len(sk)):
                    r = res["deskew_true"][k + j]
                    pts, tau = sk[j], ts[j]
                    if f.get("source_voxel"):
                        pts, idx = voxel_downsample(pts, f["source_voxel"])
                        tau = tau[idx]
                    ref = pts if j == 0 else deskew_points(pts, tau, deltas[k + j - 1])
                    ulp = np.spacing(np.abs(ref)).astype(np.float64)
                    parity &= bool((np.abs(r.deskewed.astype(np.float64) - ref) <= np.maximum(ulp, 1e-12)).all())
                k += len(sk)
            ok_all &= parity
            out = {"frames": n_frames, "parity": parity, "arms": {}}
            for a in ARMS:
                if isinstance(res[a], str):
                    out["arms"][a] = {"error": res[a]}
                    continue
                dt, dr = h.pose_errors(T_true, [r.T for r in res[a]])
                out["arms"][a] = {"frames_per_s": round(n_frames / (med[a] * 1e-3), 1),
                                  "iterations": int(sum(r.iterations for r in res[a])),
                                  "converged": int(sum(r.converged for r in res[a])),
                                  "max_trans_err_m": round(dt, 4), "max_rot_err_deg": round(dr, 4)}
                dumps.update(h.result_dumps(f"{name}_{a}", res[a], ("T",)))
            out["mid_overhead_pct"] = round(100.0 * (med["mid"] / med["unskewed"] - 1.0), 2)
            line["workloads"][name] = out
    line["parity"] = bool(ok_all)
    h.finish(args, line, dumps, ok_all, 1)


if __name__ == "__main__":
    main()
