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
from bench_sequences import pose_errors  # noqa: E402

MAP_FRAMES = 10
CELL = 0.5


def map_sizes(seqs_sizes):
    """Map points of every step over the sequences, from the frames' point counts (unfiltered maps)"""
    out = []
    for i in range(1, max(len(f) for f in seqs_sizes)):
        out.append(sum(sum(f[j] for j in range(max(0, i - MAP_FRAMES), i)) for f in seqs_sizes if len(f) > i))
    return out


def dump_results(path, prefix, runs):
    """runs: {name: [OdometryResult]} -> PATH/PREFIX_NAME_{T,T_prior,iterations,converged,status,n_points}.npy"""
    os.makedirs(path, exist_ok=True)
    for name, res in runs.items():
        for k in ("T", "T_prior", "iterations", "converged", "status", "n_points"):
            np.save(os.path.join(path, f"{prefix}_{name}_{k}.npy"), np.asarray([getattr(r, k) for r in res], np.float64))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--source-voxel", type=float, default=0.25)
    ap.add_argument("--map-voxel", type=float, default=0.25)
    ap.add_argument("--small", action="store_true", help="a quick rehearsal: 2 small workloads")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    import dcreg_oracle as o
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import map_points, voxel_downsample
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_odometry_voxel.py: no CUDA device - dcreg_b200 has no CPU fallback")
    sv, mv = args.source_voxel, args.map_voxel
    prm = default_params(max_iterations=30, search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    if args.small:
        workloads = {"1x8": [(8, 47)], "2x4": [(4, 71), (4, 72)]}
        n_map, n_scan, n_clouds = 200_000, 10_000, 4
    else:
        workloads = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}
        n_map, n_scan, n_clouds = 2_000_000, 100_000, 64
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "source_voxel": sv, "map_voxel": mv,
            "n_scan": n_scan, "n_map": n_map, "workloads": {}, "card": card()}
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
            w = time.perf_counter() - w
            return out, max(e0.elapsed_time(e1), w * 1e3)

        for name, spec in workloads.items():
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in spec:
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_map=n_map, n_scan=n_scan, max_range=20.0)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, deltas, T_true = np.array(T0), np.concatenate(deltas), np.concatenate(T_true)
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
            for fn in arms.values():                                           # warm-up
                fn()
            ms = {a: [] for a in arms}
            res = {}
            for _ in range(max(1, args.runs)):
                for a, fn in arms.items():
                    res[a], t = timed(fn)
                    ms[a].append(t)
            # parity of the device arm, and its filtered map sizes
            same, worst, k, dev_maps = True, 0.0, 0, {}
            for s, frames in enumerate(seqs):
                rs = res["device"][k:k + len(frames)]
                filt = [voxel_downsample(f, sv)[0] for f in frames]
                for j in range(1, len(frames)):
                    M = np.concatenate([map_points(rs[w].T, filt[w]) for w in range(max(0, j - MAP_FRAMES), j)])
                    M = voxel_downsample(M, mv)[0]
                    dev_maps[j] = dev_maps.get(j, 0) + len(M)
                    ctx.set_target(M, CELL)
                    ctx.set_source(filt[j])
                    single = ctx.icp_run(prm, rs[j].T_prior, want_log=False)
                    b = rs[j]
                    same = same and (b.status, b.iterations, b.converged) == (single.status, single.iterations,
                                                                               single.converged)
                    worst = max(worst, float(o.se3_log_distance(single.T, b.T)))
                    same = same and b.n_points == len(filt[j])
                k += len(frames)
            ok = same and worst <= 1e-8
            ok_all = ok_all and ok

            def sizes(rs):
                out, k = [], 0
                for s in seqs:
                    out.append([r.n_points for r in rs[k:k + len(s)]])
                    k += len(s)
                return out
            maps = {"raw": map_sizes(sizes(res["raw"])), "host": map_sizes(sizes(res["host"])),
                    "device": [dev_maps[j] for j in sorted(dev_maps)]}
            w = {"sequences": len(seqs), "frames": n_frames,
                 "parity": {"ok": ok, "identical_status_iterations_converged_points": same, "max_pose_err": worst,
                            "tolerance": 1e-8}}
            for a in arms:
                m = float(np.median(ms[a]))
                reg = [r for r in res[a] if r.iterations > 0]
                pts = [r.n_points for r in res[a]]
                drift = pose_errors(T_true, [r.T for r in res[a]])
                w[a] = {"frames_per_s": n_frames / (m * 1e-3), "ms": m, "runs_ms": ms[a],
                        "mean_iterations": float(np.mean([r.iterations for r in reg])),
                        "converged": int(sum(r.converged for r in reg)), "registered": len(reg),
                        "points_per_frame_mean": float(np.mean(pts)),
                        "map_points_per_step": {"mean": float(np.mean(maps[a])), "max": int(max(maps[a]))},
                        "max_err_vs_truth": {"trans_m": drift[0], "rot_deg": drift[1]}}
            line["workloads"][name] = w
            dumps.update({f"{name}_{a}": res[a] for a in arms})
        # the standalone filter: one device call over n_clouds clouds against the twin on each
        frames, _, _, _, _ = make_parking_sequence(n_clouds, seed=90, n_map=n_map, n_scan=n_scan, max_range=20.0)
        clouds = [f[:n_scan] for f in frames]
        n_pts = sum(len(c) for c in clouds)
        ctx.voxel_downsample(clouds, sv)
        dev_ms, twin_ms = [], []
        for _ in range(max(1, args.runs)):
            got, t = timed(lambda: ctx.voxel_downsample(clouds, sv))
            dev_ms.append(t)
            t0 = time.perf_counter()
            twin = [voxel_downsample(c, sv) for c in clouds]
            twin_ms.append((time.perf_counter() - t0) * 1e3)
        equal = all(p.tobytes() == tp.tobytes() and np.array_equal(i, ti) for (p, i), (tp, ti) in zip(got, twin))
        ok_all = ok_all and equal
        dm, tm = float(np.median(dev_ms)), float(np.median(twin_ms))
        line["filter"] = {"clouds": len(clouds), "points": n_pts, "voxel": sv, "kept": int(sum(len(i) for _, i in got)),
                          "device_ms": dm, "device_points_per_s": n_pts / (dm * 1e-3), "device_runs_ms": dev_ms,
                          "twin_ms": tm, "twin_points_per_s": n_pts / (tm * 1e-3), "twin_runs_ms": twin_ms,
                          "equal_to_twin": equal}
    print(json.dumps(line))
    if args.dump_outputs:
        dump_results(args.dump_outputs, "odometry_voxel", dumps)
        for c, (p, i) in enumerate(got):
            np.save(os.path.join(args.dump_outputs, f"voxel_filter_{c}_xyz.npy"), np.asarray(p, np.float64))
            np.save(os.path.join(args.dump_outputs, f"voxel_filter_{c}_index.npy"), np.asarray(i, np.float64))
    if not ok_all:
        raise SystemExit("bench_odometry_voxel.py: parity FAILED")


if __name__ == "__main__":
    main()
