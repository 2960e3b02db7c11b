"""Streaming scan-to-map odometry: the odometry session (dcreg_odometry_open / _push) fed as frames arrive, against the
one-shot call and the two ways a user streams without a session.

Arms, on the same frames:
  (a) session   Context.odometry_session, one frame per sequence per push; every push ends in a host sync (its results
                come back), so its wall-clock time is the latency a robot sees for a new frame: p50 / p90 / max over the
                pushes of the timed runs
  (b) call      one icp_run_odometry call over the whole recording (offline)
  (c) loop      the per-frame host loop: the local map from the loop's own results with map_points, then set_target +
                set_source + icp_run from compose_prior of the previous result (filtered workload: the frame and the map
                through Context.voxel_downsample first)
  (d) per_frame today's streaming workaround: one icp_run_odometry call per new frame with the previous frame as its
                anchor, at the pose the previous call returned, so every frame registers against a one-frame map

Workloads as tools/bench_odometry.py: make_parking_sequence(n, n_scan = 20 000, max_range = 20 m), "1x256" (one
sequence of 256 frames, seed 47) and "8x64" (eight sequences of 64 frames, seeds 71..78); and one filtered workload
as tools/sweep_odometry_voxel.py: "1x128v" (n_map = 2 000 000, n_scan = 100 000: about 94 k points a frame, seed 47)
with source voxel 0.25 and map voxel 0.25 keeping 4 points per voxel.  Every sequence is anchored at its first true
pose.  map_frames 10, radius and cell 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours, motion "increments".
Timing: host arrays in, results out, the max of CUDA events on the context's stream and the host wall clock, after a
warm-up of every arm; --runs rounds of the arms in turn, medians reported.

Parity (asserted; the tool exits non-zero if it fails): every frame of (a) equals (b) byte for byte (T, T_prior,
status, iterations, converged, n_points).  Reported: frames/s per arm, and the drift against the true poses of (a) and
(d).  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes (a)'s outputs as float64
.npy files."""
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
WORKLOADS = {
    "1x256": dict(spec=[(256, 47)], n_scan=20_000, n_map=500_000, filters={}),
    "8x64": dict(spec=[(64, 71 + i) for i in range(8)], n_scan=20_000, n_map=500_000, filters={}),
    "1x128v": dict(spec=[(128, 47)], n_scan=100_000, n_map=2_000_000,
                   filters=dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)),
}


def same_bytes(a, b):
    return ((a.status, a.iterations, a.converged, a.n_points) == (b.status, b.iterations, b.converged, b.n_points)
            and a.T.tobytes() == b.T.tobytes() and a.T_prior.tobytes() == b.T_prior.tobytes())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    args = ap.parse_args()
    import torch
    from dcreg_b200 import Context, default_params
    from dcreg_b200.api import compose_prior, map_points
    from dcreg_b200.scenes import make_parking_sequence
    if not torch.cuda.is_available():
        raise SystemExit("bench_odometry_stream.py: no CUDA device - dcreg_b200 has no CPU fallback")
    prm = default_params(max_iterations=30, search_radius=0.5, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
                         kappa_target=10.0, detection="SCHUR_CONDITION_NUMBER", handling="PRECONDITIONED_CG")
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "workloads": {}, "card": card()}
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

        for name in args.workloads.split(","):
            wl = WORKLOADS[name]
            filt = wl["filters"]
            seqs, T0, deltas, T_true = [], [], [], []
            for n, seed in wl["spec"]:
                frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, n_map=wl["n_map"], n_scan=wl["n_scan"],
                                                            max_range=20.0)
                seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
            T0, T_true = np.array(T0), np.concatenate(T_true)
            first = np.concatenate([[0], np.cumsum([len(f) for f in seqs])])
            D_all = np.concatenate(deltas)
            n_frames, S, L = len(D_all), len(seqs), max(len(f) for f in seqs)

            def one_call():
                return ctx.icp_run_odometry(prm, seqs, T0, D_all, map_frames=MAP_FRAMES, cell_size=CELL, **filt)

            def session(lat=None):
                out = [[] for _ in seqs]
                with ctx.odometry_session(prm, S, T0, map_frames=MAP_FRAMES, cell_size=CELL, **filt) as sess:
                    for k in range(L):
                        part = [[f[k]] if k < len(f) else [] for f in seqs]
                        D = np.stack([deltas[s][k] for s in range(S) if k < len(seqs[s])])
                        w = time.perf_counter()
                        res = sess.push(part, D)
                        if lat is not None:
                            lat.append((time.perf_counter() - w) * 1e3)
                        for s, r in enumerate(res):
                            out[s].extend(r)
                return [r for rs in out for r in rs]

            def host_loop():
                out = []
                for s, frames in enumerate(seqs):
                    src = [f if not filt else ctx.voxel_downsample([f], filt["source_voxel"])[0][0] for f in frames]
                    Ts = [T0[s]]
                    for j in range(1, len(frames)):
                        T = compose_prior(Ts[j - 1], deltas[s][j - 1])
                        m = np.concatenate([map_points(Ts[i], src[i]) for i in range(max(0, j - MAP_FRAMES), j)])
                        if filt:
                            m = ctx.voxel_downsample([m], filt["map_voxel"], filt["map_max_points"])[0][0]
                        ctx.set_target(m, CELL)
                        ctx.set_source(src[j])
                        r = ctx.icp_run(prm, T, want_log=False)
                        out.append(r)
                        Ts.append(r.T)
                return out

            def per_frame_calls():
                Ts = [[T0[s]] for s in range(S)]
                for k in range(1, L):
                    live = [s for s in range(S) if k < len(seqs[s])]
                    res = ctx.icp_run_odometry(prm, [[seqs[s][k - 1], seqs[s][k]] for s in live],
                                               np.stack([Ts[s][-1] for s in live]),
                                               np.concatenate([[deltas[s][k - 1], np.eye(4)] for s in live]),
                                               map_frames=MAP_FRAMES, cell_size=CELL, **filt)
                    for i, s in enumerate(live):
                        Ts[s].append(res[2 * i + 1].T)
                return [T for s in range(S) for T in Ts[s]]

            arms = {"session": session, "call": one_call, "loop": host_loop, "per_frame": per_frame_calls}
            for fn in arms.values():                                            # warm-up of every arm
                fn()
            ms = {a: [] for a in arms}
            lat = []
            outs = {}
            for _ in range(max(1, args.runs)):
                for a, fn in arms.items():
                    outs[a], t = timed((lambda: session(lat)) if a == "session" else fn)
                    ms[a].append(t)
            # parity: the session against the call, byte for byte
            sess_res, call_res = outs["session"], outs["call"]
            by_frame = [None] * n_frames                                        # the session's results in call order
            k = 0
            for s in range(S):
                for j in range(len(seqs[s])):
                    by_frame[first[s] + j] = sess_res[k]
                    k += 1
            ok = len(sess_res) == n_frames and all(same_bytes(a, b) for a, b in zip(by_frame, call_res))
            ok_all = ok_all and ok
            reg = [r for r in call_res if r.iterations > 0]
            w = {"sequences": S, "frames": n_frames, "filters": filt,
                 "points_per_frame_mean": float(np.mean([r.n_points for r in call_res])),
                 "mean_iterations": float(np.mean([r.iterations for r in reg])),
                 "parity": {"session_equals_call_bytes": ok}}
            for a in arms:
                m = float(np.median(ms[a]))
                w[a] = {"frames_per_s": n_frames / (m * 1e-3), "ms": m, "runs_ms": ms[a]}
            w["session"]["push_latency_ms"] = {"p50": float(np.percentile(lat, 50)), "p90": float(np.percentile(lat, 90)),
                                               "max": float(np.max(lat)), "pushes": len(lat)}
            drift_a = pose_errors(T_true, [r.T for r in by_frame])
            drift_d = pose_errors(T_true, outs["per_frame"])
            w["session"]["max_err_vs_truth"] = {"trans_m": drift_a[0], "rot_deg": drift_a[1]}
            w["per_frame"]["max_err_vs_truth"] = {"trans_m": drift_d[0], "rot_deg": drift_d[1]}
            line["workloads"][name] = w
            dumps[name] = by_frame
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for name, res in dumps.items():
            for k, v in {"T": [r.T for r in res], "T_prior": [r.T_prior for r in res],
                         "iterations": [r.iterations for r in res], "converged": [r.converged for r in res],
                         "status": [r.status for r in res], "n_points": [r.n_points for r in res]}.items():
                np.save(os.path.join(args.dump_outputs, f"odometry_stream_{name}_{k}.npy"), np.asarray(v, dtype=np.float64))
    if not ok_all:
        bad = [n for n, w in line["workloads"].items() if not w["parity"]["session_equals_call_bytes"]]
        raise SystemExit(f"bench_odometry_stream.py: the session's outputs differ from the call's in {bad}")


if __name__ == "__main__":
    main()
