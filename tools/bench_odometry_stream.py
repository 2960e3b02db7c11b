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
import time

import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
WORKLOADS = {
    "1x256": dict(spec=[(256, 47)], n_scan=20_000, n_map=500_000, filters={}),
    "8x64": dict(spec=[(64, 71 + i) for i in range(8)], n_scan=20_000, n_map=500_000, filters={}),
    "1x128v": dict(spec=[(128, 47)], n_scan=100_000, n_map=2_000_000,
                   filters=dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)),
}


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import compose_prior
    prm = h.c3_params()
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        for name in args.workloads.split(","):
            wl = WORKLOADS[name]
            filt = wl["filters"]
            seqs, T0, D_all, T_true = h.parking_sequences(wl["spec"], n_map=wl["n_map"], n_scan=wl["n_scan"],
                                                          max_range=20.0)
            deltas = h.per_sequence(seqs, D_all)
            first = np.concatenate([[0], np.cumsum([len(f) for f in seqs])])
            n_frames, S, L = len(D_all), len(seqs), max(len(f) for f in seqs)

            def one_call():
                return ctx.icp_run_odometry(prm, seqs, T0, D_all, map_frames=MAP_FRAMES, cell_size=CELL, **filt)

            lats = []                                                           # every session's push latencies

            def session():
                out = [[] for _ in seqs]
                lats.append([])
                with ctx.odometry_session(prm, S, T0, map_frames=MAP_FRAMES, cell_size=CELL, **filt) as sess:
                    for k in range(L):
                        part = [[f[k]] if k < len(f) else [] for f in seqs]
                        D = np.stack([deltas[s][k] for s in range(S) if k < len(seqs[s])])
                        w = time.perf_counter()
                        res = sess.push(part, D)
                        lats[-1].append((time.perf_counter() - w) * 1e3)
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
                        m = h.window_map(src, Ts, j, MAP_FRAMES)
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
            outs, ms, med = h.run_arms(ctx, arms, args.runs)
            lat = [t for x in lats[1:] for t in x]                              # the timed rounds' pushes
            # parity: the session against the call, byte for byte
            sess_res, call_res = outs["session"], outs["call"]
            by_frame = [None] * n_frames                                        # the session's results in call order
            k = 0
            for s in range(S):
                for j in range(len(seqs[s])):
                    by_frame[first[s] + j] = sess_res[k]
                    k += 1
            ok = len(sess_res) == n_frames and all(h.same_bytes(a, b) for a, b in zip(by_frame, call_res))
            ok_all = ok_all and ok
            reg = [r for r in call_res if r.iterations > 0]
            w = {"sequences": S, "frames": n_frames, "filters": filt,
                 "points_per_frame_mean": float(np.mean([r.n_points for r in call_res])),
                 "mean_iterations": float(np.mean([r.iterations for r in reg])),
                 "parity": {"session_equals_call_bytes": ok}}
            for a in arms:
                w[a] = h.rate(n_frames, med[a], ms[a])
            w["session"]["push_latency_ms"] = {"p50": float(np.percentile(lat, 50)), "p90": float(np.percentile(lat, 90)),
                                               "max": float(np.max(lat)), "pushes": len(lat)}
            drift_a = h.pose_errors(T_true, [r.T for r in by_frame])
            drift_d = h.pose_errors(T_true, outs["per_frame"])
            w["session"]["max_err_vs_truth"] = {"trans_m": drift_a[0], "rot_deg": drift_a[1]}
            w["per_frame"]["max_err_vs_truth"] = {"trans_m": drift_d[0], "rot_deg": drift_d[1]}
            line["workloads"][name] = w
            dumps.update(h.result_dumps(f"odometry_stream_{name}", by_frame, h.FIELDS + ("n_points",)))
    bad = [n for n, w in line["workloads"].items() if not w["parity"]["session_equals_call_bytes"]]
    h.finish(args, line, dumps, ok_all, f"bench_odometry_stream.py: the session's outputs differ from the call's in {bad}")


if __name__ == "__main__":
    main()
