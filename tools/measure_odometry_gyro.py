"""Gyroscope input for scan-to-map odometry (dcreg_icp_run_odometry_gyro): what it costs and what it changes.

Workloads: make_parking_imu(n, n_scan = 20 000, max_range = 20 m, 200 Hz gyro, 10 Hz sweeps), "1x128" (one sequence of
128 frames, seed 47) and "8x32" (eight sequences of 32 frames, seeds 71..78), every sequence anchored at its first true
pose, every frame skewed by the sensor's motion during its sweep.  Window of 10 frames, cell 0.5, radius 0.5, 30
iterations, ROT 1e-5 / TRANS 1e-3, method Ours, the constant-velocity model's translation.

Arms:
  cv          constant-velocity deskew and prior (dcreg_icp_run_odometry_deskew, the call before gyro input)
  gyro_exact  gyro with the exact body rates
  gyro_noisy  gyro with seeded white noise (NOISE rad/s per sample) and a constant bias (BIAS rad/s) left unmodelled
  gyro_bias   the same samples with that bias passed in
Reported per arm: frames/s (median of --runs rounds of the arms in turn after a warm-up; CUDA events on the context's
stream and the host clock, the larger), mean iterations per registered frame, converged frames, the largest translation
and rotation error against the true poses, and, per sequence that loses the track, the first frame whose translation
error exceeds 1 m (or the call's error message).  Parity (the tool exits non-zero if it fails): every registered frame of
gyro_exact equals set_target(its window of deskewed frames) + set_source(its deskewed points) + icp_run(T_prior), and
repeated runs give the same bytes.  Prints one JSON line with the card name and power limit; --dump-outputs DIR writes
every arm's poses as float64 .npy files."""
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
NOISE = 0.01
BIAS = (0.01, -0.01, 0.02)
LOST_M = 1.0
WORKLOADS = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)]}


def scene(spec, noise=0.0, bias=(0.0, 0.0, 0.0)):
    """The sequences of spec: (skewed frames, timestamps, frame_times, samples per sequence, T0, T_true)"""
    from dcreg_b200.scenes import make_parking_imu
    out = [make_parking_imu(n, noise=noise, bias=bias, seed=seed, n_scan=20_000, max_range=20.0) for n, seed in spec]
    return ([list(o[0]) for o in out], [list(o[1]) for o in out], np.concatenate([o[2] for o in out]),
            [o[3] for o in out], np.array([o[4][0] for o in out]), np.concatenate([o[4] for o in out]))


def lost_at(seqs, T_true, res):
    """{sequence: first frame whose translation error exceeds LOST_M} over the sequences that lose the track"""
    out = {}
    for s, (Tt, rs) in enumerate(zip(h.per_sequence(seqs, T_true), h.per_sequence(seqs, res))):
        bad = [j for j, (A, r) in enumerate(zip(Tt, rs)) if np.linalg.norm(A[:3, 3] - r.T[:3, 3]) > LOST_M]
        if bad:
            out[str(s)] = bad[0]
    return out


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import DcregError, Gyro

    prm = h.c3_params()
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "cell": CELL, "noise_rad_s": NOISE, "bias_rad_s": BIAS,
            "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:

        def call(seqs, stamps, T0, ft=None, smp=None, gyro=None, deskewed=False):
            kw = dict(gyro=gyro, frame_times=ft, gyro_samples=smp) if gyro is not None else {}
            return ctx.icp_run_odometry(prm, seqs, T0, None, motion="constant_velocity", map_frames=MAP_FRAMES,
                                        cell_size=CELL, timestamps=stamps, want_deskewed=deskewed, **kw)

        for name in args.workloads.split(","):
            seqs, stamps, ft, exact, T0, T_true = scene(WORKLOADS[name])
            noisy = scene(WORKLOADS[name], NOISE, BIAS)[3]
            n_frames = len(T_true)
            arms = {"cv": lambda: call(seqs, stamps, T0),
                    "gyro_exact": lambda: call(seqs, stamps, T0, ft, exact, Gyro()),
                    "gyro_noisy": lambda: call(seqs, stamps, T0, ft, noisy, Gyro()),
                    "gyro_bias": lambda: call(seqs, stamps, T0, ft, noisy, Gyro(None, BIAS))}
            warm, repeats = {}, []

            def check(a, out):
                if a in warm:
                    repeats.append(all(h.same_bytes(x, y) for x, y in zip(out, warm[a])))
                else:
                    warm[a] = out
            outs, runs_ms, med = h.run_arms(ctx, arms, args.runs, DcregError, check)
            res = {a: warm.get(a, o) for a, o in outs.items()}
            ok_all &= all(repeats)
            out = {"frames": n_frames, "arms": {}}
            for a in arms:
                if isinstance(res[a], str):
                    out["arms"][a] = {"error": res[a]}
                    continue
                rec = h.arm_block(n_frames, med[a], runs_ms[a], res[a], T_true)
                rec["lost_at_frame"] = lost_at(seqs, T_true, res[a])
                out["arms"][a] = rec
                dumps.update(h.result_dumps(f"{name}_{a}", res[a], ("T",)))
            if not isinstance(res["gyro_exact"], str):
                desk = call(seqs, stamps, T0, ft, exact, Gyro(), deskewed=True)
                src = [[r.deskewed for r in rs] for rs in h.per_sequence(seqs, desk)]
                same, worst, _ = h.replay(ctx, prm, src, desk,
                                          lambda s, j, rs, M: h.window_map(src[s], [r.T for r in rs], j, MAP_FRAMES), CELL)
                out["replay_gyro_exact"] = bool(same and worst < 1e-8
                                                and all(h.same_bytes(x, y) for x, y in zip(desk, res["gyro_exact"])))
                ok_all &= out["replay_gyro_exact"]
            line["workloads"][name] = out
    line["parity"] = bool(ok_all)
    h.finish(args, line, dumps, ok_all, 1)


if __name__ == "__main__":
    main()
