"""Accelerometer input for scan-to-map odometry (dcreg_icp_run_odometry_imu): what it costs and what it changes.

Workloads: make_parking_imu_accel(n, n_scan = 20 000, max_range = 20 m, 200 Hz IMU, 10 Hz sweeps; a speed that varies
by +-30 %, a 5 cm lateral and vertical shake at 3 and 3.9 Hz, a yaw wobble), "1x128" (one sequence of 128 frames, seed
73, about 0.3 m a frame) and "8x32" (eight sequences of 32 frames, seeds 81..88, about 1.3 m a frame), every sequence
anchored at its first true pose, every point measured at its own time.  Each workload runs three ways: the window of 10
frames, the voxel map (map_voxel 0.25, max_distance 30 m), and the window call localising in the scene's prior map
(dcreg_set_prior_map(1), first frames registered from their true pose).  Cell 0.5, radius 0.5, 30 iterations, ROT
1e-5 / TRANS 1e-3, method Ours.

Arms:
  cv            constant-velocity deskew and prior (the deskew call)
  gyro          gyro input, exact rates (the constant-velocity translation)
  imu_exact     accelerometer input, exact samples, v_init the true velocity
  imu_exact_v0  the same with v_init = 0
  imu_noisy     samples with seeded white noise (GYRO_NOISE rad/s, ACCEL_NOISE m/s^2) and constant biases left unmodelled
  imu_bias      the same samples with the biases passed in
Reported per arm: frames/s (median of --runs rounds of the arms in turn after a warm-up), the prior's translation error
against the true pose over the registered frames (median, max), the drift (the translation error of T_out) at every
sequence's end and at its worst, and the first frame that loses the track (error over 1 m).  Parity (the tool exits
non-zero if it fails): every registered frame of imu_exact on the window equals set_target(its window of deskewed frames)
+ set_source(its deskewed points) + icp_run(T_prior), and repeated runs give the same bytes.  Prints one JSON line with
the card name and power limit; --dump-outputs DIR writes every arm's poses and velocities as float64 .npy files."""
import numpy as np

import bench_harness as h

MAP_FRAMES = 10
CELL = 0.5
MV, DIST = 0.25, 30.0
GYRO_NOISE, ACCEL_NOISE = 0.01, 0.05
GYRO_BIAS, ACCEL_BIAS = (0.01, -0.01, 0.02), (0.1, -0.1, 0.05)
LOST_M = 1.0
WORKLOADS = {"1x128": [(128, 73)], "8x32": [(32, 81 + i) for i in range(8)]}
MAPS = ("window", "voxel_map", "prior_map")


def scene(spec, noisy=False):
    """The sequences of spec: (skewed frames, timestamps, frame_times, samples per sequence, T0, v0, T_true)"""
    from dcreg_b200.scenes import make_parking_imu_accel
    kw = dict(gyro_noise=GYRO_NOISE, accel_noise=ACCEL_NOISE, gyro_bias=GYRO_BIAS, accel_bias=ACCEL_BIAS) if noisy else {}
    out = [make_parking_imu_accel(n, seed=seed, n_scan=20_000, max_range=20.0, **kw) for n, seed in spec]
    return ([list(o[0]) for o in out], [list(o[1]) for o in out], np.concatenate([o[2] for o in out]),
            [o[3] for o in out], np.array([o[4][0] for o in out]), np.array([o[5][0] for o in out]),
            np.concatenate([o[4] for o in out]))


def accuracy(seqs, T_true, res):
    """Prior translation error over the registered frames (median, max), drift at the ends and at its worst, and
    {sequence: first frame whose translation error exceeds LOST_M}"""
    prior, end, lost = [], [], {}
    worst = 0.0
    for s, (Tt, rs) in enumerate(zip(h.per_sequence(seqs, T_true), h.per_sequence(seqs, res))):
        err = [float(np.linalg.norm(A[:3, 3] - r.T[:3, 3])) for A, r in zip(Tt, rs)]
        prior += [float(np.linalg.norm(A[:3, 3] - r.T_prior[:3, 3])) for A, r in zip(Tt[1:], rs[1:])]
        end.append(err[-1])
        worst = max(worst, max(err))
        bad = [j for j, e in enumerate(err) if e > LOST_M]
        if bad:
            lost[str(s)] = bad[0]
    return {"prior_err_median_m": float(np.median(prior)), "prior_err_max_m": max(prior), "drift_end_m": max(end),
            "drift_worst_m": worst, "lost_at_frame": lost}


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    ap.add_argument("--maps", default=",".join(MAPS), help="comma-separated subset of " + ",".join(MAPS))
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import DcregError, Gyro, Imu
    from dcreg_b200.scenes import _parking_map

    prm = h.c3_params()
    line = {"metric": "frames_per_s", "map_frames": MAP_FRAMES, "cell": CELL, "gyro_noise_rad_s": GYRO_NOISE,
            "accel_noise_m_s2": ACCEL_NOISE, "gyro_bias_rad_s": GYRO_BIAS, "accel_bias_m_s2": ACCEL_BIAS,
            "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:
        prior_target = False

        def call(which, seqs, stamps, T0, deskewed=False, **kw):
            common = dict(motion="constant_velocity", cell_size=CELL, timestamps=stamps, want_deskewed=deskewed, **kw)
            ctx.set_prior_map(which == "prior_map")
            try:
                if which == "voxel_map":
                    return ctx.icp_run_odometry_map(prm, seqs, T0, None, map_voxel=MV, max_distance=DIST, **common)
                return ctx.icp_run_odometry(prm, seqs, T0, None, map_frames=MAP_FRAMES, **common)
            finally:
                ctx.set_prior_map(False)

        for name in args.workloads.split(","):
            seqs, stamps, ft, exact, T0, v0, T_true = scene(WORKLOADS[name])
            noisy = scene(WORKLOADS[name], noisy=True)[3]
            n_frames = len(T_true)
            for which in args.maps.split(","):
                if which == "prior_map" and not prior_target:
                    ctx.set_target(_parking_map(np.random.default_rng(43), 500_000, 60.0), CELL)
                    prior_target = True

                def imu(smp, settings, v=v0, desk=False):
                    return call(which, seqs, stamps, T0, desk, imu=settings, frame_times=ft, imu_samples=smp, v_init=v,
                                want_velocity=True)
                arms = {"cv": lambda: call(which, seqs, stamps, T0),
                        "gyro": lambda: call(which, seqs, stamps, T0, gyro=Gyro(), frame_times=ft,
                                             gyro_samples=[s[:, :4] for s in exact]),
                        "imu_exact": lambda: imu(exact, Imu()),
                        "imu_exact_v0": lambda: imu(exact, Imu(), np.zeros_like(v0)),
                        "imu_noisy": lambda: imu(noisy, Imu()),
                        "imu_bias": lambda: imu(noisy, Imu(None, GYRO_BIAS, ACCEL_BIAS))}
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
                    rec = h.rate(n_frames, med[a], runs_ms[a])
                    rec.update(accuracy(seqs, T_true, res[a]))
                    out["arms"][a] = rec
                    dumps.update(h.result_dumps(f"{name}_{which}_{a}", res[a], ("T",)))
                    if a.startswith("imu"):
                        dumps[f"{name}_{which}_{a}_velocity"] = [r.velocity for r in res[a]]
                if which == "window" and not isinstance(res["imu_exact"], str):
                    desk = imu(exact, Imu(), desk=True)
                    src = [[r.deskewed for r in rs] for rs in h.per_sequence(seqs, desk)]
                    same, worst, _ = h.replay(ctx, prm, src, desk,
                                              lambda s, j, rs, M: h.window_map(src[s], [r.T for r in rs], j, MAP_FRAMES),
                                              CELL)
                    out["replay_imu_exact"] = bool(same and worst < 1e-8
                                                   and all(h.same_bytes(x, y) for x, y in zip(desk, res["imu_exact"])))
                    ok_all &= out["replay_imu_exact"]
                line["workloads"][f"{name}_{which}"] = out
    line["parity"] = bool(ok_all)
    h.finish(args, line, dumps, ok_all, 1)


if __name__ == "__main__":
    main()
