"""Localisation in a prior map through the odometry front end (dcreg_set_prior_map): what it costs and how far it drifts,
against dcreg_icp_run_sequences, today's route for a prior map.

Workloads: make_parking_imu(n, n_scan = 20 000, max_range = 20 m, 200 Hz gyro, 10 Hz sweeps), "1x128" (one sequence of
128 frames, seed 47) and "8x32" (eight sequences of 32 frames, seeds 71..78), registered against the scene's own
parking map (_parking_map with map_seed 43, 500 k points, a dense grid), every frame skewed by the sensor's motion
during its sweep.  Each sequence starts from its first true pose times the icp_pk01.yaml offsets (0.15 / 0.12 / 0.13 m,
0.015 / 1.31 / 2.17 deg, seeded signs).  "tiles": the 4 x 4 tile map of make_large_map (a sparse row index) with 128
unskewed frames of make_large_map_frames, one sequence of 8 frames per tile.  Cell 0.5, radius 0.5, 30 iterations,
ROT 1e-5 / TRANS 1e-3, method Ours.

Arms (the deskew and gyro arms on the parking workloads only):
  seq_null         dcreg_icp_run_sequences with deltas = NULL (every frame from the previous frame's result)
  seq_true         dcreg_icp_run_sequences with the true increments (the bound)
  prior_cv         the prior map, constant velocity, no deskew
  prior_cv_deskew  the prior map, constant velocity and deskew
  prior_gyro       the prior map, gyro input (exact rates) and deskew
  prior_gyro_noisy the same with seeded white noise (NOISE rad/s) and an unmodelled bias (BIAS rad/s) in the samples
  window_gyro      the window odometry (10 frames, no map) with gyro input and deskew, for reference
Reported per arm: frames/s (median of --runs rounds of the arms in turn after a warm-up), mean iterations per
registered frame, converged frames, and the largest translation and rotation error against the true poses.  Repeated
runs must give the same bytes (the tool exits non-zero otherwise).  Prints one JSON line with the card name and power
limit; --dump-outputs DIR writes every arm's poses as float64 .npy files."""
import math

import numpy as np

import bench_harness as h

CELL = 0.5
MAP_FRAMES = 10
NOISE = 0.01
BIAS = (0.01, -0.01, 0.02)
WORKLOADS = {"1x128": [(128, 47)], "8x32": [(32, 71 + i) for i in range(8)], "tiles": None}


def offsets(T, seed):
    """T times the icp_pk01.yaml offsets with seeded random signs"""
    from dcreg_b200.scenes import pose6d_to_matrix
    d = math.pi / 180.0
    mag = np.array([0.15, 0.12, 0.13, 0.015 * d, 1.31 * d, 2.17 * d])
    return T @ pose6d_to_matrix(*(mag * np.random.default_rng(seed).choice([-1.0, 1.0], 6)))


def true_deltas(T_per_seq):
    """inv(T_k) T_{k+1} inside every sequence, the identity after its last frame, in frame order"""
    out = []
    for T in T_per_seq:
        out += [np.linalg.inv(a) @ b for a, b in zip(T[:-1], T[1:])] + [np.eye(4)]
    return np.array(out)


def parking(spec, noise=0.0, bias=(0.0, 0.0, 0.0)):
    from dcreg_b200.scenes import make_parking_imu
    out = [make_parking_imu(n, noise=noise, bias=bias, seed=seed, n_scan=20_000, max_range=20.0) for n, seed in spec]
    T0 = np.array([offsets(o[4][0], seed) for o, (_, seed) in zip(out, spec)])
    return dict(seqs=[list(o[0]) for o in out], stamps=[list(o[1]) for o in out], ft=np.concatenate([o[2] for o in out]),
                samples=[o[3] for o in out], T0=T0, T_true=np.concatenate([o[4] for o in out]),
                deltas=true_deltas([o[4] for o in out]))


def tiles(n_frames=128):
    from dcreg_b200.scenes import make_large_map, make_large_map_frames
    tgt, _ = make_large_map()
    frames, T_true, T_init, tile = make_large_map_frames(n_frames)
    order = np.argsort(tile, kind="stable")
    seqs = [[frames[k] for k in order if tile[k] == t] for t in range(int(tile.max()) + 1)]
    T_seq = [T_true[order][tile[order] == t] for t in range(int(tile.max()) + 1)]
    T0 = np.array([T_init[order][tile[order] == t][0] for t in range(int(tile.max()) + 1)])
    return dict(seqs=seqs, T0=T0, T_true=T_true[order], deltas=true_deltas(T_seq), map=tgt)


def main():
    ap = h.parser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS), help="comma-separated subset of " + ",".join(WORKLOADS))
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.api import DcregError, Gyro
    from dcreg_b200.scenes import _parking_map

    prm = h.c3_params()
    line = {"metric": "frames_per_s", "cell": CELL, "window_map_frames": MAP_FRAMES, "noise_rad_s": NOISE,
            "bias_rad_s": BIAS, "workloads": {}, "card": h.card()}
    ok_all = True
    dumps = {}
    with Context(0) as ctx:

        def prior(fn):
            ctx.set_prior_map(1)
            try:
                return fn()
            finally:
                ctx.set_prior_map(0)

        def odo(d, stamps=False, samples=None, window=False):
            kw = dict(timestamps=d["stamps"] if stamps else None)
            if samples is not None:
                kw.update(gyro=Gyro(), frame_times=d["ft"], gyro_samples=samples)
            f = lambda: ctx.icp_run_odometry(prm, d["seqs"], d["T0"], None, motion="constant_velocity",  # noqa: E731
                                             map_frames=MAP_FRAMES, cell_size=CELL, **kw)
            return f if window else (lambda: prior(f))

        for name in args.workloads.split(","):
            if name == "tiles":
                d = tiles()
                ctx.set_target(d["map"], CELL)
            else:
                d = parking(WORKLOADS[name])
                noisy = parking(WORKLOADS[name], NOISE, BIAS)["samples"]
                ctx.set_target(_parking_map(np.random.default_rng(43), 500_000, 60.0), CELL)
            arms = {"seq_null": lambda: ctx.icp_run_sequences(prm, d["seqs"], d["T0"], None),
                    "seq_true": lambda: ctx.icp_run_sequences(prm, d["seqs"], d["T0"], d["deltas"]),
                    "prior_cv": odo(d)}
            if name != "tiles":
                arms.update({"prior_cv_deskew": odo(d, stamps=True),
                             "prior_gyro": odo(d, stamps=True, samples=d["samples"]),
                             "prior_gyro_noisy": odo(d, stamps=True, samples=noisy),
                             "window_gyro": odo(d, stamps=True, samples=d["samples"], window=True)})
            warm, repeats = {}, []

            def check(a, out):
                if a in warm:
                    repeats.append(all(h.same_bytes(x, y) for x, y in zip(out, warm[a])))
                else:
                    warm[a] = out
            outs, runs_ms, med = h.run_arms(ctx, arms, args.runs, DcregError, check)
            res = {a: warm.get(a, o) for a, o in outs.items()}
            ok_all &= all(repeats)
            n_frames = len(d["T_true"])
            out = {"frames": n_frames, "sequences": len(d["seqs"]), "arms": {}}
            for a in arms:
                if isinstance(res[a], str):
                    out["arms"][a] = {"error": res[a]}
                    continue
                out["arms"][a] = h.arm_block(n_frames, med[a], runs_ms[a], res[a], d["T_true"])
                dumps.update(h.result_dumps(f"{name}_{a}", res[a], ("T",)))
            line["workloads"][name] = out
    line["reproducible"] = bool(ok_all)
    h.finish(args, line, dumps, ok_all, 1)


if __name__ == "__main__":
    main()
