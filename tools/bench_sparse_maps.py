"""Frames/s of scan-to-map odometry whose local maps are too large for dense grids (dcreg_set_sparse_maps), against the
only route such maps had before, and the cost of the sparse index on maps that would fit.

Arms (radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, method Ours; the increments are the scene's true ones, so that
every arm runs the whole recording):
  (a) long range: make_long_range_sequence (parking frames plus facades at 150 - 200 m, 20 m tall) at 0.25 m cells,
      whose window maps span about 2e8 cells (past 2^27), with the setting on:
        window     - dcreg_icp_run_odometry, map_frames 10, as 1 x --frames and as --lanes x (--frames / --lanes);
        voxel map  - dcreg_icp_run_odometry_map, map_voxel 0.25, 20 points per voxel, max_distance = inf, same shapes;
        host loop  - the per-frame route: api.map_points of the window + set_target_sparse + set_source + icp_run from
                     the call's own priors (the window's 1 x --frames recording; the voxel map's host route would
                     spend its time in the NumPy map update, so it is not timed).
  (b) index cost: the same recording without the facades (every step dense) against the same recording plus one point
      30 km away, above every other point, in every frame, which makes every step sparse; both window calls,
      1 x --frames and --lanes x (--frames / --lanes).  forced_sparse_equals_dense_bit_for_bit reports whether their
      poses and iteration counts agree (the extra point changes the largest frame, and with it the tile size, so they
      need not).
Each call is timed as tools/bench_scans.py times its calls (the max of CUDA events on the context's stream and the host
wall clock), after one warm-up call of the same shape; the arms alternate, --runs rounds, medians reported.  Prints one
JSON line with the card name and power limit read in the same run; --dump-outputs DIR writes every odometry arm's poses,
iterations, converged flags and statuses as .npy."""
import numpy as np

import bench_harness as h

RADIUS = 0.5
CELL = 0.25


def split(frames, lanes):
    n = len(frames) // lanes
    return [frames[s * n:(s + 1) * n] for s in range(lanes)]


def main():
    ap = h.parser()
    ap.add_argument("--frames", type=int, default=128)
    ap.add_argument("--lanes", type=int, default=8)
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.scenes import make_long_range_sequence

    prm = h.c3_params(search_radius=RADIUS)
    far_frames, T_true, deltas = make_long_range_sequence(args.frames, seed=91)
    near_frames = [f[:len(f) - 2_000] for f in far_frames]              # the same recording without the facades
    one_far = np.array([[3.0e4, 3.0e4, 60.0]], np.float32)
    shapes = {"1x%d" % args.frames: 1, "%dx%d" % (args.lanes, args.frames // args.lanes): args.lanes}

    def recording(frames, lanes, plus_far=False):
        seqs = split(frames, lanes)
        if plus_far:
            seqs = [[np.concatenate([f, one_far]) for f in s] for s in seqs]
        T0 = np.stack([T_true[s * len(seqs[0])] for s in range(lanes)])
        return seqs, T0

    ctx = Context(0)
    ctx.set_sparse_maps(True)
    arms = {}
    for tag, lanes in shapes.items():
        arms["window_%s" % tag] = (recording(far_frames, lanes), "window")
        arms["voxel_map_%s" % tag] = (recording(far_frames, lanes), "voxel")
        arms["dense_%s" % tag] = (recording(near_frames, lanes), "window")
        arms["forced_sparse_%s" % tag] = (recording(near_frames, lanes, plus_far=True), "window")

    def run(name):
        (seqs, T0), kind = arms[name]
        if kind == "window":
            return ctx.icp_run_odometry(prm, seqs, T0, deltas, map_frames=10, cell_size=CELL)
        return ctx.icp_run_odometry_map(prm, seqs, T0, deltas, map_voxel=CELL,
                                        map_max_points=20, max_distance=float("inf"), cell_size=CELL)

    host = "host_loop_window_1x%d" % args.frames
    seqs_w, _ = arms["window_1x%d" % args.frames][0]
    res_w = run("window_1x%d" % args.frames)                        # the priors the host loop starts from

    def host_loop():
        seq = seqs_w[0]
        for k in range(1, len(seq)):
            ctx.set_target_sparse(h.window_map(seq, [r.T for r in res_w], k, 10), CELL)
            ctx.set_source(seq[k])
            ctx.icp_run(prm, res_w[k].T_prior, want_log=False)
    outs, _, med = h.run_arms(ctx, {**{name: lambda name=name: run(name) for name in arms}, host: host_loop}, args.runs)
    result = {"bench": "sparse_maps", "card": h.card(), "frames": args.frames, "lanes": args.lanes, "cell": CELL,
              "runs": args.runs, "frames_per_s": {}}
    for name in arms:
        nf = sum(len(s) for s in arms[name][0][0])
        result["frames_per_s"][name] = nf / (med[name] * 1e-3)
    result["frames_per_s"][host] = (args.frames - 1) / (med[host] * 1e-3)
    m9 = h.window_map(seqs_w[0], [r.T for r in res_w], 10, 10)
    c = np.floor(m9.astype(np.float64) / CELL)
    result["window_map_box_cells"] = float(np.prod(c.max(0) - c.min(0) + 1))
    same = []
    for tag in shapes:
        a, b = outs["dense_%s" % tag], outs["forced_sparse_%s" % tag]
        same.append(all(x.T.tobytes() == y.T.tobytes() and x.iterations == y.iterations for x, y in zip(a, b)))
    result["forced_sparse_equals_dense_bit_for_bit"] = same
    dumps = {}
    for name in arms:
        dumps[name + "_T"] = [x.T for x in outs[name]]
        dumps[name + "_iters"] = [[x.iterations, x.converged, x.status] for x in outs[name]]
    ctx.close()
    h.finish(args, result, dumps)


if __name__ == "__main__":
    main()
