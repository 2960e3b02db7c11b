"""Frames/s of localisation against maps too large for a dense grid (their sparse row index), in the batched calls against
the dense grid, and against the per-frame loop.

Arms (radius = cell = 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3 (icp_pk01.yaml), method Ours):
  (a) dense : the 0.5 M-point parking map, dense grid; --frames frames of make_parking_frames as one dcreg_icp_run_scans
              call, and make_parking_sequence's frames in --lanes sequences as one dcreg_icp_run_sequences call;
  (b) sparse: the same map plus two far points that sort last in cell order and in index, so the box passes 2^27 cells:
              the same two calls on the sparse row index (b_equals_a_bit_for_bit reports whether they equal (a)'s: they must
              wherever every query cell under its initial pose lies inside the map's box, since the sorts agree there);
  (c) large : make_large_map (4 x 4 parking maps 1 km apart, --tile-points each, 2.7e8 cells of box) on the sparse index,
              --frames frames of make_large_map_frames as one _scans call and as one _sequences call (a sequence per
              tile, its increments from the true poses);
  (d) loop  : the large map through dcreg_set_target (the same sparse index as (c)) and the per-frame dcreg_set_source
              + dcreg_icp_run loop over (c)'s frames.
Calls are timed as tools/bench_scans.py times them (the max of CUDA events on the context's stream and the host wall
clock, host arrays in, results out, after a warm-up), --runs times, medians reported.  The sparse index's device bytes
(points, positions and table, computed from the build rule) are reported against the dense tables' 12 B per cell of the
box, with its build time (timed as the calls, the median of three).  Prints one JSON line with the card name and
power limit; --dump-outputs DIR writes every arm's poses, iterations, converged flags and statuses as float64 .npy."""
import numpy as np

import bench_harness as h

RADIUS = 0.5
FAR = np.array([[2000.0, 1500.0, 400.0], [3000.0, 3000.0, 500.0]], dtype=np.float32)


def index_bytes(xyz, cell):
    """Device bytes of the sparse row index of xyz (sparse_index.hpp): float4 points and int positions, and 12 B per table
    slot (a power of two at least twice the entries, an entry per (row, x) within [x' - 8, x' + 9] of an occupied x' of
    its row, clipped to [0, nx]); and the box's cell count."""
    c = np.floor(xyz.astype(np.float64) / cell).astype(np.int64)
    c -= c.min(axis=0)
    nx = int(c[:, 0].max()) + 1
    occ = np.unique(c, axis=0)                                   # (x, y, z) of occupied cells
    row = occ[:, 2] * (1 << 21) + occ[:, 1]
    xs = (occ[:, 0][:, None] + np.arange(-8, 10)[None, :])
    keys = row[:, None] * (1 << 21) + xs
    keys = keys[(xs >= 0) & (xs <= nx)]
    entries = int(np.unique(keys).size)
    cap = 1024
    while cap < 2 * entries:
        cap <<= 1
    box = float(np.prod(c.max(axis=0) + 1))
    return {"points": int(len(xyz)), "occupied_cells": int(len(occ)), "entries": entries, "table_slots": cap,
            "index_bytes": int(len(xyz) * 20 + cap * 12), "box_cells": box, "dense_table_bytes": 12.0 * box}


def main():
    ap = h.parser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--lanes", type=int, default=8)
    ap.add_argument("--tile-points", type=int, default=500_000)
    args = ap.parse_args()
    h.require_gpu()
    from dcreg_b200 import Context
    from dcreg_b200.scenes import make_large_map, make_large_map_frames, make_parking_frames, make_parking_sequence
    prm = h.c3_params(search_radius=RADIUS)
    n, L = args.frames, args.lanes
    frames, _, T_init, park = make_parking_frames(n, seed=47)
    sq_frames, _, sq_T0, sq_deltas, _ = make_parking_sequence(n, seed=47)
    per = n // L
    sq_frames, sq_deltas = sq_frames[:per * L], sq_deltas[:per * L]
    # every lane starts where the dead-reckoned sequence is at its first frame
    Tdr = [sq_T0]
    for k in range(per * L - 1):
        Tdr.append(Tdr[-1] @ sq_deltas[k])
    seq_T0 = np.array([Tdr[l * per] for l in range(L)])
    seqs = [sq_frames[l * per:(l + 1) * per] for l in range(L)]
    big, _ = make_large_map(n_map=args.tile_points)
    lf, lT_true, lT_init, tile = make_large_map_frames(n, n_map=args.tile_points)
    order = np.argsort(tile, kind="stable")
    groups = [order[tile[order] == t] for t in range(int(tile.max()) + 1)]
    groups = [g for g in groups if g.size]
    l_seqs = [[lf[k] for k in g] for g in groups]
    l_deltas = np.concatenate([[np.linalg.inv(lT_true[g[i]]) @ lT_true[g[min(i + 1, g.size - 1)]] for i in range(g.size)]
                               for g in groups])
    l_T0 = np.array([lT_init[g[0]] for g in groups])
    out, dumps = {}, {}
    with Context(0) as ctx:

        def arm(name, n_frames, fn):
            outs, ms, med = h.run_arms(ctx, {name: fn}, args.runs)
            res = outs[name]
            out[name] = {**h.rate(n_frames, med[name], ms[name]), "converged": int(sum(r.converged for r in res)),
                         "mean_iterations": float(np.mean([r.iterations for r in res]))}
            dumps.update(h.result_dumps(name, res, ("T", "iterations", "converged", "status")))
            return res

        def build_time(fn):
            return float(np.median([h.timed(ctx, fn)[1] for _ in range(3)]))

        ctx.set_target(park, RADIUS)
        a_scans = arm("a_dense_scans", n, lambda: ctx.icp_run_scans(prm, frames, T_init))
        a_seqs = arm("a_dense_sequences", per * L, lambda: ctx.icp_run_sequences(prm, seqs, seq_T0, sq_deltas))
        park_far = np.ascontiguousarray(np.concatenate([park, FAR]))
        out["b_build_ms"] = build_time(lambda: ctx.set_target_sparse(park_far, RADIUS))
        b_scans = arm("b_sparse_scans", n, lambda: ctx.icp_run_scans(prm, frames, T_init))
        b_seqs = arm("b_sparse_sequences", per * L, lambda: ctx.icp_run_sequences(prm, seqs, seq_T0, sq_deltas))
        same = all(x.T.tobytes() == y.T.tobytes() and (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
                   for x, y in zip(a_scans + a_seqs, b_scans + b_seqs))
        out["b_equals_a_bit_for_bit"] = same
        out["c_build_ms"] = build_time(lambda: ctx.set_target_sparse(big, RADIUS))
        arm("c_sparse_scans", n, lambda: ctx.icp_run_scans(prm, lf, lT_init))
        arm("c_sparse_sequences", n, lambda: ctx.icp_run_sequences(prm, l_seqs, l_T0, l_deltas))
        out["d_build_ms"] = build_time(lambda: ctx.set_target(big, RADIUS))

        def frame_loop():
            res = []
            for f, T in zip(lf, lT_init):
                ctx.set_source(f)
                res.append(ctx.icp_run(prm, T, want_log=False))
            return res
        arm("d_frame_loop", n, frame_loop)
    out["index_parking_sparse"] = index_bytes(park_far, RADIUS)
    out["index_large"] = index_bytes(big, RADIUS)
    out["speedup_c_scans_vs_d"] = out["c_sparse_scans"]["frames_per_s"] / out["d_frame_loop"]["frames_per_s"]
    out["speedup_c_sequences_vs_d"] = out["c_sparse_sequences"]["frames_per_s"] / out["d_frame_loop"]["frames_per_s"]
    line = {"metric": "frames_per_s", "frames": n, "lanes": L, "tile_points": args.tile_points, **out, "card": h.card()}
    h.finish(args, line, dumps)


if __name__ == "__main__":
    main()
