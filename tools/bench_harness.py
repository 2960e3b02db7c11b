"""What the benchmark tools share: paths, the card, the GPU check, the common flags, the C3 solver settings, one timer,
the arms driver, the parking-sequence workloads, pose errors, map sizes, the replay check, the per-arm JSON block and
the output.

torch and dcreg_b200 are imported inside the functions that use them, so that every tool's --help works on a machine
without a GPU."""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))

METHODS = {                       # the six methods the CLI's SO(3) path recognises: (detection, handling)
    "Ours": ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG"),
    "NONE": ("NONE_DETE", "NONE_HAND"),
    "ME-SR": ("FULL_EVD_MIN_EIGENVALUE", "SOLUTION_REMAPPING"),
    "FCN-SR": ("FULL_SVD_CONDITION", "SOLUTION_REMAPPING"),
    "ME-TSVD": ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD"),
    "ME-TReg": ("FULL_EVD_MIN_EIGENVALUE", "STANDARD_REGULARIZATION"),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power}
    except Exception:
        return {"name": None, "power_limit": None}


def parser():
    """The tools' argument parser: --runs (timed rounds) and --dump-outputs DIR; each tool adds its own flags."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None)
    return ap


def require_gpu():
    import torch
    if not torch.cuda.is_available():
        raise SystemExit(f"{os.path.basename(sys.argv[0])}: no CUDA device - dcreg_b200 has no CPU fallback")


def c3_params(method="Ours", **over):
    """The C3 settings of icp_pk01.yaml: radius 0.5, 30 iterations, ROT 1e-5 / TRANS 1e-3, kappa 10, under `method`"""
    from dcreg_b200 import default_params
    detection, handling = METHODS[method]
    kw = dict(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0,
              detection=detection, handling=handling)
    return default_params(**{**kw, **over})


def timed(ctx, fn):
    """(fn(), ms): the larger of CUDA events on the context's stream around the call and the host wall clock around it.
    The events end in a synchronise inside the wall-clock window, so for calls that return host results the larger is
    the wall time."""
    import torch
    stream = torch.cuda.ExternalStream(ctx.stream)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w = time.perf_counter()
    e0.record(stream)
    out = fn()
    e1.record(stream)
    e1.synchronize()
    w = time.perf_counter() - w
    return out, max(e0.elapsed_time(e1), w * 1e3)


def run_arms(ctx, arms, runs, errors=(), check=None):
    """Warm every arm of {name: fn} up once, in order, then time `runs` rounds (at least one) of the arms in turn.  The
    warm-up goes through the timer too, so the first round pays none of its set-up.  An arm whose warm-up raises one of
    `errors` keeps the message as its output and is not timed.  check(arm, output), if given, sees every output, the
    warm-up's first; only an arm's latest output is kept, so a timed call reuses the memory of the output before it.
    Returns ({arm: the last round's output}, {arm: [ms of every round]}, {arm: median ms})."""
    outs = {}
    for a, fn in arms.items():
        try:
            out = timed(ctx, fn)[0]
        except errors as e:
            outs[a] = str(e)
            continue
        if check:
            check(a, out)
    ms = {a: [] for a in arms if a not in outs}
    for _ in range(max(1, runs)):
        for a in ms:
            outs[a], t = timed(ctx, arms[a])
            ms[a].append(t)
            if check:
                check(a, outs[a])
    return outs, ms, {a: float(np.median(t)) for a, t in ms.items()}


def parking_sequences(spec, **scene):
    """The sequences make_parking_sequence(n, seed, **scene) draws for every (n, seed) of spec (scene: n_map, n_scan,
    max_range), each anchored at its first true pose: (frames per sequence, T0 (S, 4, 4), the increments and the true
    poses concatenated over the sequences)."""
    from dcreg_b200.scenes import make_parking_sequence
    seqs, T0, deltas, T_true = [], [], [], []
    for n, seed in spec:
        frames, Tt, _, D, _ = make_parking_sequence(n, seed=seed, **scene)
        seqs.append(frames); T0.append(Tt[0]); deltas.append(D); T_true.append(Tt)
    return seqs, np.array(T0), np.concatenate(deltas), np.concatenate(T_true)


def per_sequence(seqs, res):
    """res, one entry per frame of seqs in order, split into one list per sequence"""
    ends = np.cumsum([len(s) for s in seqs])
    return [res[e - len(s):e] for s, e in zip(seqs, ends)]


def pose_errors(T_true, T):
    """Largest translation (m) and rotation (deg) error of the poses T against T_true."""
    import dcreg_oracle as o
    dt, dr = 0.0, 0.0
    for A, B in zip(T_true, T):
        E = np.linalg.inv(A) @ B
        dt = max(dt, float(np.linalg.norm(E[:3, 3])))
        dr = max(dr, float(np.degrees(np.linalg.norm(o.so3_log(E[:3, :3])))))
    return dt, dr


def map_sizes(seqs_sizes, map_frames):
    """Map points of every step over the sequences of a window map of unfiltered frames, from the frames' point counts"""
    out = []
    for i in range(1, max(len(f) for f in seqs_sizes)):
        out.append(sum(sum(f[j] for j in range(max(0, i - map_frames), i)) for f in seqs_sizes if len(f) > i))
    return out


def window_map(frames, poses, j, map_frames):
    """The local map of a window odometry at frame j: frames[j - map_frames:j] placed at their poses"""
    from dcreg_b200.api import map_points
    return np.concatenate([map_points(poses[i], frames[i]) for i in range(max(0, j - map_frames), j)])


def same_bytes(a, b):
    return ((a.status, a.iterations, a.converged, a.n_points) == (b.status, b.iterations, b.converged, b.n_points)
            and a.T.tobytes() == b.T.tobytes() and a.T_prior.tobytes() == b.T_prior.tobytes())


def replay(ctx, prm, sources, res, target, cell, points=False):
    """Every registered frame of an odometry call against its single run: set_target(its map, cell) +
    set_source(its source) + icp_run from its T_prior.  sources: each sequence's frames as the call registered them;
    res: the call's results in order; target(s, j, rs, M): the map of frame j >= 1 of sequence s, rebuilt from the
    sequence's results rs and frame j - 1's map M (frame 1's M is empty); prm: the settings, or a function of the
    frame's result that gives them, or None to rebuild the maps only; points: also require n_points == the source's
    size.  Returns (status, iterations and converged identical on every frame, the largest SE(3) log distance of the
    poses, the map points of every step summed over the sequences)."""
    import dcreg_oracle as o
    same, worst, sizes = True, 0.0, {}
    for s, rs in enumerate(per_sequence(sources, res)):
        M = np.zeros((0, 3), np.float32)
        for j in range(1, len(rs)):
            M = target(s, j, rs, M)
            sizes[j] = sizes.get(j, 0) + len(M)
            if prm is None:
                continue
            ctx.set_target(M, cell)
            ctx.set_source(sources[s][j])
            one = ctx.icp_run(prm(rs[j]) if callable(prm) else prm, rs[j].T_prior, want_log=False)
            same = same and (one.status, one.iterations, one.converged) == (rs[j].status, rs[j].iterations,
                                                                            rs[j].converged)
            same = same and (not points or rs[j].n_points == len(sources[s][j]))
            d = float(o.se3_log_distance(one.T, rs[j].T))
            worst = d if d > worst or math.isnan(d) else worst                 # a NaN stays, and fails any tolerance
    return same, worst, [sizes[j] for j in sorted(sizes)]


def spread(sizes):
    return {"min": int(min(sizes)), "max": int(max(sizes)), "total": int(sum(sizes))}


def rate(n, ms, runs_ms, prefix="", unit="frames"):
    """The {prefix}{unit}_per_s, {prefix}ms and {prefix}runs_ms keys of n items in a median of ms"""
    return {f"{prefix}{unit}_per_s": n / (ms * 1e-3), f"{prefix}ms": ms, f"{prefix}runs_ms": runs_ms}


def arm_block(n_frames, ms, runs_ms, res, T_true):
    """An odometry arm's JSON block: its rate, iterations and converged frames over the registered frames (those that
    ran an iteration), and the largest error against the true poses"""
    reg = [r for r in res if r.iterations > 0]
    dt, dr = pose_errors(T_true, [r.T for r in res])
    return {**rate(n_frames, ms, runs_ms), "mean_iterations": float(np.mean([r.iterations for r in reg])),
            "converged": int(sum(r.converged for r in reg)), "registered": len(reg),
            "max_err_vs_truth": {"trans_m": dt, "rot_deg": dr}}


FIELDS = ("T", "T_prior", "iterations", "converged", "status")


def result_dumps(prefix, res, fields=FIELDS):
    """{prefix_field: the field of every result} for the dump writer"""
    return {f"{prefix}_{k}": [getattr(r, k) for r in res] for k in fields}


def finish(args, line, dumps, ok=True, failure=None):
    """Print the JSON line, write dumps ({file name: values}) under --dump-outputs as float64 .npy files, and exit with
    `failure` unless ok."""
    print(json.dumps(line))
    if args.dump_outputs:
        os.makedirs(args.dump_outputs, exist_ok=True)
        for k, v in dumps.items():
            np.save(os.path.join(args.dump_outputs, k + ".npy"), np.asarray(v, dtype=np.float64))
    if not ok:
        raise SystemExit(failure)
