"""Synthetic scan pairs for the BASELINE.json configs (SURVEY.md §8d).  NumPy only; seeds fixed.

C2  make_cylinder : the shipped cylinder's geometry (wall R = 40 m, z in [0, 20] + floor disc z = 0) at any size
C3  make_parking  : ground-dominated local map + sparse verticals, LiDAR-like frame (stand-in, pair not shipped)
    make_parking_frames : the same map and a sequence of frames along a path through it (batched localisation)
    make_parking_pairs  : frame k+1 of that path against the local submap around pose k (scan/target pairs)
    make_parking_sequence : those frames with drifting odometry increments (sequences with chained priors)
    make_parking_sweeps : those frames skewed by the sensor's motion during each sweep, with per-point timestamps
    make_large_map / make_large_map_frames : 4 x 4 parking maps 1 km apart (too large for a dense grid) and frames in them
C4  make_corridor : two parallel walls + floor + ceiling, rank-deficient along x
C5  trial_poses   : seeded perturbations t ~ U[-1, 1]^3 m, rpy ~ U[-3, 3]^3 deg for the Monte-Carlo (SURVEY.md §8d)
    load_pcd_xyz  : PCD v0.7 `DATA binary` with float32 fields (the shipped clouds, SURVEY.md Appendix B.3)
"""
from __future__ import annotations

import math

import numpy as np


def pose6d_to_matrix(x, y, z, roll, pitch, yaw):
    """T = Trans * Rz * Ry * Rx (radians) - the reference's Pose6D2Matrix convention (utils.hpp:452-460)."""
    cr, sr, cp, sp, cy, sy = math.cos(roll), math.sin(roll), math.cos(pitch), math.sin(pitch), math.cos(yaw), math.sin(yaw)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]], dtype=np.float64)
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]], dtype=np.float64)
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]], dtype=np.float64)
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = [x, y, z]
    return T


def g2_initial_pose():
    """The perturbation of the reference's published cylinder run (0.2, 0.8, 0.5 m; 0.1, 0.1, 2 deg)."""
    d = math.pi / 180.0
    return pose6d_to_matrix(0.2, 0.8, 0.5, 0.1 * d, 0.1 * d, 2.0 * d)


def make_cylinder(n, seed=42, radius=40.0, height=20.0, noise=0.0):
    rng = np.random.default_rng(seed)
    nw = n // 2
    nf = n - nw
    th = rng.uniform(0, 2 * np.pi, nw); z = rng.uniform(0, height, nw)
    wall = np.stack([radius * np.cos(th), radius * np.sin(th), z], axis=1)
    rr = radius * np.sqrt(rng.uniform(0, 1, nf)); th2 = rng.uniform(0, 2 * np.pi, nf)
    floor = np.stack([rr * np.cos(th2), rr * np.sin(th2), np.zeros(nf)], axis=1)
    pts = np.concatenate([wall, floor], axis=0)
    if noise > 0:
        pts = pts + rng.normal(0, noise, pts.shape)
    return np.ascontiguousarray(pts, dtype=np.float32)


def make_corridor(n, seed=44, length=200.0, half_width=2.0, height=3.0, noise=0.0):
    rng = np.random.default_rng(seed)
    k = n // 4
    parts = []
    for ysign in (1.0, -1.0):
        x = rng.uniform(0, length, k); z = rng.uniform(0, height, k)
        parts.append(np.stack([x, np.full(k, ysign * half_width), z], axis=1))
    x = rng.uniform(0, length, k); y = rng.uniform(-half_width, half_width, k)
    parts.append(np.stack([x, y, np.zeros(k)], axis=1))
    m = n - 3 * k
    x = rng.uniform(0, length, m); y = rng.uniform(-half_width, half_width, m)
    parts.append(np.stack([x, y, np.full(m, height)], axis=1))
    pts = np.concatenate(parts, axis=0)
    if noise > 0:
        pts = pts + rng.normal(0, noise, pts.shape)
    return np.ascontiguousarray(pts, dtype=np.float32)


def _parking_map(rng, n_map, extent):
    ng = int(n_map * 0.9)
    g = np.stack([rng.uniform(-extent, extent, ng), rng.uniform(-extent, extent, ng),
                  -1.8 + rng.normal(0, 0.01, ng)], axis=1)
    nv = n_map - ng
    npil = 12
    centers = rng.uniform(-extent * 0.8, extent * 0.8, (npil, 2))
    which = rng.integers(0, npil, nv)
    ang = rng.uniform(0, 2 * np.pi, nv)
    v = np.stack([centers[which, 0] + 0.4 * np.cos(ang), centers[which, 1] + 0.4 * np.sin(ang),
                  rng.uniform(-1.8, 1.5, nv)], axis=1)
    return np.concatenate([g, v], axis=0).astype(np.float32)


def make_parking(n_map=500_000, n_scan=6_000, seed=43, extent=60.0, max_range=30.0):
    """Ground plane (z = -1.8 + 1 cm noise) with a few pillars/walls; the scan is a range-limited subsample of
    the map seen from the origin.  Planar degeneracy: x, y, yaw weakly constrained."""
    rng = np.random.default_rng(seed)
    tgt = _parking_map(rng, n_map, extent)
    rngs = np.linalg.norm(tgt[:, :2], axis=1)
    cand = np.nonzero(rngs < max_range)[0]
    pick = rng.choice(cand, size=min(n_scan, cand.size), replace=False)
    scan = (tgt[pick].astype(np.float64) + rng.normal(0, 0.005, (pick.size, 3))).astype(np.float32)
    return np.ascontiguousarray(scan), np.ascontiguousarray(tgt)


def make_parking_frames(n_frames, seed=47, n_map=500_000, n_scan=6_000, map_seed=43, extent=60.0, max_range=30.0,
                        path_half_length=20.0):
    """C3-shaped frames for map-based localisation: one make_parking map (same map_seed -> same map) and n_frames sensor
    poses along an S-shaped path through it (z = 0, heading along the path).  Frame k keeps every map point within
    max_range (horizontal) of the sensor with one fixed probability, chosen so that a frame at the path's start has about
    n_scan points (so the sizes are ragged), adds 5 mm noise and expresses the points in the sensor frame.
    The initial guesses are the true poses offset by the magnitudes of icp_pk01.yaml:30-44 (0.15 / 0.12 / 0.13 m,
    0.015 / 1.31 / 2.17 deg) with random signs.  Returns (frames: list of (N_k, 3) float32, T_true (n, 4, 4),
    T_init (n, 4, 4), map (n_map, 3) float32)."""
    tgt = _parking_map(np.random.default_rng(map_seed), n_map, extent)
    rng = np.random.default_rng(seed)
    s = np.linspace(-1.0, 1.0, n_frames) if n_frames > 1 else np.zeros(1)
    xs = path_half_length * s
    ys = 0.25 * path_half_length * np.sin(np.pi * s)
    heading = np.arctan2(0.25 * path_half_length * np.pi * np.cos(np.pi * s), path_half_length)
    T_true = np.array([pose6d_to_matrix(xs[k], ys[k], 0.0, 0.0, 0.0, heading[k]) for k in range(n_frames)])
    near0 = np.count_nonzero(np.hypot(tgt[:, 0] - xs[0], tgt[:, 1] - ys[0]) < max_range)
    keep_p = min(1.0, n_scan / max(near0, 1))
    frames, T_init = [], []
    d = math.pi / 180.0
    mag = np.array([0.15, 0.12, 0.13, 0.015 * d, 1.31 * d, 2.17 * d])
    for k in range(n_frames):
        near = np.nonzero(np.hypot(tgt[:, 0] - xs[k], tgt[:, 1] - ys[k]) < max_range)[0]
        pick = near[rng.random(near.size) < keep_p]
        pm = tgt[pick].astype(np.float64) + rng.normal(0, 0.005, (pick.size, 3))
        R, t = T_true[k][:3, :3], T_true[k][:3, 3]
        frames.append(np.ascontiguousarray(((pm - t) @ R).astype(np.float32)))        # R^T (p - t), row by row
        off = mag * rng.choice([-1.0, 1.0], 6)
        T_init.append(T_true[k] @ pose6d_to_matrix(*off))
    return frames, T_true, np.array(T_init), tgt


def make_parking_pairs(n_pairs, seed=53, n_map=500_000, n_scan=6_000, map_seed=43, extent=60.0, max_range=30.0,
                       path_half_length=20.0):
    """Scan-to-submap pairs (odometry along a recorded sequence, loop-closure checks): the n_pairs + 1 sensor poses and
    frames of make_parking_frames(n_pairs + 1, seed, ...).  Pair k registers frame k + 1 (in its own sensor frame)
    against the local submap around pose k: every map point within max_range (horizontal) of sensor k, plus 5 mm noise,
    in sensor frame k (about 100 k points at the defaults, ragged from pair to pair).  T_true[k] = inv(T_k) T_{k+1} maps
    the source onto its target; T_init[k] = T_true[k] times the icp_pk01.yaml offsets with random signs, as in
    make_parking_frames.  Returns (sources: list of (N_k, 3) float32, targets: list of (M_k, 3) float32,
    T_true (n, 4, 4), T_init (n, 4, 4))."""
    frames, T_world, _, tgt = make_parking_frames(n_pairs + 1, seed=seed, n_map=n_map, n_scan=n_scan, map_seed=map_seed,
                                                  extent=extent, max_range=max_range, path_half_length=path_half_length)
    rng = np.random.default_rng([seed, 1])
    d = math.pi / 180.0
    mag = np.array([0.15, 0.12, 0.13, 0.015 * d, 1.31 * d, 2.17 * d])
    targets, T_true, T_init = [], [], []
    for k in range(n_pairs):
        R, t = T_world[k][:3, :3], T_world[k][:3, 3]
        near = np.nonzero(np.hypot(tgt[:, 0] - t[0], tgt[:, 1] - t[1]) < max_range)[0]
        pm = tgt[near].astype(np.float64) + rng.normal(0, 0.005, (near.size, 3))
        targets.append(np.ascontiguousarray(((pm - t) @ R).astype(np.float32)))
        Tk = np.linalg.inv(T_world[k]) @ T_world[k + 1]
        T_true.append(Tk)
        T_init.append(Tk @ pose6d_to_matrix(*(mag * rng.choice([-1.0, 1.0], 6))))
    return frames[1:], targets, np.array(T_true), np.array(T_init)


def make_parking_sequence(n_frames, seed=47, odo_sigma=(0.03, 0.3), n_map=500_000, n_scan=6_000, map_seed=43,
                          extent=60.0, max_range=30.0, path_half_length=20.0):
    """A localisation sequence: the frames and true poses of make_parking_frames(n_frames, seed, ...) with the odometry
    a front end would feed dcreg_icp_run_sequences.  deltas[k] = inv(T_k) T_{k+1} times a seeded perturbation (each
    translation axis ~ N(0, odo_sigma[0]) m, each roll / pitch / yaw ~ N(0, odo_sigma[1]) deg), so that composing the
    increments alone (dead reckoning) drifts; the last entry is the identity (unused).  T_init0 = T_true[0] times the
    icp_pk01.yaml offsets with random signs, as in make_parking_frames.  Returns (frames: list of (N_k, 3) float32,
    T_true (n, 4, 4), T_init0 (4, 4), deltas (n, 4, 4), map (n_map, 3) float32)."""
    frames, T_true, T_init, tgt = make_parking_frames(n_frames, seed=seed, n_map=n_map, n_scan=n_scan, map_seed=map_seed,
                                                      extent=extent, max_range=max_range,
                                                      path_half_length=path_half_length)
    rng = np.random.default_rng([seed, 2])
    d = math.pi / 180.0
    deltas = np.tile(np.eye(4), (n_frames, 1, 1))
    for k in range(n_frames - 1):
        e = np.concatenate([rng.normal(0.0, odo_sigma[0], 3), rng.normal(0.0, odo_sigma[1] * d, 3)])
        deltas[k] = np.linalg.inv(T_true[k]) @ T_true[k + 1] @ pose6d_to_matrix(*e)
    return frames, T_true, T_init[0], deltas, tgt


def make_parking_sweeps(n_frames, seed=47, n_map=500_000, n_scan=6_000, map_seed=43, extent=60.0, max_range=30.0,
                        path_half_length=20.0):
    """make_parking_frames' path captured by a spinning LiDAR: each frame is a sweep during which the sensor moves.
    The frames of make_parking_frames(n_frames, seed, ...) are the unskewed frames, in the mid-sweep sensor frame of
    T_true[k].  Point i of frame k gets tau = (azimuth + pi) / (2 pi) in [0, 1] from its azimuth in that frame, and is
    measured from the sensor pose T_k Exp((tau - 0.5) xi_k) with xi_k = Log(inv(T_{k-1}) T_k) (frame 0 takes frame 1's):
    the skewed point is fl32(Exp(-(tau - 0.5) xi_k) p) (api.se3_exp_apply).  So the sweep motion is exactly the backward
    increment, and deskewing frame k with D = inv(T_{k-1}) T_k (api.deskew_points) gives the unskewed frame back up to
    float rounding.  Returns (skewed frames: list of (N_k, 3) float32, timestamps: list of (N_k,) float32, T_true
    (n, 4, 4) mid-sweep poses, deltas (n, 4, 4) with deltas[k] = inv(T_k) T_{k+1} (the last the identity), the
    unskewed frames)."""
    from dcreg_b200 import api
    frames, T_true, _, _ = make_parking_frames(n_frames, seed=seed, n_map=n_map, n_scan=n_scan, map_seed=map_seed,
                                               extent=extent, max_range=max_range, path_half_length=path_half_length)
    deltas = np.tile(np.eye(4), (n_frames, 1, 1))
    for k in range(n_frames - 1):
        deltas[k] = np.linalg.inv(T_true[k]) @ T_true[k + 1]
    skewed, stamps = [], []
    for k in range(n_frames):
        xi = api.se3_log(deltas[k - 1] if k > 0 else deltas[0]) if n_frames > 1 else np.zeros(6)
        p = frames[k].astype(np.float64)
        tau = ((np.arctan2(p[:, 1], p[:, 0]) + np.pi) / (2.0 * np.pi)).astype(np.float32)
        tau = np.clip(tau, np.float32(0.0), np.float32(1.0))
        s = tau.astype(np.float64) - 0.5
        skewed.append(np.ascontiguousarray(api.se3_exp_apply(xi, -s, p).astype(np.float32)))
        stamps.append(tau)
    return skewed, stamps, T_true, deltas, frames


def make_large_map(n_side=4, spacing=1000.0, n_map=500_000, map_seed=43, extent=60.0):
    """A prior map too large for a dense grid: n_side x n_side parking maps (_parking_map, tile t from seed map_seed + t),
    their centres spacing metres apart on a square lattice starting at the origin.  At 0.5 m cells the 4 x 4 default
    spans about 6 240 x 6 240 x 7 = 2.7e8 cells (dcreg_set_target_sparse).  Returns (map (n_side^2 n_map, 3) float32,
    tile centres (n_side^2, 3))."""
    tiles, centres = [], []
    for t in range(n_side * n_side):
        c = np.array([spacing * (t % n_side), spacing * (t // n_side), 0.0])
        tiles.append(_parking_map(np.random.default_rng(map_seed + t), n_map, extent).astype(np.float64) + c)
        centres.append(c)
    return np.ascontiguousarray(np.concatenate(tiles).astype(np.float32)), np.array(centres)


def make_large_map_frames(n_frames, seed=61, n_side=4, spacing=1000.0, n_map=500_000, n_scan=6_000, map_seed=43,
                          extent=60.0, max_range=30.0, path_half_length=20.0):
    """Frames for localisation against make_large_map(n_side, spacing, n_map, map_seed, extent): frame k lies in tile
    k % n_side^2, on that tile's make_parking_frames path (seed + t, map_seed + t), its poses shifted to the tile's centre,
    so that the frames of one tile form one sequence.  Returns (frames: list of (N_k, 3) float32, T_true (n, 4, 4),
    T_init (n, 4, 4), tile of every frame (n,))."""
    n_tiles = n_side * n_side
    tile = np.arange(n_frames) % n_tiles
    frames = [None] * n_frames
    T_true, T_init = np.zeros((n_frames, 4, 4)), np.zeros((n_frames, 4, 4))
    for t in range(n_tiles):
        ks = np.nonzero(tile == t)[0]
        if ks.size == 0:
            continue
        f, Tt, Ti, _ = make_parking_frames(ks.size, seed=seed + t, n_map=n_map, n_scan=n_scan, map_seed=map_seed + t,
                                           extent=extent, max_range=max_range, path_half_length=path_half_length)
        c = np.array([spacing * (t % n_side), spacing * (t // n_side), 0.0])
        for j, k in enumerate(ks):
            frames[k] = f[j]
            T_true[k], T_init[k] = Tt[j], Ti[j]
            T_true[k][:3, 3] += c
            T_init[k][:3, 3] += c
    return frames, T_true, T_init, tile


def trial_poses(n, seed=45, max_trans=1.0, max_rot_deg=3.0):
    """(n, 4, 4) initial poses of a perturbation Monte-Carlo (BASELINE.json configs[4])."""
    rng = np.random.default_rng(seed)
    t = rng.uniform(-max_trans, max_trans, (n, 3))
    rpy = np.deg2rad(rng.uniform(-max_rot_deg, max_rot_deg, (n, 3)))
    return np.array([pose6d_to_matrix(t[i, 0], t[i, 1], t[i, 2], rpy[i, 0], rpy[i, 1], rpy[i, 2]) for i in range(n)])


def load_pcd_xyz(path):
    """x, y, z columns of a PCD v0.7 file with `DATA binary` and 4-byte float fields (pcl::PointXYZI on disk)."""
    with open(path, "rb") as f:
        raw = f.read()
    head_end = raw.index(b"DATA binary") + len(b"DATA binary")
    head_end = raw.index(b"\n", head_end - 1) + 1
    hdr = {}
    for ln in raw[:head_end].decode("ascii", "replace").splitlines():
        tok = ln.split()
        if tok and not tok[0].startswith("#"):
            hdr[tok[0]] = tok[1:]
    if any(s != "4" for s in hdr["SIZE"]) or any(t != "F" for t in hdr["TYPE"]):
        raise ValueError("only 4-byte float fields are supported")
    nf, npts = len(hdr["FIELDS"]), int(hdr["POINTS"][0])
    a = np.frombuffer(raw, dtype="<f4", count=npts * nf, offset=head_end).reshape(npts, nf)
    cols = [hdr["FIELDS"].index(c) for c in ("x", "y", "z")]
    return np.ascontiguousarray(a[:, cols], dtype=np.float32)


def make_long_range_sequence(n_frames, seed=47, n_far=2_000, far_range=(150.0, 200.0), far_height=20.0, n_facades=8,
                             n_map=500_000, n_scan=6_000, map_seed=43, extent=60.0, max_range=30.0,
                             path_half_length=20.0):
    """A long-range sensor's recording: the frames of make_parking_frames(n_frames, seed, ...) plus sparse far
    structure, n_facades world-fixed vertical facades (30 m wide, far_height tall from the ground at z = -1.8) at
    horizontal distances in far_range from the origin, at evenly spaced azimuths.  Every frame sees n_far of their points
    (5 mm noise), in its sensor frame.  With the defaults a window map spans about 400 x 400 x 20 m: at 0.25 m cells about
    1 600 x 1 600 x 81 = 2.1e8 cells, past the dense grid's 2^27 (dcreg_set_sparse_maps).  Returns (frames: list of
    (N_k, 3) float32, T_true (n, 4, 4), deltas (n, 4, 4) with deltas[k] = inv(T_k) T_{k+1} (the last the identity))."""
    frames, T_true, _, _ = make_parking_frames(n_frames, seed=seed, n_map=n_map, n_scan=n_scan, map_seed=map_seed,
                                               extent=extent, max_range=max_range, path_half_length=path_half_length)
    rng = np.random.default_rng([seed, 3])
    walls = []
    for f in range(n_facades):
        az = 2.0 * np.pi * f / n_facades
        dist = rng.uniform(far_range[0], far_range[1])
        c, u = dist * np.array([np.cos(az), np.sin(az)]), np.array([-np.sin(az), np.cos(az)])
        m = 4 * n_far
        w = rng.uniform(-15.0, 15.0, m)
        walls.append(np.stack([c[0] + w * u[0], c[1] + w * u[1], -1.8 + rng.uniform(0.0, far_height, m)], axis=1))
    far = np.concatenate(walls)
    deltas = np.tile(np.eye(4), (n_frames, 1, 1))
    for k in range(n_frames - 1):
        deltas[k] = np.linalg.inv(T_true[k]) @ T_true[k + 1]
    out = []
    for k in range(n_frames):
        pm = far[rng.choice(far.shape[0], n_far, replace=False)] + rng.normal(0, 0.005, (n_far, 3))
        R, t = T_true[k][:3, :3], T_true[k][:3, 3]
        out.append(np.ascontiguousarray(np.concatenate([frames[k], ((pm - t) @ R).astype(np.float32)])))
    return out, T_true, deltas
