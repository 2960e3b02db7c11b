"""Every instantiation of the loop kernel icp_iter2_kernel<kUseWd, kGrids, kSeq, kPlanes, kSparse> against the
slot-level reference oracle/dcreg_oracle_rows.py, each one proven to have run by the context's per-variant launch
counter (dcreg_loop_variant_launches).

CASES maps a case to the loop_plan.hpp variant it must run, the planner inputs that give that variant, and its call.
A case's call runs on the module's context and returns how to rebuild each record's source, target and pose; the test
asserts that the call's loop launches all landed on the case's variant, then checks iterations 0, 1 and the last of
every registered frame with rows_harness.check_record (seam 1: every slot's plane against knn5 + fit_planes_qr) and
prints records, slots, band counts and the worst |error| / allowance.  The cases:
  * the weight derivative at every entry point on dense grids (1, 3, 5, 7): the batch, scans, ME-TSVD on icp_run (the
    ticket path), pairs, sequences, and odometry with the window, the voxel map at a finite max_distance and deskewed
    frames; the twins without it (2, 4, 6);
  * sparse row indexes with and without it (8 - 15): icp_run and the batch on a target past the dense-grid limit,
    pairs under dcreg_set_sparse_maps whose targets carry a far point, sequences on a sparse context target, odometry
    whose anchor carries a far point (so that every window is past the limit);
  * the adaptive threshold with it (7 on the voxel map, 15 on sparse windows): each frame checked at its own radius;
  * non-default plane_thickness, min_normal_norm, weight_slope and weight_gate on pairs with it (3);
  * seam 1, find_planes on a dense grid and on a sparse index (16, 17).

CPU: the table's expected variants cover all 18, and each agrees with loop_plan::variant_flags (read from the header
through tools/test_loop_plan.cpp).  GPU: the cheapest case of every variant once on a fresh context: all 18 counts
positive."""
import subprocess
from dataclasses import dataclass
from functools import cached_property
from typing import Callable

import numpy as np
import pytest
from scipy.spatial import cKDTree

import dcreg_oracle_rows as rows
from harness import METHODS, ctx, tool_program  # noqa: F401
from rows_harness import check_run, report

F = np.float32
CELL = 0.5
FAR = np.array([[3.0e4, 3.0e4, 50.0]], F)        # 6e4 cells of 0.5 m from the scenes: a box far past 2^27 cells
CEILING = 2.0                                     # the adaptive cases' search_radius: four rings of 0.5 m cells


@dataclass(frozen=True)
class Flags:
    """the inputs of loop_plan::variant a call gives"""
    use_wd: bool = False
    grids: bool = False       # every trial its own grid (pairs, odometry)
    seq: bool = False         # sequence lanes (sequences, odometry)
    sparse: bool = False
    planes: bool = False      # seam 1 (find_planes)


@dataclass(frozen=True)
class Case:
    variant: int
    flags: Flags
    call: Callable            # (ctx, scenes) -> (params, verify(label)): the call, then the checks of its records
    cost: int                 # rough relative cost, for the coverage test's cheapest case of each variant


# ------------------------------------------------------------------------------------------------------------------
# scenes, built when a case first needs them
# ------------------------------------------------------------------------------------------------------------------
class Scenes:
    def __init__(self, cylinder):
        self.cylinder = np.ascontiguousarray(cylinder, F)

    @cached_property
    def cylinder_far(self):
        """the shipped cylinder and two far points (as test_gpu_normal_equations' sparse index): past 2^27 cells of 1 m"""
        far = np.array([[4000.0, 4500.0, 5000.0], [-4000.0, -3000.0, 2000.0]], F)
        return np.ascontiguousarray(np.concatenate([self.cylinder, far]))

    @cached_property
    def pairs(self):
        """3 pairs: 4 k-point frames against their 20 m submaps"""
        from dcreg_b200.scenes import make_parking_pairs
        src, tgt, _, T_init = make_parking_pairs(3, seed=55, n_scan=4_000, max_range=20.0)
        return src, tgt, T_init

    @cached_property
    def sequence(self):
        """4 frames of 4 k points, the drifting increments, the map"""
        from dcreg_b200.scenes import make_parking_sequence
        frames, T_true, _, deltas, tgt = make_parking_sequence(4, seed=61, n_scan=4_000)
        return frames, T_true[:1], deltas, tgt

    @cached_property
    def odometry(self):
        """5 frames of about 6 k points within 20 m"""
        from dcreg_b200.scenes import make_parking_sequence
        frames, T_true, _, deltas, _ = make_parking_sequence(5, seed=71, n_scan=6_000, max_range=20.0)
        return frames, T_true[:1], deltas

    @cached_property
    def odometry_far(self):
        """odometry with FAR in the anchor: with a window as long as the sequence, every frame's map holds it"""
        frames, T0, deltas = self.odometry
        return [np.ascontiguousarray(np.concatenate([frames[0], FAR]))] + list(frames[1:]), T0, deltas

    @cached_property
    def sweeps(self):
        """4 skewed sweeps of about 6 k points with per-point timestamps, the anchor unskewed"""
        from dcreg_b200.scenes import make_parking_sweeps
        skewed, stamps, T_true, deltas, unskewed = make_parking_sweeps(4, seed=71, n_scan=6_000, max_range=20.0)
        skewed[0] = unskewed[0]
        return skewed, stamps, T_true[:1], deltas


@pytest.fixture(scope="module")
def scenes(cylinder):
    return Scenes(cylinder)


# ------------------------------------------------------------------------------------------------------------------
# helpers
# ------------------------------------------------------------------------------------------------------------------
def ours(**over):
    from dcreg_b200 import default_params
    det, hand = METHODS["Ours"]
    kw = dict(detection=det, handling=hand, kappa_target=10.0)
    kw.update(over)
    return default_params(**kw)


def parking_params(wd, **over):
    kw = dict(search_radius=0.5, max_iterations=12, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3,
              use_weight_derivative=wd)
    kw.update(over)
    return ours(**kw)


def ends(res):
    """iterations 0, 1 and the last"""
    return {0, 1, len(res.logs) - 1}


def box_cells(pts, cell):
    c = np.floor(np.asarray(pts, dtype=np.float64) * (1.0 / cell))
    return int(np.prod(c.max(0) - c.min(0) + 1))


def assert_sparse(pts, cell):
    assert box_cells(pts, cell) > 2 ** 27, box_cells(pts, cell)


def check_frames(label, prm, jobs, radius=None):
    """jobs: (result, source, target, pose of iteration 0[, radius]) per registered frame; iterations 0, 1 and the last
    of each.  Returns the radii checked."""
    radii = []
    for job in jobs:
        r, src, tgt, T0 = job[:4]
        rad = job[4] if len(job) > 4 else radius
        assert r.status == 0 and len(r.logs) >= 1, (label, r.status, len(r.logs))
        assert check_run(label, r, src, tgt, T0, prm, pick=ends(r), radius=rad) >= 1, label
        radii.append(prm.search_radius if rad is None else rad)
    report(label)
    return radii


def with_sparse_maps(ctx, fn):
    ctx.set_sparse_maps(True)
    try:
        return fn()
    finally:
        ctx.set_sparse_maps(False)


# ------------------------------------------------------------------------------------------------------------------
# the calls
# ------------------------------------------------------------------------------------------------------------------
def batch(wd, sparse):
    def call(ctx, sc):
        from dcreg_b200.scenes import trial_poses
        tgt = sc.cylinder_far if sparse else sc.cylinder
        ctx.set_target(tgt, 1.0)
        ctx.set_source(sc.cylinder)
        prm = ours(max_iterations=8, use_weight_derivative=wd)
        poses = trial_poses(4, seed=45)
        res = ctx.icp_run_batch(prm, poses, want_log=True)

        def verify(label):
            if sparse:
                assert_sparse(tgt, 1.0)
            return check_frames(label, prm, [(r, sc.cylinder, tgt, T) for r, T in zip(res, poses)])
        return prm, verify
    return call


def scans(wd):
    def call(ctx, sc):
        from dcreg_b200.scenes import g2_initial_pose
        cyl = sc.cylinder
        ctx.set_target(cyl, 1.0)
        prm = ours(max_iterations=8, use_weight_derivative=wd)
        T0 = g2_initial_pose()
        sl = [cyl[:4000], cyl[3000:]]
        res = ctx.icp_run_scans(prm, sl, np.stack([T0, T0]), want_log=True)
        return prm, lambda label: check_frames(label, prm, [(r, s, cyl, T0) for r, s in zip(res, sl)])
    return call


def single(wd, sparse, method="Ours"):
    def call(ctx, sc):
        from dcreg_b200 import default_params
        from dcreg_b200.scenes import g2_initial_pose
        tgt = sc.cylinder_far if sparse else sc.cylinder
        ctx.set_target(tgt, 1.0)
        ctx.set_source(sc.cylinder)
        det, hand = METHODS[method]
        prm = default_params(detection=det, handling=hand, kappa_target=10.0, max_iterations=8,
                             use_weight_derivative=wd)
        T0 = g2_initial_pose()
        res = ctx.icp_run(prm, T0)

        def verify(label):
            if sparse:
                assert_sparse(tgt, 1.0)
            return check_frames(label, prm, [(res, sc.cylinder, tgt, T0)])
        return prm, verify
    return call


SETTINGS = dict(plane_thickness=0.15, min_normal_norm=0.1, weight_slope=0.8, weight_gate=0.15)


def pairs(wd, sparse, settings=False):
    def call(ctx, sc):
        src, tgt, T_init = sc.pairs
        if sparse:
            tgt = [np.ascontiguousarray(np.concatenate([t, FAR])) for t in tgt]
        prm = parking_params(wd, **(SETTINGS if settings else {}))
        run = lambda: ctx.icp_run_pairs(prm, src, tgt, T_init, want_log=True)      # noqa: E731
        res = with_sparse_maps(ctx, run) if sparse else run()

        def verify(label):
            if settings:
                for k, v in SETTINGS.items():
                    assert getattr(prm, k) == v and getattr(prm, k) != getattr(ours(), k), k
            for t in tgt if sparse else ():
                assert_sparse(t, CELL)
            return check_frames(label, prm, [(r, s, t, T) for r, s, t, T in zip(res, src, tgt, T_init)])
        return prm, verify
    return call


def sequences(wd, sparse):
    def call(ctx, sc):
        frames, S0, deltas, tgt = sc.sequence
        if sparse:
            tgt = np.ascontiguousarray(np.concatenate([tgt, FAR]))
        ctx.set_target(tgt, CELL)
        prm = parking_params(wd)
        res = ctx.icp_run_sequences(prm, [frames], S0, deltas, want_log=True)

        def verify(label):
            if sparse:
                assert_sparse(tgt, CELL)
            return check_frames(label, prm, [(r, f, tgt, r.T_prior) for f, r in zip(frames, res)])
        return prm, verify
    return call


def window_jobs(frames, res, map_frames, sources=None):
    """frame k >= 1: (result, source, the window's frames at their registered poses, T_prior, the returned radius)"""
    from dcreg_b200.api import map_points
    sources = frames if sources is None else sources
    out = []
    for k in range(1, len(frames)):
        tgt = np.concatenate([map_points(res[j].T, sources[j]) for j in range(max(0, k - map_frames), k)]).astype(F)
        out.append((res[k], sources[k], tgt, res[k].T_prior, res[k].search_radius or None))
    return out


def odometry_window(wd, sparse, adaptive=False):
    def call(ctx, sc):
        from dcreg_b200.api import AdaptiveThreshold
        frames, T0, deltas = sc.odometry_far if sparse else sc.odometry
        map_frames = len(frames) if sparse else 3
        prm = parking_params(wd, search_radius=CEILING if adaptive else 0.5)
        kw = dict(adaptive=AdaptiveThreshold(0.12, 0.01, 20.0)) if adaptive else {}
        run = lambda: ctx.icp_run_odometry(prm, [frames], T0, deltas, map_frames=map_frames, cell_size=CELL,  # noqa: E731
                                           want_log=True, **kw)
        res = with_sparse_maps(ctx, run) if sparse else run()

        def verify(label):
            jobs = window_jobs(frames, res, map_frames)
            for job in jobs if sparse else ():
                assert_sparse(job[2], CELL)
            if not adaptive:
                jobs = [j[:4] for j in jobs]
            return check_frames(label, prm, jobs)
        return prm, verify
    return call


def odometry_voxel_map(wd, adaptive=False):
    def call(ctx, sc):
        from dcreg_b200.api import AdaptiveThreshold, voxel_downsample, voxel_map_update
        frames, T0, deltas = sc.odometry
        sv, mv, dist = (0.0, 0.25, 10.0) if adaptive else (0.3, 0.25, 10.0)
        prm = parking_params(wd, search_radius=CEILING if adaptive else 0.5)
        kw = dict(adaptive=AdaptiveThreshold(0.12, 0.01, 20.0)) if adaptive else dict(source_voxel=sv)
        res = ctx.icp_run_odometry_map(prm, [frames], T0, deltas, map_voxel=mv, max_distance=dist, cell_size=CELL,
                                       want_log=True, map_max_points=4, **kw)

        def verify(label):
            fs = [voxel_downsample(f, sv, 1)[0] for f in frames] if sv else frames
            jobs, M = [], np.zeros((0, 3), F)
            for k in range(1, len(frames)):
                M = voxel_map_update(M, fs[k - 1], res[k - 1].T, mv, 4, dist)
                jobs.append((res[k], fs[k], M, res[k].T_prior, res[k].search_radius if adaptive else None))
            return check_frames(label, prm, jobs)
        return prm, verify
    return call


def odometry_deskew(wd):
    def call(ctx, sc):
        skewed, stamps, T0, deltas = sc.sweeps
        prm = parking_params(wd)
        res = ctx.icp_run_odometry(prm, [skewed], T0, deltas, map_frames=3, cell_size=CELL, want_log=True,
                                   timestamps=[stamps], want_deskewed=True)

        def verify(label):
            moved = sum(int((res[k].deskewed != np.asarray(skewed[k], F)[:, :3]).any(axis=1).sum())
                        for k in range(1, len(skewed)))
            assert moved > 0
            jobs = window_jobs(skewed, res, 3, sources=[r.deskewed for r in res])
            return check_frames(label, prm, [j[:4] for j in jobs])
        return prm, verify
    return call


def find_planes(sparse):
    def call(ctx, sc):
        from dcreg_b200 import default_params
        from dcreg_b200.scenes import pose6d_to_matrix
        tgt = sc.cylinder_far if sparse else sc.cylinder
        ctx.set_target(tgt, 1.0)
        ctx.set_source(sc.cylinder)
        T = pose6d_to_matrix(0.02, -0.01, 0.01, 0.002, 0.001, -0.004)       # near the cylinder: 4x G2's planes
        planes, npt = ctx.find_planes(T, 1.0)

        def verify(label):
            if sparse:
                assert_sparse(tgt, 1.0)
            check_planes(label, sc.cylinder, tgt, T, 1.0, planes, npt)
        return default_params(), verify
    return call


PLANE_STATS = {}


def check_planes(label, src, tgt, T, radius, planes, npt):
    """find_planes slot by slot: N_pt exactly up to slots whose q is in band; outside the band (q, and the fit's rank,
    norm and thickness decisions) a slot has a plane exactly when the reference does, and its plane lies within 64 times
    the FP64 fit's measured distance from the extended-precision one (with a floor of 16 eps per entry)"""
    p64 = np.asarray(src, F).astype(np.float64)
    R, t = T[:3, :3], T[:3, 3]
    qv, q32 = rows.transform_f32(p64, R, t)
    qband = rows.q_band_mask(qv) & np.isfinite(q32).all(axis=1)
    tree = cKDTree(np.asarray(tgt, np.float64))
    idx, _, near = rows.knn5(tree, np.asarray(tgt, F), q32.astype(F), radius)
    assert abs(npt - int(near.sum())) <= int(qband.sum()), (label, npt, int(near.sum()), int(qband.sum()))
    n_slots = len(src)
    ref = np.zeros((n_slots, 4))
    allow = np.full((n_slots, 4), np.inf)
    band = np.where(qband, "q", "").astype(object)
    sel = np.nonzero(near)[0]
    nb = np.asarray(tgt, F)[idx[sel]].astype(np.float64)
    n, d, ok, nl, dl, reason = rows.fit_planes_qr(nb)
    ref[sel, :3], ref[sel, 3] = n, d
    allow[sel, :3] = rows.BAND_FACTOR * (np.abs(n - nl) + 16 * rows.EPS)
    allow[sel, 3] = rows.BAND_FACTOR * (np.abs(d - dl) + 16 * rows.EPS * np.abs(d))
    band[sel] = np.where(band[sel] == "", reason, band[sel])
    has_ref = np.zeros(n_slots, bool)
    has_ref[sel] = ok
    clear = band == ""
    has_gpu = np.abs(planes[:, :3]).sum(axis=1) > 0
    bad = np.nonzero(clear & (has_gpu != has_ref))[0]
    assert bad.size == 0, (label, bad[:5], has_gpu[bad[:5]], has_ref[bad[:5]])
    assert not planes[clear & ~has_ref].any(), label
    chk = clear & has_ref
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.abs(planes[chk] - ref[chk])
        ratio = np.where(err == 0.0, 0.0, err / allow[chk])
    worst = float(ratio.max()) if ratio.size else 0.0
    assert worst <= 1.0, (label, np.nonzero(chk)[0][int(ratio.argmax()) // 4], worst)
    counts = {r: int(np.sum(band == r)) for r in rows.REASONS if np.any(band == r)}
    assert int((~clear).sum()) <= 1e-3 * n_slots + 1, (label, counts)
    assert int(has_ref.sum()) > 0 and int(chk.sum()) >= 0.9 * int(has_ref.sum()), (label, int(chk.sum()))
    print(f"{label}: {n_slots} slots, {int(chk.sum())} planes checked, band {counts or 'none'}, "
          f"worst |error| / allowance {worst:.3g}")


# ------------------------------------------------------------------------------------------------------------------
# the table
# ------------------------------------------------------------------------------------------------------------------
WD = Flags(use_wd=True)
CASES = {
    "icp_run": Case(0, Flags(), single(0, False), 1),
    "icp_run wd": Case(1, WD, single(1, False), 1),
    "batch wd": Case(1, WD, batch(1, False), 4),
    "scans wd": Case(1, WD, scans(1), 2),
    "icp_run ME-TSVD wd": Case(1, WD, single(1, False, "ME-TSVD"), 1),
    "pairs": Case(2, Flags(grids=True), pairs(0, False), 3),
    "pairs wd": Case(3, Flags(use_wd=True, grids=True), pairs(1, False), 3),
    "pairs wd fit and weight settings": Case(3, Flags(use_wd=True, grids=True), pairs(1, False, settings=True), 4),
    "sequences": Case(4, Flags(seq=True), sequences(0, False), 3),
    "sequences wd": Case(5, Flags(use_wd=True, seq=True), sequences(1, False), 3),
    "odometry window": Case(6, Flags(grids=True, seq=True), odometry_window(0, False), 3),
    "odometry window wd": Case(7, Flags(use_wd=True, grids=True, seq=True), odometry_window(1, False), 3),
    "odometry voxel map wd": Case(7, Flags(use_wd=True, grids=True, seq=True), odometry_voxel_map(1), 4),
    "odometry deskew wd": Case(7, Flags(use_wd=True, grids=True, seq=True), odometry_deskew(1), 4),
    "odometry voxel map adaptive wd": Case(7, Flags(use_wd=True, grids=True, seq=True),
                                           odometry_voxel_map(1, adaptive=True), 5),
    "icp_run sparse": Case(8, Flags(sparse=True), single(0, True), 1),
    "icp_run sparse wd": Case(9, Flags(use_wd=True, sparse=True), single(1, True), 1),
    "batch sparse wd": Case(9, Flags(use_wd=True, sparse=True), batch(1, True), 4),
    "pairs sparse": Case(10, Flags(grids=True, sparse=True), pairs(0, True), 3),
    "pairs sparse wd": Case(11, Flags(use_wd=True, grids=True, sparse=True), pairs(1, True), 3),
    "sequences sparse": Case(12, Flags(seq=True, sparse=True), sequences(0, True), 3),
    "sequences sparse wd": Case(13, Flags(use_wd=True, seq=True, sparse=True), sequences(1, True), 3),
    "odometry sparse": Case(14, Flags(grids=True, seq=True, sparse=True), odometry_window(0, True), 3),
    "odometry sparse wd": Case(15, Flags(use_wd=True, grids=True, seq=True, sparse=True), odometry_window(1, True), 3),
    "odometry sparse adaptive wd": Case(15, Flags(use_wd=True, grids=True, seq=True, sparse=True),
                                        odometry_window(1, True, adaptive=True), 4),
    "find_planes": Case(16, Flags(planes=True), find_planes(False), 1),
    "find_planes sparse": Case(17, Flags(planes=True, sparse=True), find_planes(True), 1),
}


# ------------------------------------------------------------------------------------------------------------------
# CPU: the table against loop_plan.hpp
# ------------------------------------------------------------------------------------------------------------------
def test_cases_cover_every_variant_with_its_flags(tmp_path):
    exe = tool_program(tmp_path, "test_loop_plan.cpp")
    res = subprocess.run([str(exe), "--flags"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    table = {}
    for line in res.stdout.split("\n"):
        if line.strip():
            v, wd, grids, seq, planes, sparse = (int(x) for x in line.split())
            table[v] = Flags(use_wd=bool(wd), grids=bool(grids), seq=bool(seq), sparse=bool(sparse), planes=bool(planes))
    assert sorted(table) == list(range(18))
    assert sorted({c.variant for c in CASES.values()}) == list(range(18))
    for name, c in CASES.items():
        assert table[c.variant] == c.flags, (name, c.variant, table[c.variant], c.flags)


# ------------------------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------------------------
def launches_of(ctx, case, scenes):
    """the case's call, and the loop launches it took per variant"""
    before = ctx.loop_variant_launches
    prm, verify = case.call(ctx, scenes)
    return prm, verify, ctx.loop_variant_launches - before


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_case_records_against_the_reference(ctx, scenes, name):
    case = CASES[name]
    prm, verify, delta = launches_of(ctx, case, scenes)
    others = {v: int(n) for v, n in enumerate(delta) if v != case.variant and n}
    print(f"{name}: variant {case.variant}, {int(delta[case.variant])} loop launches")
    assert delta[case.variant] > 0 and not others, (name, case.variant, delta.tolist())
    if not case.flags.planes:
        assert bool(prm.use_weight_derivative) == case.flags.use_wd, name
    radii = verify(name)
    if "adaptive" in name:
        # the frames were checked at their own radii: at least two, neither the ceiling params.search_radius
        print(f"{name}: radii checked {radii}")
        assert len(set(radii) - {prm.search_radius}) >= 2, (name, radii)


@pytest.mark.gpu
def test_every_variant_runs(scenes):
    """the cheapest case of every variant, once, on a fresh context: each of the 18 counts goes up"""
    from dcreg_b200 import Context
    cheapest = {}
    for name, c in CASES.items():
        if c.variant not in cheapest or c.cost < CASES[cheapest[c.variant]].cost:
            cheapest[c.variant] = name
    with Context(0) as c:
        assert not c.loop_variant_launches.any()
        for v in sorted(cheapest):
            CASES[cheapest[v]].call(c, scenes)
        counts = c.loop_variant_launches
    print("loop launches per variant:", counts.tolist())
    assert (counts > 0).all(), counts.tolist()
