"""The middle of an ICP iteration - plane fit, per-slot row, Gram, world-frame congruence, sum of the block rows - against
the slot-level reference oracle/dcreg_oracle_rows.py, record by record at every entry point of the loop kernel and slot
by slot at the streaming kernel K1's edges, with its float32 ties bit for bit.

A record is recomputed from the pose its iteration ran at (the previous record's T; T_init, or T_prior for sequences
and odometry, for iteration 0) and must match: H27, the objective (1/2 sum b^2) and the rmse (sqrt(sum r^2 / N_eff))
within the reference's allowance; N_pt exactly up to slots whose q is in band; N_eff_clear <= N_eff <= N_eff_clear +
N_band; gradient == -H27[21:] byte for byte; fitness == N_pt / N_total exactly.  Entry points: icp_run (lean and
coherent iterations, ticket and solver-block paths), the batch, scans, pairs, sequences, and odometry with the window,
the capped voxel filters, the persistent voxel map and deskewed frames.  Outside the rank-deficient lattice the
band holds fewer than 1e-3 of the slots, so it cannot absorb a wrong row.  Each test prints records and slots checked,
band slots by reason and the worst |error| / allowance.

CPU tests (no GPU): the NumPy QR restatement against dla::colpiv_qr_solve<5,3> built as host code, bit for bit; the
reference against the plain oracle (find_correspondences + build_rows) on tie-free clouds; and the allowance's
sensitivity to a dropped, doubled, stale or foreign slot row.
"""
import math
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import dcreg_oracle as o
import dcreg_oracle_rows as rows
from harness import METHODS, ctx, init_T, ties_lattice, tool_program  # noqa: F401

F = np.float32
STATS = {}             # label -> [records, slots, band counts {reason: n}, worst error / allowance]


# ------------------------------------------------------------------------------------------------------------------
# shared checks
# ------------------------------------------------------------------------------------------------------------------
def check_record(label, rec, src, tgt, tree, T, prm, n_total=None, lattice=False):
    ref = rows.iteration_reference(src, tgt, tree, T, prm.search_radius, bool(prm.use_weight_derivative),
                                   slope=prm.weight_slope, gate=prm.weight_gate, min_norm=prm.min_normal_norm,
                                   thickness=prm.plane_thickness)
    n_total = len(src) if n_total is None else n_total
    H27 = np.array(rec.H27)
    n_eff = rec.n_effective
    sum_b2 = 2.0 * rec.objective
    sum_r2 = rec.rmse * rec.rmse * n_eff
    ref.allow[28] += 8 * rows.EPS * ref.sum_r2              # the rmse's square root and division
    ratio = ref.check(H27, sum_b2, sum_r2)
    where = (label, rec.iter)
    assert abs(rec.n_corr_pt - ref.n_pt) <= ref.n_pt_band, where + (rec.n_corr_pt, ref.n_pt, ref.n_pt_band)
    assert ref.n_eff_clear <= n_eff <= ref.n_eff_clear + ref.n_band, where + (n_eff, ref.n_eff_clear, ref.n_band)
    assert np.array(rec.gradient).tobytes() == (-H27[21:]).tobytes(), where
    assert rec.fitness == rec.n_corr_pt / n_total, where
    worst = float(ratio.max())
    assert worst <= 1.0, where + (int(ratio.argmax()), worst, ref.band_counts())
    if not lattice:
        assert ref.n_band <= 1e-3 * max(ref.n_slots, 1) + 1, where + (ref.band_counts(),)
    st = STATS.setdefault(label, [0, 0, {}, 0.0])
    st[0] += 1
    st[1] += ref.n_slots
    for k, v in ref.band_counts().items():
        st[2][k] = st[2].get(k, 0) + v
    st[3] = max(st[3], worst)
    return ref


def report(label):
    n, slots, band, worst = STATS[label]
    print(f"{label}: {n} records, {slots} slots, band {band or 'none'}, worst |error| / allowance {worst:.3g}")


def poses_of(res, T0):
    """the pose each record's iteration ran at"""
    return [np.asarray(T0, np.float64)] + [np.array(r.T).reshape(4, 4) for r in res.logs[:-1]]


def check_run(label, res, src, tgt, T0, prm, pick=None, tree=None, n_total=None, lattice=False):
    tree = cKDTree(np.asarray(tgt, np.float64)) if tree is None else tree
    poses = poses_of(res, T0)
    done = 0
    for i, rec in enumerate(res.logs):
        if rec.status != 0 or (pick is not None and i not in pick):
            continue
        check_record(label, rec, src, tgt, tree, poses[i], prm, n_total=n_total, lattice=lattice)
        done += 1
    return done


# ------------------------------------------------------------------------------------------------------------------
# CPU: the QR restatement, the reference against the plain oracle, sensitivity
# ------------------------------------------------------------------------------------------------------------------
def qr_systems(n=48_000, seed=3):
    """random, ill-conditioned, zero-column, dependent, duplicated, collinear, thin and all-zero 5x3 systems (float32
    coordinates, as the fit sees them)"""
    rng = np.random.default_rng(seed)
    P = ((rng.uniform(size=(n, 5, 3)) - 0.5) * 2.0).astype(F).astype(np.float64)
    kind = np.arange(n) % 9
    P[kind == 1] = ((rng.uniform(size=(np.sum(kind == 1), 5, 3)) - 0.5) * 80.0).astype(F)
    P[kind == 2, :, 2] = 0.0                                                   # z = 0 floor
    P[kind == 3, :, 1] = (2.0 * P[kind == 3, :, 0]).astype(F)                  # dependent columns
    P[kind == 4, 1] = P[kind == 4, 0]; P[kind == 4, 3] = P[kind == 4, 2]       # duplicated rows
    lat = np.array([[i * (j + 1) * 0.25 for j in range(3)] for i in range(5)])
    P[kind == 5] = lat.astype(F)                                               # collinear lattice
    P[kind == 6, :, 2] = (1e-6 * (rng.uniform(size=(np.sum(kind == 6), 5)) - 0.5)).astype(F)   # thin
    P[kind == 7] = 0.0
    off = rng.uniform(-30, 30, (np.sum(kind == 8), 1, 3))
    P[kind == 8] = (off + 0.3 * (rng.uniform(size=(np.sum(kind == 8), 5, 3)) - 0.5)).astype(F)  # far from the origin
    return P


def test_qr_restatement_is_bit_identical_to_the_host_build(tmp_path):
    exe = tool_program(tmp_path, "qr53_host.cu", compiler="nvcc")
    P = qr_systems()
    P.astype(np.float64).tofile(tmp_path / "a.bin")
    res = subprocess.run([str(exe), str(tmp_path / "a.bin"), str(tmp_path / "x.bin")], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    host = np.fromfile(tmp_path / "x.bin", dtype=np.float64).reshape(-1, 3)
    x, _ = rows.qr53(P)
    same = (x.view(np.uint64) == host.view(np.uint64)) | (np.isnan(x) & np.isnan(host))
    bad = np.nonzero(~same.all(axis=1))[0]
    assert bad.size == 0, (bad[:5], x[bad[:5]], host[bad[:5]])
    assert np.isnan(host[np.arange(len(P)) % 9 == 7]).all() or np.isinf(host[np.arange(len(P)) % 9 == 7]).any()


def surface_cloud(n, seed):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-4.0, 4.0, (n, 2))
    z = 0.15 * np.sin(1.3 * xy[:, 0]) * np.cos(0.9 * xy[:, 1]) + rng.normal(0, 0.01, n)
    return np.column_stack([xy, z]).astype(F)


@pytest.mark.parametrize("use_wd", [False, True])
def test_reference_agrees_with_the_plain_oracle(use_wd):
    """On a tie-free random cloud the reference's counts, gate decisions and sums are the plain oracle's (pinv fit,
    float64 kd-tree ranks): they differ only by rounding."""
    tgt = surface_cloud(6000, 11)
    src = surface_cloud(3000, 12)
    T = o.pose6d_to_matrix(0.03, -0.02, 0.01, 0.002, -0.001, 0.01)
    tree = cKDTree(tgt.astype(np.float64))
    ref = rows.iteration_reference(src, tgt, tree, T, 0.5, use_wd)
    corr = o.find_correspondences(src, tgt, tree, T[:3, :3], T[:3, 3], 0.5, use_wd)
    A, b = o.build_rows(src, corr, T[:3, :3])
    H, g = o.normal_equations(A, b)
    assert ref.n_pt == corr.n_pt and ref.n_eff == int(corr.valid.sum())
    assert np.array_equal(ref.valid, corr.valid)
    assert ref.n_band <= 0.005 * len(src)
    want = o.pack27(H, g)
    assert np.abs(ref.H27 - want).max() <= 1e-9 * np.abs(want).max()
    assert abs(ref.sum_b2 - float(b @ b)) <= 1e-9 * float(b @ b)
    assert abs(ref.sum_r2 - float(np.sum(corr.r[corr.valid] ** 2))) <= 1e-9 * ref.sum_r2


def faulty_sums(ref, slot_rows):
    """sums (27, sum b^2, sum r^2) of the per-slot rows (K, 8) given"""
    P = rows._pack_outer(slot_rows, slot_rows)
    s = np.array([math.fsum(P[:, i]) for i in range(29)])
    return s[:27], s[27], s[28]


def breaks(ref, H27, b2, r2):
    return ref.check(H27, b2, r2).max() > 1.0


def reference_rows(src, tgt, tree, T, prm_wd):
    """the reference and its per-slot rows (valid slots, reference frame)"""
    ref = rows.iteration_reference(src, tgt, tree, T, 1.0, prm_wd)
    e = ref.extras
    R = T[:3, :3]
    p64 = src.astype(np.float64)
    s = np.where(ref.valid, e["s"], 1.0)
    r = np.where(ref.valid, e["r"], 0.0)
    slot_rows, _, _ = rows._slot_rows(p64, R, np.where(ref.valid[:, None], e["n"], 0.0), r, s, prm_wd, 0.9)
    return ref, slot_rows


def test_allowance_catches_a_wrong_slot_row(cylinder):
    """On the shipped cylinder at the G2 pose every one of these faults breaks the allowance in at least one entry:
    dropping a clear valid slot (every slot of a random 200), counting a slot twice, one slot's plane from the previous
    iteration's pose, another trial's row in place of a slot's own."""
    from dcreg_b200.scenes import g2_initial_pose, trial_poses
    T0 = g2_initial_pose()
    tree = cKDTree(cylinder.astype(np.float64))
    conv, T_ref, logs, status = o.icp_so3(cylinder, cylinder, T0, o.Params(max_iterations=2, kappa_target=10.0,
                                                                           use_weight_derivative=True))
    T1 = logs[0].T
    ref, R1 = reference_rows(cylinder, cylinder, tree, T1, True)
    assert ref.n_band <= 1e-3 * ref.n_slots + 1
    H, b2, r2 = faulty_sums(ref, R1[ref.valid])
    assert not breaks(ref, H, b2, r2)                                  # the rows themselves pass
    clear_valid = np.nonzero(ref.valid & (ref.band == ""))[0]
    rng = np.random.default_rng(7)
    for i in rng.choice(clear_valid, 200, replace=False):
        keep = ref.valid.copy(); keep[i] = False
        assert breaks(ref, *faulty_sums(ref, R1[keep])), ("drop", i)
    i = clear_valid[0]
    assert breaks(ref, *faulty_sums(ref, np.concatenate([R1[ref.valid], R1[i:i + 1]]))), "twice"
    # stale plane: the slot's plane (and so its row) from the fit at the previous pose T0, at pose T1
    ref0, _ = reference_rows(cylinder, cylinder, tree, T0, True)
    e0, e1 = ref0.extras, ref.extras
    both = np.nonzero(ref.valid & ref0.valid & (ref.band == "") &
                      (np.abs(e0["n"] - e1["n"]).max(axis=1) > 0))[0]
    j = both[0]
    q = e1["q32"][j].astype(np.float64)
    r_st = float(e0["n"][j] @ q + e0["d"][j])
    s_st = 1.0 - 0.9 * abs(r_st)
    stale, _, _ = rows._slot_rows(cylinder[j:j + 1].astype(np.float64), T1[:3, :3], e0["n"][j:j + 1],
                                  np.array([r_st]), np.array([s_st]), True, 0.9)
    bad = R1.copy(); bad[j] = stale[0]
    assert breaks(ref, *faulty_sums(ref, bad[ref.valid])), "stale plane"
    # another trial's row: the same slot at a different trial's pose
    Tb = trial_poses(2, seed=45)[1]
    refb, Rb = reference_rows(cylinder, cylinder, tree, Tb, True)
    k = np.nonzero(ref.valid & refb.valid & (ref.band == ""))[0][0]
    bad = R1.copy(); bad[k] = Rb[k]
    assert breaks(ref, *faulty_sums(ref, bad[ref.valid])), "foreign row"


# ------------------------------------------------------------------------------------------------------------------
# GPU: the loop's records at every entry point
# ------------------------------------------------------------------------------------------------------------------
def ours(**over):
    from dcreg_b200 import default_params
    det, hand = METHODS["Ours"]
    kw = dict(detection=det, handling=hand, kappa_target=10.0)
    kw.update(over)
    return default_params(**kw)


@pytest.mark.gpu
@pytest.mark.parametrize("use_wd", [0, 1])
def test_c2_records(ctx, use_wd):
    """C2: 100 k cylinder, 50 fixed iterations: lean and coherent iterations, certificate and plane-cache reuse, the
    solver block"""
    from dcreg_b200.scenes import make_cylinder, g2_initial_pose
    pts = make_cylinder(100_000, seed=42)
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    prm = ours(max_iterations=50, fixed_iterations=1, use_weight_derivative=use_wd)
    res = ctx.icp_run(prm, g2_initial_pose())
    assert len(res.logs) == 50
    label = f"C2 wd={use_wd}"
    assert check_run(label, res, pts, pts, g2_initial_pose(), prm, pick={0, 1, 2, 3, 10, 30, 49}) == 7
    report(label)


@pytest.mark.gpu
def test_shipped_cylinder_g1_g2(ctx, golden, cylinder):
    tree = cKDTree(cylinder.astype(np.float64))
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    for setup, wd in (("G1", 0), ("G2", 1)):
        T0 = init_T(golden[setup]["setup"])
        prm = ours(use_weight_derivative=wd)
        res = ctx.icp_run(prm, T0)
        check_run("shipped cylinder", res, cylinder, cylinder, T0, prm, tree=tree)
    report("shipped cylinder")


@pytest.mark.gpu
def test_ragged_sizes_cells_and_sparse_index(ctx, cylinder):
    """tile tails (1 tile - 1, 32 k + 1, a last block with one slot), cells of radius / 2, 3, 4 (rings 2-4) and a
    sparse-row-index target"""
    from dcreg_b200.scenes import g2_initial_pose
    T0 = g2_initial_pose()
    tree = cKDTree(cylinder.astype(np.float64))
    ctx.set_target(cylinder, 1.0)
    prm = ours(max_iterations=6, fixed_iterations=1)
    for n in (255, 32 * 100 + 1, 256 * 21 + 1):
        src = cylinder[:n]
        ctx.set_source(src)
        check_run("ragged sizes", ctx.icp_run(prm, T0), src, cylinder, T0, prm, tree=tree)
    report("ragged sizes")
    ctx.set_source(cylinder)
    for div in (2, 3, 4):
        ctx.set_target(cylinder, 1.0 / div)
        check_run("cells r/2..r/4", ctx.icp_run(prm, T0), cylinder, cylinder, T0, prm, tree=tree, pick={0, 1, 5})
    report("cells r/2..r/4")
    tgt = np.concatenate([cylinder, np.array([[4000.0, 4500.0, 5000.0], [-4000.0, -3000.0, 2000.0]], F)]).astype(F)
    ctx.set_target(tgt, 1.0)
    check_run("sparse index", ctx.icp_run(prm, T0), cylinder, tgt, T0, prm)
    report("sparse index")


@pytest.mark.gpu
def test_lattice_with_duplicates_and_ties(ctx):
    tgt = ties_lattice()
    rng = np.random.default_rng(5)
    src = tgt[rng.permutation(len(tgt))[:7001]].copy()
    T0 = o.pose6d_to_matrix(0.06, -0.05, 0.04, math.radians(0.2), math.radians(-0.1), math.radians(0.4))
    prm = ours(max_iterations=25, fixed_iterations=1)
    ctx.set_source(src)
    ctx.set_target(tgt, 1.0)
    check_run("lattice", ctx.icp_run(prm, T0), src, tgt, T0, prm, pick={0, 1, 2, 12, 24}, lattice=True)
    report("lattice")


def with_nonfinite_rows(pts, frac, seed):
    rng = np.random.default_rng(seed)
    out = pts.copy()
    pick = rng.choice(len(pts), max(1, int(frac * len(pts))), replace=False)
    for k, i in enumerate(pick):
        out[i, k % 3] = (np.nan, np.inf, -np.inf)[k % 3]
    return out


@pytest.mark.gpu
def test_nonfinite_source_rows(ctx, cylinder):
    """1 % of the source rows with a NaN or +-Inf coordinate: no correspondence, no row, but they count in the
    fitness denominator (icp_run and the scan batch)"""
    from dcreg_b200.scenes import g2_initial_pose
    T0 = g2_initial_pose()
    src = with_nonfinite_rows(cylinder, 0.01, 3)
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(src)
    prm = ours(max_iterations=8, fixed_iterations=1)
    res = ctx.icp_run(prm, T0)
    assert res.status == 0 and len(res.logs) == 8
    check_run("non-finite rows", res, src, cylinder, T0, prm)
    scans = [src[:3000], with_nonfinite_rows(cylinder[3000:], 0.01, 4)]
    for sc, r in zip(scans, ctx.icp_run_scans(prm, scans, np.stack([T0, T0]), want_log=True)):
        assert r.status == 0
        check_run("non-finite rows", r, sc, cylinder, T0, prm)
    report("non-finite rows")


@pytest.mark.gpu
def test_me_tsvd_and_batch(ctx, cylinder):
    """ME-TSVD single run (ticket path, k2_step_kernel) and a 16-trial batch (per-trial records)"""
    from dcreg_b200 import default_params
    from dcreg_b200.scenes import g2_initial_pose, trial_poses
    T0 = g2_initial_pose()
    tree = cKDTree(cylinder.astype(np.float64))
    ctx.set_target(cylinder, 1.0)
    ctx.set_source(cylinder)
    prm = default_params(detection="FULL_EVD_MIN_EIGENVALUE", handling="TRUNCATED_SVD", max_iterations=10)
    check_run("ME-TSVD", ctx.icp_run(prm, T0), cylinder, cylinder, T0, prm, tree=tree)
    report("ME-TSVD")
    prm = ours(max_iterations=12)
    poses = trial_poses(16, seed=45)
    for k, r in enumerate(ctx.icp_run_batch(prm, poses, want_log=True)):
        check_run("icp_run_batch", r, cylinder, cylinder, poses[k], prm, tree=tree, pick={0, 1, 5, 11})
    report("icp_run_batch")


@pytest.fixture(scope="module")
def parking():
    from dcreg_b200.scenes import make_parking_frames, make_parking_pairs, make_parking_sequence
    frames, _, T_init, tgt = make_parking_frames(6, seed=51, n_scan=8_000)
    frames = [f[:n] for f, n in zip(frames, (40, 300, 2_001, 4_097, 8_000, 6_500))]
    src, ptgt, _, P_init = make_parking_pairs(3, seed=55, n_scan=4_000)
    seq, S_true, _, deltas, _ = make_parking_sequence(5, seed=61, n_scan=4_000)
    return frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_true[:1]


@pytest.mark.gpu
def test_scans_pairs_sequences(ctx, parking):
    frames, T_init, tgt, src, ptgt, P_init, seq, deltas, S_init = parking
    prm = ours(search_radius=0.5, max_iterations=20, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    ctx.set_target(tgt, 0.5)
    tree = cKDTree(tgt.astype(np.float64))
    for f, T0, r in zip(frames, T_init, ctx.icp_run_scans(prm, frames, T_init, want_log=True)):
        check_run("icp_run_scans", r, f, tgt, T0, prm, tree=tree, pick={0, 1, 2, 7})
    for s, t, T0, r in zip(src, ptgt, P_init, ctx.icp_run_pairs(prm, src, ptgt, P_init, want_log=True)):
        check_run("icp_run_pairs", r, s, t, T0, prm, pick={0, 1, 2, 7})
    for f, r in zip(seq, ctx.icp_run_sequences(prm, [seq], S_init, deltas, want_log=True)):
        check_run("icp_run_sequences", r, f, tgt, r.T_prior, prm, tree=tree, pick={0, 1, 4})
    for lab in ("icp_run_scans", "icp_run_pairs", "icp_run_sequences"):
        report(lab)


@pytest.mark.gpu
def test_odometry_window(ctx):
    """scan-to-map odometry: frame k's target is the map of the frames before it at their registered poses"""
    from dcreg_b200.api import map_points
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(6, seed=71, n_scan=8_000, max_range=20.0)
    prm = ours(search_radius=0.5, max_iterations=20, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)
    res = ctx.icp_run_odometry(prm, [frames], T_true[:1], deltas, map_frames=3, cell_size=0.5, want_log=True)
    for k in range(1, len(frames)):
        lo = max(0, k - 3)
        tgt = np.concatenate([map_points(res[j].T, frames[j]) for j in range(lo, k)]).astype(F)
        check_run("icp_run_odometry", res[k], frames[k], tgt, res[k].T_prior, prm, pick={0, 1, 3})
    report("icp_run_odometry")


@pytest.fixture(scope="module")
def odo_frames():
    from dcreg_b200.scenes import make_parking_sequence, make_parking_sweeps
    frames, T_true, _, deltas, _ = make_parking_sequence(6, seed=71, n_scan=8_000, max_range=20.0)
    skewed, stamps, S_true, s_deltas, unskewed = make_parking_sweeps(6, seed=71, n_scan=8_000, max_range=20.0)
    skewed[0] = unskewed[0]                                   # an unskewed anchor
    return frames, T_true, deltas, skewed, stamps, S_true, s_deltas


def odo_params():
    return ours(search_radius=0.5, max_iterations=20, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("caps", [(1, 4), (4, 1)], ids=["map-cap-4", "source-cap-4"])
def test_odometry_voxel_n(ctx, odo_frames, caps):
    """the capped voxel filters (dcreg_icp_run_odometry_voxel_n): source = frame k filtered with source_max_points,
    target = voxel_downsample(the window's filtered frames at their registered poses, map_voxel, map_max_points)"""
    from dcreg_b200.api import map_points, voxel_downsample
    frames, T_true, deltas = odo_frames[:3]
    sv, mv = 0.3, 0.25
    prm = odo_params()
    res = ctx.icp_run_odometry(prm, [frames], T_true[:1], deltas, map_frames=3, cell_size=0.5, want_log=True,
                               source_voxel=sv, map_voxel=mv, source_max_points=caps[0], map_max_points=caps[1])
    fs = [voxel_downsample(f, sv, caps[0])[0] for f in frames]
    label = f"odometry voxel_n caps {caps}"
    for k in range(1, len(frames)):
        assert res[k].n_points == len(fs[k])
        M = np.concatenate([map_points(res[j].T, fs[j]) for j in range(max(0, k - 3), k)])
        tgt = voxel_downsample(M, mv, caps[1])[0]
        check_run(label, res[k], fs[k], tgt, res[k].T_prior, prm, pick={0, 1, 3})
    report(label)


@pytest.mark.gpu
def test_odometry_voxel_map(ctx, odo_frames):
    """the persistent voxel map at a finite max_distance (dcreg_icp_run_odometry_map): target = the map twin M_k
    (api.voxel_map_update of the filtered frames at their registered poses)"""
    from dcreg_b200.api import voxel_downsample, voxel_map_update
    frames, T_true, deltas = odo_frames[:3]
    sv, mv, dist = 0.3, 0.25, 10.0
    prm = odo_params()
    res = ctx.icp_run_odometry_map(prm, [frames], T_true[:1], deltas, map_voxel=mv, max_distance=dist, cell_size=0.5,
                                   want_log=True, source_voxel=sv, map_max_points=4)
    fs = [voxel_downsample(f, sv, 1)[0] for f in frames]
    M = np.zeros((0, 3), F)
    for k in range(1, len(frames)):
        M = voxel_map_update(M, fs[k - 1], res[k - 1].T, mv, 4, dist)
        check_run("odometry voxel map", res[k], fs[k], M, res[k].T_prior, prm, pick={0, 1, 3})
    report("odometry voxel map")


@pytest.mark.gpu
def test_odometry_deskew(ctx, odo_frames):
    """deskewed frames (dcreg_icp_run_odometry_deskew): source = the frame's kept points after deskewing, target = the
    window's deskewed frames at their registered poses"""
    from dcreg_b200.api import map_points
    skewed, stamps, S_true, s_deltas = odo_frames[3:]
    prm = odo_params()
    res = ctx.icp_run_odometry(prm, [skewed], S_true[:1], s_deltas, map_frames=3, cell_size=0.5, want_log=True,
                               timestamps=[stamps], want_deskewed=True)
    moved = 0
    for k in range(1, len(skewed)):
        src = res[k].deskewed
        moved += int((src != np.asarray(skewed[k], F)[:, :3]).any(axis=1).sum())
        tgt = np.concatenate([map_points(res[j].T, res[j].deskewed) for j in range(max(0, k - 3), k)])
        check_run("odometry deskew", res[k], src, tgt, res[k].T_prior, prm, pick={0, 1, 3})
    assert moved > 0
    report("odometry deskew")


# ------------------------------------------------------------------------------------------------------------------
# GPU: K1 slot by slot at its edges
# ------------------------------------------------------------------------------------------------------------------
ROT_Z90 = np.array([[0.0, -1.0, 0.0, 0.0], [1.0, 0.0, 0.0, 0.0], [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]])
K_DEPTH, WARPS = 4, 8                          # k1_stream.cuh: ring depth, warps per CTA (a warp's chunks are 8 apart)
# residuals r whose s r = (1 - 0.9 r) r is exactly a float32 tie under both evaluation orders of s (the first rounds
# up to even, the second down)
SR_TIES = (0.30000000919984754, 0.30000010638135555)


def designed_slots(T, plane_dtype):
    """(points (k, 4) float32, planes (k, 4) plane_dtype, huge (k,) bool) of the edge cases at pose T (identity or
    axis-aligned); huge marks the slots with coordinates of 1e5 m and beyond"""
    R, t = T[:3, :3], T[:3, 3]
    pts, pls, huge = [], [], []

    def add(p, n, d=None, big=False):
        p = np.array(p, np.float64)
        n = np.array(n, np.float64)
        if d is None:                  # a plane through q = fl32(R p + t) where that is finite: r = 0
            with np.errstate(all="ignore"):
                q = (np.where(np.isfinite(p), p, 0.0) @ R.T + t).astype(F).astype(np.float64)
            d = -float(np.where(n != 0.0, n * q, 0.0).sum())
        pts.append(list(p) + [0.0]); pls.append(list(n) + [d]); huge.append(big)

    bad = (np.nan, np.inf, -np.inf)
    for v in bad:                                  # a non-finite point coordinate, plane with zero components
        for axis in range(3):
            p = [0.5, -0.25, 0.75]; p[axis] = v
            for nrm in ((0.0, 0.0, 1.0), (0.0, 1.0, 0.0), (1.0, 0.0, 0.0)):
                add(p, nrm)
    for v in bad:                                  # a non-finite plane component
        for comp in range(4):
            n = [0.0, 0.0, 1.0, None]
            if comp < 3:
                n[comp] = v
                add([0.0, 0.5, 0.0], n[:3], d=0.0)
            else:
                add([0.0, 0.5, 0.0], n[:3], d=v)
    add([0.0, -0.0, 0.0], (0.0, 0.0, 1.0))         # +-0 and float32 denormals: a documented deviation
    add([1e-40, -1e-42, 2.0], (0.0, 0.0, 1.0))
    add([3e-39, 0.5, -1e-45], (1.0, 0.0, 0.0))
    add([1.0e5, -3.0e5, 12.5], (0.0, 0.0, 1.0), big=True)    # far coordinates
    add([-7.0e5, 1.0e6, -2.0], (0.0, 1.0, 0.0), big=True)
    add([3.4e38, 0.0, 1.0], (0.0, 0.0, 1.0), big=True)       # up to FLT_MAX (q stays finite at these poses)
    add([0.0, -3.4e38, 1.0], (0.0, 0.0, 1.0), big=True)
    # s at the gate and one ulp either side: r = d at a point whose q is 0 (t = 0 at these poses).  FP64 planes: the
    # FP64 neighbours of the residual where 1 - 0.9 |r| (both evaluation orders) crosses 0.1; float32 planes: the float32
    # neighbours of 1.0, where it crosses (s(1 - 2^-24) > 0.1 >= s(1))
    if plane_dtype == np.float64:
        r_gate = gate_residual()
        gate_rs = (np.nextafter(r_gate, 0.0), r_gate, np.nextafter(r_gate, 2.0))
    else:
        gate_rs = (float(np.nextafter(F(1.0), F(0.0))), 1.0, float(np.nextafter(F(1.0), F(2.0))))
    for r in gate_rs:
        for sgn in (1.0, -1.0):
            add([0.0, 0.0, 0.0], (0.0, 0.0, 1.0), d=sgn * r)
    add([0.0, 0.0, 0.0], (0.0, 0.0, 1.0), d=0.0)          # r = 0 (s = 1, k = 1)
    pl = np.array(pls, np.float64).astype(plane_dtype)
    return np.array(pts, F), pl, np.array(huge)


def gate_residual():
    """the residual r > 0 closest to the gate for which 1 - 0.9 r equals 0.1 or crosses it under both the reference's
    two roundings and the kernel's FMA"""
    r = 1.0
    for _ in range(64):
        s_plain = 1.0 - 0.9 * r
        s_fma = rows._exact_fma(r, -0.9, 1.0)
        if s_plain > 0.1 and s_fma > 0.1:
            return r
        r = float(np.nextafter(r, 0.0))
    raise AssertionError("no residual at the gate")


def k1_check(ctx, src4, planes, T, use_wd, designed, label, stats):
    ref = rows.k1_reference(src4, planes, T, use_wd, designed=designed)
    out, st = ctx.reduce_normal_equations(src4, planes, T, use_wd)
    assert int(st[2]) == ref.n_pt, (label, st[2], ref.n_pt)
    assert ref.n_eff_clear <= int(st[1]) <= ref.n_eff_clear + ref.n_band, (label, st[1], ref.n_eff_clear, ref.n_band)
    ratio = ref.check(out, np.nan, st[0])
    ratio[27] = 0.0                                       # the seam reports no sum b^2
    assert np.isfinite(out).all(), (label, out)
    worst = float(ratio.max())
    assert worst <= 1.0, (label, int(ratio.argmax()), worst, out[int(ratio.argmax()) % 27], ref.band_counts())
    stats[0] += 1
    stats[1] += len(src4)
    for k, v in ref.band_counts().items():
        stats[2][k] = stats[2].get(k, 0) + v
    stats[3] = max(stats[3], worst)
    return ref


def random_slots(n, T, seed):
    rng = np.random.default_rng(seed)
    src = rng.uniform(-30, 30, (n, 4)).astype(F)
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    q = (src[:, :3].astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(F).astype(np.float64)
    d = -(nrm * q).sum(1) + rng.uniform(-1.2, 1.2, n)
    return src, np.concatenate([nrm, d[:, None]], axis=1)


def cta_ranges(n, sm_count):
    """k1_stream.cuh with launch_reduce's grid: each CTA's contiguous chunk range [c_lo, c_hi)"""
    nchunks = (n + 31) // 32
    g = max(1, min(2 * sm_count, (nchunks + WARPS - 1) // WARPS))
    per, rem = divmod(nchunks, g)
    lo = [tm * per + min(tm, rem) for tm in range(g)]
    return [(a, a + per + (1 if tm < rem else 0)) for tm, a in enumerate(lo)]


def edge_positions(n, sm):
    """first and last slot; around the start of every CTA range (the slot before it, its first slot, its first chunk's
    end); and, in a few CTAs, both end lanes of warps 0 and 7's chunks 3 .. 9: the prologue's last ring slot, the main
    loop's consumes and ring refills, and the drain"""
    ranges = cta_ranges(n, sm)
    pos = {0, n - 1}
    for a, _ in ranges[1:]:
        pos |= {32 * a - 1, 32 * a, 32 * a + 31}
    for tm in (0, 1, len(ranges) // 2, len(ranges) - 1):
        a, b = ranges[tm]
        for w in (0, WARPS - 1):
            for j in range(3, 10):
                c = a + w + WARPS * j
                if c < b:
                    pos |= {32 * c, 32 * c + 31}
    return sorted(p for p in pos if 0 <= p < n), ranges


def exact_row_sums(u, b):
    """the 27 sums of one slot at the origin, identity pose: c = [0, 0, 0, u, b, r]"""
    c = np.zeros(8)
    c[3:6] = u
    c[6] = b
    H = np.outer(c[:6], c[:6])
    return o.pack27(H, c[:6] * c[6])


K1_STATS = {}


@pytest.mark.gpu
@pytest.mark.parametrize("use_wd", [False, True])
@pytest.mark.parametrize("plane_dtype", [np.float32, np.float64])
def test_k1_edge_slots(ctx, use_wd, plane_dtype):
    """Every designed slot alone (n = 1); the ordinary ones embedded in a random array large enough that every warp
    runs K1's main ring loop, at the first and last slot, around every CTA range's start and at ring refills (the slots
    with coordinates of 1e5 m and beyond only alone: their magnitude would swamp the embedded array's allowance); sizes
    1, one and two chunks +-1, CTA-range boundaries +-1, and the sizes where each warp has kDepth - 1, kDepth and
    kDepth + 1 chunks (+1 slot)"""
    import torch
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    label = f"K1 edges ({plane_dtype.__name__}, wd={use_wd})"
    stats = K1_STATS.setdefault(label, [0, 0, {}, 0.0])
    for T in (np.eye(4), ROT_Z90):
        pts, pls, huge = designed_slots(T, plane_dtype)
        for i in range(len(pts)):
            k1_check(ctx, pts[i:i + 1], pls[i:i + 1], T, use_wd, [0], "alone", stats)
        pts, pls = pts[~huge], pls[~huge]
        n = 2 * sm * WARPS * (2 * K_DEPTH + 2) * 32 + 7            # 10 chunks per warp: nmain = 4
        src, planes = random_slots(n, T, 9)
        planes = planes.astype(plane_dtype)
        pos, ranges = edge_positions(n, sm)
        assert len(ranges) == 2 * sm and len(pos) >= len(pts)
        chosen = [pos[k * len(pos) // len(pts)] for k in range(len(pts))]
        chosen[0], chosen[-1] = 0, n - 1
        for k, p in enumerate(chosen):
            src[p] = pts[k]; planes[p] = pls[k]
        k1_check(ctx, src, planes, T, use_wd, chosen, "embedded", stats)
    full = 2 * sm * WARPS * 32                                       # one chunk per warp of the full grid
    sizes = [1, 31, 32, 33, 63, 64, 65, full - 1, full, full + 1]
    sizes += [c * full + e for c in (K_DEPTH - 1, K_DEPTH, K_DEPTH + 1) for e in (0, 1)]
    for n in sizes:
        src, planes = random_slots(n, ROT_Z90, n)
        k1_check(ctx, src, planes.astype(plane_dtype), ROT_Z90, use_wd, None, f"n={n}", stats)
    print(f"{label}: {stats[0]} calls, {stats[1]} slots, band {stats[2] or 'none'}, "
          f"worst |error| / allowance {stats[3]:.3g}")


@pytest.mark.gpu
@pytest.mark.parametrize("use_wd", [False, True])
def test_k1_float32_ties_bit_exact(ctx, use_wd):
    """s n_i and s r exactly on a float32 tie round to even, both directions, compared bit for bit: one slot at the
    origin at the identity pose, so every product the sums take is exact.  s n: r = 0, s = 1 (k = 1 either way);
    s r: the residuals SR_TIES (without the weight derivative: with it, k = 2 - 1/s is a Newton reciprocal)"""
    z = np.zeros((1, 4), F)
    for nx in (1.0 + 2.0 ** -24, 1.0 + 3 * 2.0 ** -24, 0.75 + 2.0 ** -25, 0.75 + 3 * 2.0 ** -25):
        plane = np.array([[nx, 0.0, 0.0, 0.0]])
        out, st = ctx.reduce_normal_equations(z, plane, np.eye(4), use_wd)
        u = float(F(nx))                                             # round half to even
        assert u != nx and st[1] == 1
        want = exact_row_sums([u, 0.0, 0.0], -0.0)
        assert out.tobytes() == want.tobytes() or np.array_equal(out, want), (nx, out, want)
    if use_wd:
        return
    ups = []
    for r in SR_TIES:
        s = 1.0 - 0.9 * r
        assert rows._exact_fma(r, -0.9, 1.0) == s
        sr = s * r
        assert (np.float64(sr).view(np.uint64) & np.uint64(0x1FFFFFFF)) == 0x10000000      # an exact tie
        b = -float(F(sr))
        ups.append(-b > sr)
        out, st = ctx.reduce_normal_equations(z, np.array([[0.0, 0.0, 1.0, r]]), np.eye(4), False)
        want = exact_row_sums([0.0, 0.0, float(F(s))], b)
        assert st[1] == 1 and np.array_equal(out, want), (r, out, want)
        assert st[0] == r * r
    assert sorted(ups) == [False, True]
