"""dcreg_set_target past the dense-grid limit, and its alias dcreg_set_target_sparse: the sparse row index for maps too
large for a dense grid (sparse_index.hpp).

Target B is a parking map (plus four points at its far corners that stretch its box in z over every query): a dense grid.
Target A is B plus two far points that sort after every map cell and come last in index, which lifts A's box past 2^27
cells: a sparse row index whose points and positions are B's, followed by the two.  For sources whose query cells stay
inside B's box, every call on A must equal the same call on B bit for bit - T, T_prior, status, iterations, converged,
cov and every log record but its iter_time_ms - and find_planes must too; A built by dcreg_set_target and by
dcreg_set_target_sparse is the same build (launches) and gives the same bits.  On the 4 x 4 tile map (make_large_map)
every scan and sequence frame equals its own single run on the same sparse target, as the batched calls' contracts
state, and a call reproduces bit for bit.
"""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o
from harness import RADIUS, ctx, log_bytes, params  # noqa: F401

pytestmark = pytest.mark.gpu

FAR = np.array([[2000.0, 1500.0, 400.0], [3000.0, 3000.0, 500.0]], dtype=np.float32)


@pytest.fixture(scope="module")
def scene():
    """B: a 300 k-point parking map and four far-corner points at z = -6 and +5; A: B and FAR.  12 frames along a path
    through it, cut to ragged sizes."""
    from dcreg_b200.scenes import make_parking_frames
    frames, T_true, T_init, tgt = make_parking_frames(12, seed=71, n_map=300_000, n_scan=6_000)
    corners = np.array([[-60, -60, -6], [60, 60, 5], [-60, 60, 5], [60, -60, -6]], dtype=np.float32)
    B = np.ascontiguousarray(np.concatenate([tgt, corners]))
    A = np.ascontiguousarray(np.concatenate([B, FAR]))
    rng = np.random.default_rng(72)
    sizes = [5_000, 40, 4_000, 256, 3_333, 6_000, 999, 4_097, 2_500, 5_555, 300, 4_444]
    cut = [f[np.sort(rng.choice(len(f), size=min(n, len(f)), replace=False))] for f, n in zip(frames, sizes)]
    return cut, T_true, T_init, A, B


def box_cells(xyz, cell):
    lo = np.floor(xyz.astype(np.float64).min(axis=0) / cell)
    hi = np.floor(xyz.astype(np.float64).max(axis=0) / cell)
    return float(np.prod(hi - lo + 1))


def assert_identical(x, y):
    assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
    assert x.T.tobytes() == y.T.tobytes()
    assert len(x.logs) == len(y.logs)
    assert [log_bytes(L) for L in x.logs] == [log_bytes(L) for L in y.logs]
    for f in ("cov", "T_prior"):
        a, b = getattr(x, f, None), getattr(y, f, None)
        assert (a is None) == (b is None)
        if a is not None:
            assert np.asarray(a).tobytes() == np.asarray(b).tobytes()


def test_scene_is_what_the_tests_need(scene):
    frames, _, T_init, A, B = scene
    assert box_cells(B, RADIUS) <= 2 ** 27 < box_cells(A, RADIUS)
    lo = np.floor(B.astype(np.float64).min(axis=0) / RADIUS)
    hi = np.floor(B.astype(np.float64).max(axis=0) / RADIUS)
    for f, T in zip(frames, T_init):                      # every query cell under its initial pose lies in B's box
        q = (f.astype(np.float64) @ T[:3, :3].T + T[:3, 3]).astype(np.float32)
        c = np.floor(q.astype(np.float64) / RADIUS)
        assert np.all(c >= lo) and np.all(c <= hi)


def test_under_the_limit_it_is_set_target(ctx, scene):
    """A box of at most 2^27 cells: the same launches and the same results as dcreg_set_target."""
    frames, _, T_init, _, B = scene
    prm = params()
    ctx.set_source(frames[0])
    n0 = ctx.launch_count
    ctx.set_target(B, RADIUS)
    n_dense = ctx.launch_count - n0
    r_dense = ctx.icp_run(prm, T_init[0])
    p_dense, n_pt_dense = ctx.find_planes(T_init[0], RADIUS)
    n0 = ctx.launch_count
    ctx.set_target_sparse(B, RADIUS)
    assert ctx.launch_count - n0 == n_dense
    r = ctx.icp_run(prm, T_init[0])
    assert_identical(r, r_dense)
    p, n_pt = ctx.find_planes(T_init[0], RADIUS)
    assert p.tobytes() == p_dense.tobytes() and n_pt == n_pt_dense
    m = ctx.point_to_point_metrics(r.T, 0.1)                # a dense grid: the metrics work
    assert m["n_valid"] > 0


def test_find_planes_sparse_equals_dense(ctx, scene):
    frames, _, T_init, A, B = scene
    out = {}
    for name, tgt in (("B", B), ("A", A)):
        ctx.set_target_sparse(tgt, RADIUS)
        ctx.set_source(frames[2])
        out[name] = ctx.find_planes(T_init[2], RADIUS)
    assert out["A"][0].tobytes() == out["B"][0].tobytes()
    assert out["A"][1] == out["B"][1] > 1000


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_every_call_sparse_equals_dense(ctx, scene, method):
    """icp_run (with its log), enqueue / fetch, _batch, _scans and _sequences on A equal the same calls on B bit for bit;
    on A from set_target they equal those on A from set_target_sparse, after a build of the same launches."""
    from dcreg_b200.scenes import trial_poses
    frames, _, T_init, A, B = scene
    prm = params(method)
    trials = T_init[3] @ trial_poses(6, seed=73, max_trans=0.2, max_rot_deg=1.0)
    seqs = [frames[0:4], frames[4:8], frames[8:12]]
    deltas = np.array([np.linalg.inv(T_init[k]) @ T_init[min(k + 1, 11)] for k in range(12)])
    out, builds = {}, {}
    for name, tgt, build in (("B", B, ctx.set_target), ("A", A, ctx.set_target_sparse), ("A2", A, ctx.set_target)):
        n0 = ctx.launch_count
        build(tgt, RADIUS)
        builds[name] = ctx.launch_count - n0
        ctx.set_source(frames[3])
        r = dict(single=ctx.icp_run(prm, T_init[3]))
        ctx.icp_enqueue(prm, T_init[3])
        r["fetch"] = ctx.icp_fetch()
        r["batch"] = ctx.icp_run_batch(prm, trials, want_log=True)
        r["scans"] = ctx.icp_run_scans(prm, frames, T_init, want_log=True, want_cov=True)
        r["seqs"] = ctx.icp_run_sequences(prm, seqs, T_init[[0, 4, 8]], deltas, want_log=True, want_cov=True)
        out[name] = r
    a, b = out["A"], out["B"]
    assert_identical(a["single"], b["single"])
    assert a["fetch"].T.tobytes() == b["fetch"].T.tobytes() == b["single"].T.tobytes()
    assert (a["fetch"].iterations, a["fetch"].converged) == (b["fetch"].iterations, b["fetch"].converged)
    for k in ("batch", "scans", "seqs"):
        assert len(a[k]) == len(b[k])
        for x, y in zip(a[k], b[k]):
            assert_identical(x, y)
    assert sum(int(x.converged) for x in b["scans"]) >= 8     # the runs do real work
    assert b["single"].iterations > 2
    a2 = out["A2"]
    assert builds["A2"] == builds["A"]
    assert_identical(a2["single"], a["single"])
    assert a2["fetch"].T.tobytes() == a["fetch"].T.tobytes()
    assert (a2["fetch"].iterations, a2["fetch"].converged) == (a["fetch"].iterations, a["fetch"].converged)
    for k in ("batch", "scans", "seqs"):
        assert len(a2[k]) == len(a[k])
        for x, y in zip(a2[k], a[k]):
            assert_identical(x, y)


def test_bad_arguments(ctx, scene):
    from dcreg_b200.api import BAD_ARG, DcregError
    frames, _, T_init, A, _ = scene
    lib, h = ctx.lib, ctx._h
    fp = A.ctypes.data_as(C.POINTER(C.c_float))
    for args in ((None, len(A), 3, RADIUS), (fp, 0, 3, RADIUS), (fp, len(A), 2, RADIUS), (fp, len(A), 3, 0.0),
                 (fp, len(A), 3, float("nan"))):
        assert lib.dcreg_set_target_sparse(h, *args) == BAD_ARG
        assert "dcreg_set_target_sparse: empty cloud" in lib.dcreg_last_error(h).decode()
    assert lib.dcreg_set_target_sparse(None, fp, len(A), 3, RADIUS) == BAD_ARG
    huge = np.concatenate([A[:1000], np.array([[1e9, 0, 0]], dtype=np.float32)])
    with pytest.raises(DcregError) as e:
        ctx.set_target_sparse(huge, RADIUS)
    assert e.value.status == BAD_ARG
    assert "grid build: coordinates / cell_size exceed the +-2^19 cell range" in str(e.value)
    ctx.set_target_sparse(A, RADIUS)
    ctx.set_source(frames[0])
    with pytest.raises(DcregError) as e:
        ctx.point_to_point_metrics(T_init[0], 0.1)
    assert e.value.status == BAD_ARG and "sparse row index" in str(e.value)


@pytest.fixture(scope="module")
def large():
    """The 4 x 4 tile map at 100 k points per tile (1.6 M points, 2.7e8 cells of box at 0.5 m) and 32 frames, two per
    tile."""
    from dcreg_b200.scenes import make_large_map, make_large_map_frames
    tgt, _ = make_large_map(n_map=100_000)
    frames, T_true, T_init, tile = make_large_map_frames(32, n_map=100_000, n_scan=4_000)
    return tgt, frames, T_true, T_init, tile


def test_large_map_batches_equal_single_runs(ctx, large):
    tgt, frames, T_true, T_init, tile = large
    assert box_cells(tgt, RADIUS) > 2 ** 27
    prm = params()
    ctx.set_target_sparse(tgt, RADIUS)
    scans = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    order = np.argsort(tile, kind="stable")                  # one sequence per tile, its frames in path order
    seqs = [[frames[k] for k in order[2 * t:2 * t + 2]] for t in range(16)]
    deltas = np.array([np.linalg.inv(T_true[k]) @ T_true[order[min(i + 1, 31)]] for i, k in enumerate(order)])
    seq = ctx.icp_run_sequences(prm, seqs, T_init[order[::2]], deltas, want_log=True)
    n_ok = 0
    for k, b in enumerate(scans):
        ctx.set_source(frames[k])
        single = ctx.icp_run(prm, T_init[k])
        assert (b.status, b.iterations, b.converged) == (single.status, single.iterations, single.converged)
        assert o.se3_log_distance(single.T, b.T) < 1e-8
        for x, y in zip(b.logs, single.logs):
            assert x.n_effective == y.n_effective and x.n_corr_pt == y.n_corr_pt
            assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)
        n_ok += int(b.converged and o.se3_log_distance(T_true[k], b.T) < 0.05)
    assert n_ok >= 24
    for i, (k, f) in enumerate(zip(order, seq)):
        ctx.set_source(frames[k])
        single = ctx.icp_run(prm, f.T_prior)
        assert (f.status, f.iterations, f.converged) == (single.status, single.iterations, single.converged)
        assert o.se3_log_distance(single.T, f.T) < 1e-8
        for x, y in zip(f.logs, single.logs):
            assert x.n_effective == y.n_effective and x.n_corr_pt == y.n_corr_pt
            assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)
    again = ctx.icp_run_scans(prm, frames, T_init, want_log=True)
    for x, y in zip(scans, again):
        assert_identical(x, y)
    seq2 = ctx.icp_run_sequences(prm, seqs, T_init[order[::2]], deltas, want_log=True)
    for x, y in zip(seq, seq2):
        assert_identical(x, y)
