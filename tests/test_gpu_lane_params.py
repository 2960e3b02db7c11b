"""Per-lane solver settings (dcreg_set_lane_params): one batched call whose lanes run different methods or thresholds.

Contract 1: lane b returns byte for byte what the same call returns for lane b when every entry is a copy of entry b
(T_out, T_prior, iterations, converged, status, cov, n_points, metrics, search_radius and every log record with
iter_time_ms zeroed).  Contract 2: identical entries are the call with one params, launches included.
"""
import numpy as np
import pytest

from harness import METHODS, RADIUS, ctx, log_bytes, params, read_csv, write_config  # noqa: F401

pytestmark = pytest.mark.gpu

CELL = 0.5
LENS = (1, 7, 12)


def kappa(k, method="Ours", radius=RADIUS):
    return params(method, radius, cond_thresh=k, kappa_target=k)


def assert_same(a, b, where):
    assert (a.status, a.iterations, a.converged) == (b.status, b.iterations, b.converged), where
    assert a.T.tobytes() == b.T.tobytes(), where
    for name in ("T_prior", "cov", "n_points", "search_radius", "metrics"):
        x, y = getattr(a, name, None), getattr(b, name, None)
        if isinstance(x, np.ndarray):
            assert x.tobytes() == y.tobytes(), (where, name)
        else:
            assert x == y, (where, name)
    assert [log_bytes(x) for x in a.logs] == [log_bytes(y) for y in b.logs], where


def lanes_vs_uniform(run, entries, lane_of=None):
    """run(params) -> results; every result k of the per-lane call equals result k of the call whose entries all are
    entry lane_of[k] (k's own lane without lane_of)"""
    got = run(list(entries))
    refs = {}
    for k, r in enumerate(got):
        b = k if lane_of is None else lane_of[k]
        key = bytes(entries[b])
        if key not in refs:
            refs[key] = run([entries[b]] * len(entries))
        assert_same(r, refs[key][k], (k, b))
    assert len(refs) > 1
    return got


# ---- the cylinder of the G2 setup: batches of trials and scans ----------------------------------------------------
@pytest.fixture(scope="module")
def g2_trials(cylinder):
    """the shipped cylinder and 12 trial poses about the G2 setup's initial pose"""
    from dcreg_b200.scenes import g2_initial_pose, trial_poses
    return cylinder, g2_initial_pose() @ trial_poses(12, seed=5, max_trans=0.3, max_rot_deg=2.0)


def g2(method, **over):
    return params(method, radius=1.0, use_weight_derivative=1, **over)


def test_batch_mixes_all_six_methods(ctx, g2_trials):
    pts, T = g2_trials
    ctx.set_source(pts)
    ctx.set_target(pts, 1.0)
    names = list(METHODS)
    entries = [g2(names[k % 6], kappa_target=1.0 + k) for k in range(len(T))]
    lanes_vs_uniform(lambda p: ctx.icp_run_batch(p, T, want_log=True), entries)


def test_identical_entries_are_the_uniform_call(ctx, g2_trials):
    """Contract 2: the same bytes and the same launch count, for "Ours" (folded) and a baseline (K2)"""
    pts, T = g2_trials
    ctx.set_source(pts)
    ctx.set_target(pts, 1.0)
    for method in ("Ours", "ME-SR"):
        p = g2(method)
        n0 = ctx.launch_count
        one = ctx.icp_run_batch(p, T, want_log=True)
        n1 = ctx.launch_count
        many = ctx.icp_run_batch([p] * len(T), T, want_log=True)
        n2 = ctx.launch_count
        assert n1 - n0 == n2 - n1
        for k, (a, b) in enumerate(zip(one, many)):
            assert_same(a, b, (method, k))


def test_swapped_mixes_at_one_shape(ctx, g2_trials):
    """Calls of one shape whose lanes are all "Ours" (no K2 launch) and then mixed (a K2 launch after every iteration
    kernel, at the same kernel arguments), with swapped mixes: each equals its uniform references (the loop's graph key
    covers whether a K2 launch follows, so a mixed call never replays the all-"Ours" call's graph)"""
    pts, T = g2_trials
    ctx.set_source(pts)
    ctx.set_target(pts, 1.0)
    a = [g2("Ours" if k % 2 else "ME-TSVD") for k in range(len(T))]
    b = [g2("ME-TSVD" if k % 2 else "Ours") for k in range(len(T))]
    c = [g2("Ours", kappa_target=2.0 + k) for k in range(len(T))]
    for entries in (c, a, c, b, a):
        lanes_vs_uniform(lambda p: ctx.icp_run_batch(p, T, want_log=True), entries)
        again = ctx.icp_run_batch(entries, T, want_log=True)              # contract 3
        for k, (x, y) in enumerate(zip(ctx.icp_run_batch(entries, T, want_log=True), again)):
            assert_same(x, y, k)


def test_scans(ctx):
    from dcreg_b200.scenes import make_parking_frames
    scans, _, T_init, tgt = make_parking_frames(6, n_map=200_000, n_scan=4_000)
    ctx.set_target(tgt, RADIUS)
    entries = [params(m) for m in ("Ours", "ME-TSVD", "Ours", "FCN-SR", "NONE", "ME-TReg")]
    entries[2] = kappa(100.0)
    lanes_vs_uniform(lambda p: ctx.icp_run_scans(p, scans, T_init, want_log=True, want_cov=True), entries)


def test_pairs_with_metrics(ctx):
    from dcreg_b200.scenes import make_parking_pairs
    src, tgt, _, T_init = make_parking_pairs(5, n_map=200_000, n_scan=3_000)
    entries = [params("Ours"), params("ME-SR"), kappa(3.0), params("ME-TSVD"), kappa(300.0)]
    lanes_vs_uniform(lambda p: ctx.icp_run_pairs(p, src, tgt, T_init, want_log=True, want_cov=True,
                                                 metrics_threshold=0.1), entries)


# ---- sequences and odometry ------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def odo():
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, tgt = make_parking_sequence(20, seed=71, n_scan=20_000, max_range=20.0)
    bounds = np.concatenate([[0], np.cumsum(LENS)])
    seqs = [list(frames[a:b]) for a, b in zip(bounds[:-1], bounds[1:])]
    return seqs, np.ascontiguousarray(T_true[bounds[:-1]]), deltas, tgt


def frame_seq(seqs):
    return [s for s, q in enumerate(seqs) for _ in q]


@pytest.fixture(scope="module")
def mixes():
    """per-lane entries of the sequence, odometry and session tests"""
    return {"kappa": [kappa(2.0), kappa(30.0), kappa(1000.0)],
            "methods": [params("ME-TSVD"), kappa(50.0), params("FCN-SR")]}


def test_sequences(ctx, odo, mixes):
    seqs, T_init, deltas, tgt = odo
    ctx.set_target(tgt, RADIUS)
    for entries in mixes.values():
        lanes_vs_uniform(lambda p: ctx.icp_run_sequences(p, seqs, T_init, deltas, want_log=True, want_cov=True), entries,
                         frame_seq(seqs))


@pytest.mark.parametrize("mix", ["kappa", "methods"])
@pytest.mark.parametrize("kind", ["window", "voxel_map", "adaptive"])
def test_odometry(ctx, odo, mixes, kind, mix):
    from dcreg_b200.api import AdaptiveThreshold
    seqs, T_init, deltas, _ = odo
    entries = mixes[mix]
    if kind == "window":
        def run(p):
            return ctx.icp_run_odometry(p, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True,
                                        want_cov=True)
    elif kind == "voxel_map":
        def run(p):
            return ctx.icp_run_odometry_map(p, seqs, T_init, deltas, map_voxel=0.25, max_distance=30.0, cell_size=CELL,
                                            want_log=True, want_cov=True)
    else:
        def run(p):
            return ctx.icp_run_odometry(p, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True,
                                        adaptive=AdaptiveThreshold(initial_threshold=0.4, min_motion=0.05,
                                                                   max_range=20.0))
    lanes_vs_uniform(run, entries, frame_seq(seqs))


RAGGED = [[1, 2, 0], [0, 0, 5], [0, 3, 1], [0, 2, 6]]


def pushed(ctx, sess, seqs, deltas, between=None):
    """The recording pushed in RAGGED chunks; between(i) runs before push i.  Returns the results in frame order."""
    first = np.concatenate([[0], np.cumsum(LENS)])
    done = [0, 0, 0]
    got = [[] for _ in seqs]
    for i, cnt in enumerate(RAGGED):
        part = [seqs[s][done[s]:done[s] + c] for s, c in enumerate(cnt)]
        D = np.concatenate([deltas[first[s] + done[s]:first[s] + done[s] + c] for s, c in enumerate(cnt)])
        if between:
            between(i)
        for s, r in enumerate(sess.push(part, D, want_log=True)):
            got[s].extend(r)
        done = [d + c for d, c in zip(done, cnt)]
    return [r for q in got for r in q]


def test_session_ragged_pushes_equal_one_call(ctx, odo, mixes):
    seqs, T_init, deltas, _ = odo
    entries = mixes["methods"]
    ref = ctx.icp_run_odometry(entries, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    with ctx.odometry_session(entries, 3, T_init, map_frames=3, cell_size=CELL) as sess:
        flat = pushed(ctx, sess, seqs, deltas)
    for k, (a, b) in enumerate(zip(flat, ref)):
        assert_same(a, b, k)


def test_session_keeps_its_setting(ctx, odo, mixes):
    """A session opened with the setting on keeps its per-lane entries when the setting goes off and on again between
    pushes, and one opened with it off keeps its one params when it goes on (the library reads no array at a push)"""
    seqs, T_init, deltas, _ = odo
    entries = mixes["kappa"]
    ref = ctx.icp_run_odometry(entries, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    ctx.set_lane_params(True)
    try:
        with ctx.odometry_session(entries, 3, T_init, map_frames=3, cell_size=CELL) as sess:
            assert ctx._lane_params                                   # the open left the caller's setting on
            flat = pushed(ctx, sess, seqs, deltas, between=lambda i: ctx.set_lane_params(i % 2 == 0))
    finally:
        ctx.set_lane_params(False)
    for k, (a, b) in enumerate(zip(flat, ref)):
        assert_same(a, b, k)
    one = ctx.icp_run_odometry(entries[1], seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True)
    try:
        with ctx.odometry_session(entries[1], 3, T_init, map_frames=3, cell_size=CELL) as sess:
            flat = pushed(ctx, sess, seqs, deltas, between=lambda i: ctx.set_lane_params(i % 2 == 1))
    finally:
        ctx.set_lane_params(False)
    for k, (a, b) in enumerate(zip(flat, one)):
        assert_same(a, b, k)


# ---- refusals and single runs ----------------------------------------------------------------------------------------
COMMON = {"search_radius": 0.6, "max_iterations": 29, "fixed_iterations": 1, "use_weight_derivative": 2,
          "plane_thickness": 0.3, "weight_slope": 0.8, "weight_gate": 0.2, "min_normal_norm": 1e-5}


def test_common_fields_refused(ctx, g2_trials, odo):
    from dcreg_b200 import DcregError
    pts, T = g2_trials
    seqs, T_init, deltas, _ = odo
    ctx.set_source(pts)
    ctx.set_target(pts, 1.0)
    ref = ctx.icp_run_batch(g2("Ours"), T[:3])
    for field, value in COMMON.items():
        entries = [g2("Ours"), g2("ME-SR"), g2("Ours")]
        setattr(entries[2], field, value)
        with pytest.raises(DcregError) as e:
            ctx.icp_run_batch(entries, T[:3])
        assert "icp_run_batch: entry 2: " + field in str(e.value)
        with pytest.raises(DcregError) as e:
            ctx.odometry_session([params(), params(), params(**{field: value})], 3, T_init, map_frames=3, cell_size=CELL)
        assert "entry 2: " + field in str(e.value)
    assert not ctx._lane_params
    for a, b in zip(ctx.icp_run_batch(g2("Ours"), T[:3]), ref):              # the context is still usable
        assert_same(a, b, "after")
    with ctx.odometry_session([params(), kappa(3.0), params()], 3, T_init, map_frames=3, cell_size=CELL) as sess:
        bad = [params(), params(), params(weight_gate=0.3)]
        with pytest.raises(DcregError):
            ctx.icp_run_odometry(bad, seqs, T_init, deltas, map_frames=3, cell_size=CELL)
        assert len(sess.push([[seqs[0][0]], [], []])[0]) == 1                  # the session too
    with pytest.raises(ValueError):
        ctx.icp_run_batch([g2("Ours")] * 2, T[:3])
    h = ctx._h
    assert ctx.lib.dcreg_set_lane_params(h, 2) != 0
    assert "enable must be 0 or 1" in ctx.lib.dcreg_last_error(h).decode()


def test_single_runs_read_entry_zero(ctx, g2_trials):
    """With the setting on, dcreg_icp_run, _enqueue and dcreg_analyze_and_solve given an array whose later entries
    differ (another method, an invalid iteration count) return what they return for entry 0 alone"""
    import ctypes as C
    from dcreg_b200.api import Analysis, IcpParams, IterLog
    pts, T = g2_trials
    ctx.set_source(pts)
    ctx.set_target(pts, 1.0)
    lib, h = ctx.lib, ctx._h
    p0 = g2("Ours")
    arr = (IcpParams * 3)(p0, g2("ME-SR", max_iterations=-1), g2("NONE", weight_gate=2.0))
    dp = C.POINTER(C.c_double)

    def run(params):
        T_in = np.ascontiguousarray(T[0]); T_out = np.empty((4, 4))
        logs = (IterLog * 30)(); n_it = C.c_int(0); conv = C.c_int(0)
        rc = lib.dcreg_icp_run(h, params, T_in.ctypes.data_as(dp), T_out.ctypes.data_as(dp), logs, 30, C.byref(n_it),
                               C.byref(conv))
        return rc, T_out.tobytes(), n_it.value, conv.value, [log_bytes(logs[i]) for i in range(min(n_it.value, 30))]

    def enqueue(params):
        T_in = np.ascontiguousarray(T[1]); T_out = np.empty((4, 4)); n_it = C.c_int(0); conv = C.c_int(0)
        rc = lib.dcreg_icp_enqueue(h, params, T_in.ctypes.data_as(dp))
        return rc, lib.dcreg_icp_fetch(h, T_out.ctypes.data_as(dp), C.byref(n_it), C.byref(conv)), T_out.tobytes(), n_it.value

    H27 = np.ascontiguousarray(ctx.icp_run(p0, T[0]).logs[0].H27)

    def solve(params):
        a = Analysis(); dx = np.empty(6)
        rc = lib.dcreg_analyze_and_solve(h, H27.ctypes.data_as(dp), params, C.byref(a), dx.ctypes.data_as(dp))
        return rc, bytes(a), dx.tobytes()

    ref = [f(C.byref(p0)) for f in (run, enqueue, solve)]
    ctx.set_lane_params(True)
    try:
        got = [f(arr) for f in (run, enqueue, solve)]
    finally:
        ctx.set_lane_params(False)
    assert ref[0][0] == 0 and ref[0][2] > 1
    assert got == ref


def test_cli_one_call_csvs(golden, tmp_path):
    """The CLI's monte_carlo.one_call: the six recognised methods x trials as one batched call write the same files as
    one call per method: the same drawn poses, iterations, flags and status, poses to 1e-8 (the call's shape differs,
    so its FP64 grouping does), and a summary whose Trials/s counts every lane of the one call"""
    import subprocess
    from dcreg_b200 import build as b
    runner = b.build_runner()
    names = ["Ours", "ME-SR", "FCN-SR", "ME-TSVD", "ME-TReg"]
    mc = "monte_carlo:\n  trials: 40\n  seed: 13\n  max_trans_m: 0.6\n  max_rot_deg: 2.0\n"
    dirs = {}
    for one in (False, True):
        out_dir = tmp_path / ("one" if one else "per_method")
        cfg = tmp_path / f"icp_{int(one)}.yaml"
        write_config(cfg, out_dir, golden["G2"]["setup"], names, extra_methods='  "NONE": [ "NONE_DETE", "NONE_HAND" ]',
                     extra=mc + ("  one_call: true\n" if one else ""))
        res = subprocess.run([runner, str(cfg)], capture_output=True, text=True, timeout=600)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
        dirs[one] = out_dir
    for m in names + ["NONE"]:
        a, c = read_csv(dirs[False] / f"monte_carlo_{m}.csv"), read_csv(dirs[True] / f"monte_carlo_{m}.csv")
        assert len(a) == len(c) == 40
        assert list(a[0]) == list(c[0])
        for i, (x, y) in enumerate(zip(a, c)):
            for col in ("Trial", "Init_x", "Init_y", "Init_z", "Init_roll_deg", "Init_pitch_deg", "Init_yaw_deg",
                        "Converged", "Iterations", "Status"):
                assert x[col] == y[col], (m, i, col)
            Tx = np.array([float(x[f"T{k // 4}{k % 4}"]) for k in range(12)])
            Ty = np.array([float(y[f"T{k // 4}{k % 4}"]) for k in range(12)])
            assert np.abs(Tx - Ty).max() < 1e-8, (m, i)
    rows = {}
    for one in (False, True):
        lines = (dirs[one] / "monte_carlo_summary.txt").read_text().splitlines()
        rows[one] = {ln.split()[0]: ln.split() for ln in lines[3:] if ln.strip()}
    assert sorted(rows[True]) == sorted(names + ["NONE"]) == sorted(rows[False])
    times = {r[-2] for r in rows[True].values()}
    assert len(times) == 1                                                  # Time(ms): the one call's, on every row
    ms = float(times.pop())
    for r in rows[True].values():
        assert abs(float(r[-1]) * ms / 1000.0 - 6 * 40) < 0.5               # Trials/s over all 240 lanes (both rounded)
    for m in rows[True]:                                                    # converged %, failures, mean iterations
        assert [rows[True][m][k] for k in (1, 2, 7)] == [rows[False][m][k] for k in (1, 2, 7)], m
