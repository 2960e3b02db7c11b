"""The capped voxel filter on the device: dcreg_voxel_downsample_n against its NumPy twin, and
dcreg_icp_run_odometry_voxel_n, scan-to-map odometry whose frame and map filters keep up to N points per voxel.

Every registered frame of a capped call is checked against its reconstruction with the twin, as in
tests/test_gpu_voxel.py: the frame's source is voxel_downsample(frame k, source_voxel, source_max_points), its map
voxel_downsample(concatenation of map_points(T_out[j], filtered frame j) over the window, map_voxel, map_max_points)."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_odometry import CELL, assert_anchor, assert_priors, assert_same_run, params, split
from test_gpu_voxel import clouds_of_every_case, raw_downsample, raw_odometry

pytestmark = pytest.mark.gpu

SV, MV = 0.3, 0.25            # source and map voxel sizes of the tests
dp = C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def odo():
    """20 frames of about 20 k points of one path with drifting odometry, in sequences of 1, 7 and 12 frames."""
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(20, seed=71, n_scan=20_000, max_range=20.0)
    bounds = [0, 1, 8, 20]
    seqs = [frames[a:b] for a, b in zip(bounds[:-1], bounds[1:])]
    return seqs, frames, T_true[bounds[:-1]], deltas, T_true


def crowded_clouds():
    """The clouds of test_gpu_voxel plus a cloud with one voxel holding 6000 points, interleaved with a sparse
    background and repeated at its end"""
    rng = np.random.default_rng(31)
    crowd = rng.uniform(0.01, 0.24, (6000, 3)).astype(np.float32)
    background = rng.uniform(-30, 30, (3000, 3)).astype(np.float32)
    crowded = np.concatenate([rng.permutation(np.concatenate([crowd, background])), crowd])
    return clouds_of_every_case() + [crowded]


def raw_downsample_n(ctx, clouds, voxel, max_points, stride=3, want_index=True):
    """dcreg_voxel_downsample_n on (N_b, stride) clouds: (rc, points, offsets, index)"""
    xyz = np.ascontiguousarray(np.concatenate([np.asarray(c, np.float32)[:, :stride] for c in clouds]), dtype=np.float32)
    off = np.zeros(len(clouds) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.empty((max(len(xyz), 1), 3), np.float32)
    kept = np.zeros(len(clouds) + 1, np.int64)
    idx = np.empty(max(len(xyz), 1), np.int64)
    rc = ctx.lib.dcreg_voxel_downsample_n(ctx._h, len(clouds), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                                          off.ctypes.data_as(C.POINTER(C.c_int64)), stride, float(voxel), int(max_points),
                                          pts.ctypes.data_as(C.POINTER(C.c_float)),
                                          kept.ctypes.data_as(C.POINTER(C.c_int64)),
                                          idx.ctypes.data_as(C.POINTER(C.c_int64)) if want_index else None)
    return rc, pts, kept, idx


def assert_equals_twin(pts, kept, idx, clouds, voxel, max_points):
    from dcreg_b200.api import voxel_downsample
    at = 0
    for b, c in enumerate(clouds):
        tp, ti = voxel_downsample(c, voxel, max_points)
        assert kept[b] == at, b
        at += len(ti)
        assert pts[kept[b]:kept[b + 1]].tobytes() == tp.tobytes() and np.array_equal(idx[kept[b]:kept[b + 1]], ti), b
    assert kept[-1] == at


@pytest.mark.parametrize("max_points", [2, 3, 20])
@pytest.mark.parametrize("voxel", [0.25, 1.0])
def test_capped_downsample_equals_twin(ctx, voxel, max_points):
    from dcreg_b200.api import voxel_downsample
    clouds = crowded_clouds()
    got = ctx.voxel_downsample(clouds, voxel, max_points)
    assert len(got) == len(clouds)
    for (p, i), c in zip(got, clouds):
        tp, ti = voxel_downsample(c, voxel, max_points)
        assert p.tobytes() == tp.tobytes() and np.array_equal(i, ti)
    # the raw call at strides 3 and 4 (xyzi), offsets and indices included; without the index output
    rng = np.random.default_rng(32)
    c4 = [np.concatenate([c, rng.uniform(0, 1, (len(c), 1)).astype(np.float32)], axis=1) for c in clouds]
    for stride in (3, 4):
        rc, pts, kept, idx = raw_downsample_n(ctx, c4, voxel, max_points, stride=stride)
        assert rc == 0
        assert_equals_twin(pts, kept, idx, clouds, voxel, max_points)
    rc, pts2, kept2, _ = raw_downsample_n(ctx, c4, voxel, max_points, stride=4, want_index=False)
    assert rc == 0 and np.array_equal(kept2, kept) and pts2[:kept[-1]].tobytes() == pts[:kept[-1]].tobytes()


def test_crowded_voxel_keeps_its_first_points(ctx):
    clouds = crowded_clouds()
    for n in (2, 20, 5999, 6000, 1 << 20):
        (p, i), = ctx.voxel_downsample(clouds[-1:], 0.25, n)
        crowd = (np.floor(clouds[-1].astype(np.float64) * 4.0) == 0).all(axis=1)
        rows = np.nonzero(crowd)[0]
        assert np.array_equal(i[np.isin(i, rows)], rows[:n])


def test_one_point_cap_is_the_first_point_call(ctx):
    clouds = crowded_clouds()
    for stride, voxel in ((3, 0.25), (4, 1.0)):
        c = [np.concatenate([x, np.ones((len(x), 1), np.float32)], axis=1) for x in clouds]
        a0 = ctx.launch_count
        a = raw_downsample(ctx, c, voxel, stride=stride)
        a1 = ctx.launch_count
        b = raw_downsample_n(ctx, c, voxel, 1, stride=stride)
        assert ctx.launch_count - a1 == a1 - a0
        assert a[0] == b[0] == 0
        kept = a[2]
        assert kept.tobytes() == b[2].tobytes()
        for x, y in ((a[1], b[1]), (a[3], b[3])):                             # the rows written: kept[-1] of them
            assert x[:kept[-1]].tobytes() == y[:kept[-1]].tobytes()


def test_capped_downsample_launches_do_not_grow_with_clouds(ctx):
    clouds = crowded_clouds()
    a = ctx.launch_count
    ctx.voxel_downsample(clouds[:1], 0.5, 4)
    b = ctx.launch_count
    ctx.voxel_downsample(clouds * 8, 0.5, 4)
    assert ctx.launch_count - b == b - a == 7


def raw_odometry_n(ctx, prm, seqs, T_init, deltas, voxel, caps, map_frames=3, motion=0, log_cap=0):
    """dcreg_icp_run_odometry_voxel_n with every output: (rc, dict of output arrays) as raw_odometry gives them"""
    from dcreg_b200 import api
    frames = [f for s in seqs for f in s]
    n = len(frames)
    xyz = np.ascontiguousarray(np.concatenate(frames), dtype=np.float32)
    off = np.zeros(n + 1, np.int64); off[1:] = np.cumsum([len(f) for f in frames])
    so = np.zeros(len(seqs) + 1, np.int32); so[1:] = np.cumsum([len(s) for s in seqs])
    out = dict(T_prior=np.full((n, 4, 4), -1.0), T_out=np.full((n, 4, 4), -1.0), n_it=np.full(n, -1, np.int32),
               conv=np.full(n, -1, np.int32), st=np.full(n, -1, np.int32), cov=np.full((n, 36), -1.0),
               npts=np.full(n, -1, np.int64), log=np.zeros(max(n * log_cap, 1) * C.sizeof(api.IterLog), np.uint8))
    T0 = np.ascontiguousarray(T_init, dtype=np.float64)
    D = None if deltas is None else np.ascontiguousarray(deltas, dtype=np.float64)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))                       # noqa: E731
    rc = ctx.lib.dcreg_icp_run_odometry_voxel_n(
        ctx._h, C.byref(prm), len(seqs), ip(so), n, xyz.ctypes.data_as(C.POINTER(C.c_float)),
        off.ctypes.data_as(C.POINTER(C.c_int64)), 3, CELL, map_frames, motion, float(voxel[0]), float(voxel[1]),
        int(caps[0]), int(caps[1]), T0.ctypes.data_as(dp), D.ctypes.data_as(dp) if D is not None else None,
        out["npts"].ctypes.data_as(C.POINTER(C.c_int64)), out["T_prior"].ctypes.data_as(dp),
        out["T_out"].ctypes.data_as(dp), ip(out["n_it"]), ip(out["conv"]), ip(out["st"]), out["cov"].ctypes.data_as(dp),
        C.cast(out["log"].ctypes.data, C.POINTER(api.IterLog)) if log_cap else None, log_cap)
    for rec in (api.IterLog * (n * log_cap)).from_buffer(out["log"]):
        rec.iter_time_ms = 0.0                                                 # a device clock reading: differs per run
    return rc, out


@pytest.mark.parametrize("voxels", [(SV, MV), (0.0, 0.0)], ids=["filtered", "unfiltered"])
def test_one_point_caps_are_the_voxel_call(ctx, odo, voxels):
    """(sv, 1, mv, 1): the same launches and the same bytes in every output as dcreg_icp_run_odometry_voxel(sv, mv)."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    a0 = ctx.launch_count
    rc_a, a = raw_odometry(ctx, prm, seqs, T_init, deltas, voxel=voxels, log_cap=30)
    a1 = ctx.launch_count
    rc_b, b = raw_odometry_n(ctx, prm, seqs, T_init, deltas, voxels, (1, 1), log_cap=30)
    assert ctx.launch_count - a1 == a1 - a0
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_unreached_map_cap_is_the_unfiltered_map(ctx, odo):
    """A map cap above every voxel's occupancy keeps the whole map in order: the outputs of (sv, 0)."""
    from dcreg_b200.api import voxel_downsample
    seqs, frames, T_init, deltas, _ = odo
    prm = params()
    rc_a, a = raw_odometry(ctx, prm, seqs, T_init, deltas, voxel=(SV, 0.0), log_cap=30)
    rc_b, b = raw_odometry_n(ctx, prm, seqs, T_init, deltas, (SV, MV), (1, 1 << 30), log_cap=30)
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    # the twin's kept map is the unfiltered map, point for point (every step of the long sequence)
    seq = seqs[2]
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, source_voxel=SV,
                               map_voxel=MV, map_max_points=1 << 30)
    rs = split(res, seqs)[2]
    assert all(r.T.tobytes() == T.tobytes() for r, T in zip(res, b["T_out"]))
    for k in range(1, len(seq)):
        M = filtered_map(seq, rs, k, 3, SV, 0.0, (1, 1))
        assert voxel_downsample(M, MV, 1 << 30)[0].tobytes() == M.tobytes()


def filtered_map(seq, res_seq, k, map_frames, sv, mv, caps):
    from dcreg_b200.api import map_points, voxel_downsample
    fs = (lambda P: voxel_downsample(P, sv, caps[0])[0]) if sv else (lambda P: P)
    M = np.concatenate([map_points(res_seq[j].T, fs(seq[j])) for j in range(max(0, k - map_frames), k)])
    return voxel_downsample(M, mv, caps[1])[0] if mv else M


def reconstruct(ctx, prm, seq, res_seq, k, map_frames, sv, mv, caps):
    from dcreg_b200.api import voxel_downsample
    ctx.set_target(filtered_map(seq, res_seq, k, map_frames, sv, mv, caps), CELL)
    ctx.set_source(voxel_downsample(seq[k], sv, caps[0])[0] if sv else seq[k])
    return ctx.icp_run(prm, res_seq[k].T_prior)


@pytest.mark.parametrize("caps", [(1, 4), (3, 4)], ids=["map", "both"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_capped_frames_equal_their_reconstruction(ctx, odo, method, caps):
    from dcreg_b200.api import voxel_downsample
    seqs, frames, T_init, deltas, _ = odo
    prm = params(method)
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, want_cov=True,
                               source_voxel=SV, map_voxel=MV, source_max_points=caps[0], map_max_points=caps[1])
    assert len(res) == len(frames)
    assert [r.n_points for r in res] == [len(voxel_downsample(f, SV, caps[0])[1]) for f in frames]
    assert_priors(res, seqs, T_init, deltas)
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        for k in range(1, len(seq)):
            assert_same_run(rs[k], reconstruct(ctx, prm, seq, rs, k, 3, SV, MV, caps))


def test_capped_reproducible_and_context_intact(ctx, odo):
    seqs, frames, T_init, deltas, T_true = odo
    prm = params()
    ctx.set_target(np.concatenate(frames[:3]), CELL)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_true[1])
    rc_a, a = raw_odometry_n(ctx, prm, seqs, T_init, deltas, (SV, MV), (2, 8), log_cap=30)
    rc_b, b = raw_odometry_n(ctx, prm, seqs, T_init, deltas, (SV, MV), (2, 8), log_cap=30)
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    again = ctx.icp_run(prm, T_true[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]
    from dcreg_b200 import Context
    with Context(0) as fresh:                                                  # a fresh context: the same bytes
        rc, ref = raw_odometry_n(fresh, prm, seqs, T_init, deltas, (SV, MV), (2, 8), log_cap=30)
        assert rc == 0
        for k in a:
            assert a[k].tobytes() == ref[k].tobytes(), k


def test_capped_launches_per_step_do_not_depend_on_sequences(ctx, odo):
    """Fixed iteration counts make every step's loop the same; the capped filters then add the same launches to a call
    of one sequence as to a call of three."""
    seqs, _, T_init, _, _ = odo
    prm = params(fixed_iterations=1, max_iterations=3)
    one = [seqs[2][:6]]
    three = [seqs[1][:6], seqs[2][:6], seqs[2][6:12]]
    T3 = np.stack([T_init[1], T_init[2], T_init[2]])
    counts = {}
    for name, ss, T0 in (("one", one, T_init[2:3]), ("three", three, T3)):
        for caps in ((1, 1), (2, 4)):
            a = ctx.launch_count
            rc, _ = raw_odometry_n(ctx, prm, ss, T0, None, (SV, MV), caps)
            assert rc == 0
            counts[name, caps] = ctx.launch_count - a
    assert counts["one", (1, 1)] == counts["three", (1, 1)] and counts["one", (2, 4)] == counts["three", (2, 4)]
    assert counts["one", (2, 4)] - counts["one", (1, 1)] == 6        # one more launch per filter: the frames', 5 maps'


def test_capped_bad_arguments(ctx, odo):
    from dcreg_b200 import api
    seqs, _, T_init, deltas, _ = odo
    good = [np.zeros((3, 3), np.float32), np.ones((2, 3), np.float32)]
    launches = ctx.launch_count
    for n in (0, -1, -(1 << 31)):
        for v in (0.5, 0.0):                                                   # rejected whatever the voxel size
            assert raw_downsample_n(ctx, good, v, n)[0] == api.BAD_ARG, (v, n)
            assert "max_points" in ctx.lib.dcreg_last_error(ctx._h).decode()
    for bad in (0, -3, 2.5, True):
        with pytest.raises(ValueError):
            ctx.voxel_downsample(good, 0.5, bad)
    prm = params()
    seq = [f[:3000] for f in seqs[2][:6]]
    T0 = T_init[2:3]
    D = deltas[8:14]
    for voxel in ((SV, MV), (0.0, 0.0)):
        for caps in ((0, 1), (1, 0), (-2, 4), (4, -2)):
            rc, out = raw_odometry_n(ctx, prm, [seq], T0, D, voxel, caps)
            assert rc == api.BAD_ARG, (voxel, caps)
            assert "max_points" in ctx.lib.dcreg_last_error(ctx._h).decode()
            assert np.all(out["n_it"] == -1)
    for kw in (dict(source_max_points=0), dict(map_max_points=-1), dict(map_max_points=2.0)):
        with pytest.raises(ValueError):
            ctx.icp_run_odometry(prm, [seq], T0, D, map_frames=3, cell_size=CELL, map_voxel=MV, **kw)
    assert ctx.launch_count == launches                                        # nothing launched
    # the voxel range is checked with a cap as without: a source frame outside it, and a map that leaves it
    s2 = list(seq)
    s2[3] = np.array([[0.0, 0.0, 0.0], [4.0e5, 0.0, 0.0]], np.float32)
    with pytest.raises(api.DcregError) as e:
        ctx.icp_run_odometry(prm, [s2], T0, D, map_frames=3, cell_size=CELL, source_voxel=SV, source_max_points=5)
    assert e.value.status == api.BAD_ARG and "frame 3" in str(e.value) and "outside" in str(e.value)
    D_far = D.copy()
    D_far[2, 0, 3] += 1.0e6
    rc, out = raw_odometry_n(ctx, prm, [seq], T0, D_far, (0.0, MV), (1, 6))
    msg = ctx.lib.dcreg_last_error(ctx._h).decode()
    assert rc == api.BAD_ARG and "frame 4" in msg and "voxel" in msg, msg
    assert all(out["n_it"][k] >= 0 for k in range(4)) and out["n_it"][4] == -1
    assert ctx.voxel_downsample(good, 0.5, 2)[1][1].tolist() == [0, 1]      # the context stays usable
