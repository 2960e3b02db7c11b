"""The voxel filter on the device: dcreg_voxel_downsample against its NumPy twin, and dcreg_icp_run_odometry_voxel, scan-to-
map odometry with voxel-filtered frames and local maps.

Every registered frame of a filtered call is checked against its reconstruction with the twin: the frame's source is
voxel_downsample(frame k, source_voxel), its map voxel_downsample(concatenation of map_points(T_out[j], filtered frame
j) over the window, map_voxel), then set_target + set_source + icp_run(T_prior[k]) with the tolerances of
tests/test_gpu_odometry.py."""
import ctypes as C

import numpy as np
import pytest

from test_gpu_odometry import CELL, assert_anchor, assert_priors, assert_same_run, params, split

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


def clouds_of_every_case():
    rng = np.random.default_rng(11)
    g = np.arange(-5, 5, dtype=np.float64) * 0.25
    lattice = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    lattice = np.concatenate([lattice, np.nextafter(lattice, np.float32(-np.inf))])
    dup = rng.uniform(-3, 3, (300, 3)).astype(np.float32)
    holes = rng.uniform(-3, 3, (700, 3)).astype(np.float32)
    holes[::5, 0] = np.nan
    holes[2::9, 1] = np.inf
    holes[4::13, 2] = -np.inf
    return [rng.standard_normal((5000, 3)).astype(np.float32) * 4, lattice, np.concatenate([dup, dup, dup[::-1]]), holes,
            np.array([[-0.1, 0.2, -0.3]], np.float32), (rng.standard_normal((20000, 3)) * 30).astype(np.float32)]


def raw_downsample(ctx, clouds, voxel, stride=3, want_index=True):
    """dcreg_voxel_downsample on (N_b, stride) clouds: (rc, points, offsets, index)"""
    xyz = np.ascontiguousarray(np.concatenate([np.asarray(c, np.float32)[:, :stride] for c in clouds]), dtype=np.float32)
    off = np.zeros(len(clouds) + 1, np.int64)
    off[1:] = np.cumsum([len(c) for c in clouds])
    pts = np.empty((max(len(xyz), 1), 3), np.float32)
    kept = np.zeros(len(clouds) + 1, np.int64)
    idx = np.empty(max(len(xyz), 1), np.int64)
    rc = ctx.lib.dcreg_voxel_downsample(ctx._h, len(clouds), xyz.ctypes.data_as(C.POINTER(C.c_float)),
                                        off.ctypes.data_as(C.POINTER(C.c_int64)), stride, float(voxel),
                                        pts.ctypes.data_as(C.POINTER(C.c_float)), kept.ctypes.data_as(C.POINTER(C.c_int64)),
                                        idx.ctypes.data_as(C.POINTER(C.c_int64)) if want_index else None)
    return rc, pts, kept, idx


@pytest.mark.parametrize("voxel", [0.1, 0.25, 1.0])
def test_downsample_equals_twin(ctx, voxel):
    from dcreg_b200.api import voxel_downsample
    clouds = clouds_of_every_case()
    got = ctx.voxel_downsample(clouds, voxel)
    assert len(got) == len(clouds)
    for (p, i), c in zip(got, clouds):
        tp, ti = voxel_downsample(c, voxel)
        assert p.tobytes() == tp.tobytes() and np.array_equal(i, ti)
    # stride 4 (xyzi), the same selection; without the index output
    rng = np.random.default_rng(12)
    c4 = [np.concatenate([c, rng.uniform(0, 1, (len(c), 1)).astype(np.float32)], axis=1) for c in clouds]
    rc, pts, kept, idx = raw_downsample(ctx, c4, voxel, stride=4)
    assert rc == 0
    for b, c in enumerate(clouds):
        tp, ti = voxel_downsample(c, voxel)
        assert pts[kept[b]:kept[b + 1]].tobytes() == tp.tobytes() and np.array_equal(idx[kept[b]:kept[b + 1]], ti)
    rc, pts2, kept2, _ = raw_downsample(ctx, c4, voxel, stride=4, want_index=False)
    assert rc == 0 and np.array_equal(kept2, kept) and pts2[:kept[-1]].tobytes() == pts[:kept[-1]].tobytes()


def test_downsample_launches_do_not_grow_with_clouds(ctx):
    clouds = clouds_of_every_case()
    a = ctx.launch_count
    ctx.voxel_downsample(clouds[:1], 0.5)
    b = ctx.launch_count
    ctx.voxel_downsample(clouds * 8, 0.5)
    assert ctx.launch_count - b == b - a


def test_downsample_bad_arguments(ctx):
    from dcreg_b200 import api
    good = [np.zeros((3, 3), np.float32), np.ones((2, 3), np.float32)]
    far = [good[0], np.array([[0.0, 0.0, 0.0], [3.0e5, 0.0, 0.0]], np.float32)]
    rc, _, _, _ = raw_downsample(ctx, far, 0.25)                             # 1.2e6 voxels > 2^20
    assert rc == api.BAD_ARG and "cloud 1" in ctx.lib.dcreg_last_error(ctx._h).decode()
    with pytest.raises(ValueError):
        api.voxel_downsample(far[1], 0.25)
    assert raw_downsample(ctx, far, 1.0)[0] == api.OK
    launches = ctx.launch_count
    for v in (0.0, -0.5, np.nan, np.inf):
        assert raw_downsample(ctx, good, v)[0] == api.BAD_ARG, v
    assert raw_downsample(ctx, good, 0.5, stride=2)[0] == api.BAD_ARG
    assert raw_downsample(ctx, [good[0], good[0][:0], good[1]], 0.5)[0] == api.BAD_ARG       # an empty cloud
    with pytest.raises(api.DcregError) as e:
        ctx.voxel_downsample([], 0.5)
    assert e.value.status == api.BAD_ARG
    assert ctx.launch_count == launches
    assert ctx.voxel_downsample(good, 0.5)[1][1].tolist() == [0]             # the context stays usable


def raw_odometry(ctx, prm, seqs, T_init, deltas, map_frames=3, voxel=None, motion=0, log_cap=0):
    """dcreg_icp_run_odometry (voxel None) or dcreg_icp_run_odometry_voxel (voxel = (source, map)) with every output:
    (rc, dict of output arrays)"""
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
    head = (ctx._h, C.byref(prm), len(seqs), ip(so), n, xyz.ctypes.data_as(C.POINTER(C.c_float)),
            off.ctypes.data_as(C.POINTER(C.c_int64)), 3, CELL, map_frames, motion)
    tail = (out["T_prior"].ctypes.data_as(dp), out["T_out"].ctypes.data_as(dp), ip(out["n_it"]), ip(out["conv"]),
            ip(out["st"]), out["cov"].ctypes.data_as(dp),
            C.cast(out["log"].ctypes.data, C.POINTER(api.IterLog)) if log_cap else None,
            log_cap)
    Dp = D.ctypes.data_as(dp) if D is not None else None
    if voxel is None:
        rc = ctx.lib.dcreg_icp_run_odometry(*head, T0.ctypes.data_as(dp), Dp, *tail)
    else:
        rc = ctx.lib.dcreg_icp_run_odometry_voxel(*head, float(voxel[0]), float(voxel[1]), T0.ctypes.data_as(dp), Dp,
                                                  out["npts"].ctypes.data_as(C.POINTER(C.c_int64)), *tail)
    for rec in (api.IterLog * (n * log_cap)).from_buffer(out["log"]):
        rec.iter_time_ms = 0.0                                                 # a device clock reading: differs per run
    return rc, out


def test_zero_voxels_are_the_existing_call(ctx, odo):
    """(0, 0): the same launches and the same bytes in every output as dcreg_icp_run_odometry."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    a0 = ctx.launch_count
    rc_a, a = raw_odometry(ctx, prm, seqs, T_init, deltas, log_cap=30)
    a1 = ctx.launch_count
    rc_b, b = raw_odometry(ctx, prm, seqs, T_init, deltas, voxel=(0.0, 0.0), log_cap=30)
    assert ctx.launch_count - a1 == a1 - a0
    assert rc_a == rc_b == 0
    for k in ("T_prior", "T_out", "n_it", "conv", "st", "cov", "log"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert b["npts"].tolist() == [len(f) for s in seqs for f in s]
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL)
    assert [r.n_points for r in res] == b["npts"].tolist()
    assert all(r.T.tobytes() == T.tobytes() for r, T in zip(res, a["T_out"]))


def filtered_map(seq, res_seq, k, map_frames, sv, mv):
    from dcreg_b200.api import map_points, voxel_downsample
    fs = (lambda P: voxel_downsample(P, sv)[0]) if sv else (lambda P: P)
    M = np.concatenate([map_points(res_seq[j].T, fs(seq[j])) for j in range(max(0, k - map_frames), k)])
    return voxel_downsample(M, mv)[0] if mv else M


def reconstruct(ctx, prm, seq, res_seq, k, map_frames, sv, mv):
    from dcreg_b200.api import voxel_downsample
    ctx.set_target(filtered_map(seq, res_seq, k, map_frames, sv, mv), CELL)
    ctx.set_source(voxel_downsample(seq[k], sv)[0] if sv else seq[k])
    return ctx.icp_run(prm, res_seq[k].T_prior)


@pytest.mark.parametrize("voxels", [(SV, 0.0), (0.0, MV), (SV, MV)], ids=["source", "map", "both"])
@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_filtered_frames_equal_their_reconstruction(ctx, odo, method, voxels):
    from dcreg_b200.api import voxel_downsample
    seqs, frames, T_init, deltas, _ = odo
    sv, mv = voxels
    prm = params(method)
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, want_log=True, want_cov=True,
                               source_voxel=sv, map_voxel=mv)
    assert len(res) == len(frames)
    assert [r.n_points for r in res] == [len(voxel_downsample(f, sv)[1]) if sv else len(f) for f in frames]
    assert_priors(res, seqs, T_init, deltas)
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        for k in range(1, len(seq)):
            assert_same_run(rs[k], reconstruct(ctx, prm, seq, rs, k, 3, sv, mv))


def test_constant_velocity_with_filters(ctx, odo):
    seqs, _, T_init, _, _ = odo
    prm = params()
    short = [s[:5] for s in seqs]
    res = ctx.icp_run_odometry(prm, short, T_init, motion="constant_velocity", map_frames=4, cell_size=CELL,
                               source_voxel=SV, map_voxel=MV)
    assert_priors(res, short, T_init, None, motion="constant_velocity")
    rs = split(res, short)[2]
    for k in (1, 2, 4):
        assert_same_run(rs[k], reconstruct(ctx, prm, short[2], rs, k, 4, SV, MV), logs=False)


def test_filtered_reproducible_and_context_intact(ctx, odo):
    seqs, frames, T_init, deltas, T_true = odo
    prm = params()
    ctx.set_target(np.concatenate(frames[:3]), CELL)
    ctx.set_source(frames[1])
    one = ctx.icp_run(prm, T_true[1])
    rc_a, a = raw_odometry(ctx, prm, seqs, T_init, deltas, voxel=(SV, MV), log_cap=30)
    rc_b, b = raw_odometry(ctx, prm, seqs, T_init, deltas, voxel=(SV, MV), log_cap=30)
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    again = ctx.icp_run(prm, T_true[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]


def test_launches_per_step_do_not_depend_on_sequences(ctx, odo):
    """Fixed iteration counts make every step's loop the same; the filters then add the same launches to a call of one
    sequence as to a call of three."""
    seqs, _, T_init, deltas, _ = odo
    prm = params(fixed_iterations=1, max_iterations=3)
    one = [seqs[2][:6]]
    three = [seqs[1][:6], seqs[2][:6], seqs[2][6:12]]
    T3 = np.stack([T_init[1], T_init[2], T_init[2]])
    counts = {}
    for name, ss, T0 in (("one", one, T_init[2:3]), ("three", three, T3)):
        for vox in (None, (SV, MV)):
            a = ctx.launch_count
            rc, _ = raw_odometry(ctx, prm, ss, T0, None, voxel=vox)
            assert rc == 0
            counts[name, vox] = ctx.launch_count - a
    assert counts["one", None] == counts["three", None] and counts["one", (SV, MV)] == counts["three", (SV, MV)]
    extra = counts["one", (SV, MV)] - counts["one", None]
    assert extra == counts["three", (SV, MV)] - counts["three", None]
    assert extra == 6 * 6                     # the frames' filter once, and each of the 5 steps' maps: 6 launches each


def test_filtered_odometry_bad_arguments(ctx, odo):
    from dcreg_b200 import api
    seqs, frames, T_init, deltas, _ = odo
    prm = params()
    seq = [f[:3000] for f in seqs[2][:6]]
    T0 = T_init[2:3]
    D = deltas[8:14]
    launches = ctx.launch_count
    for vox in ((-0.1, 0.0), (0.0, -1.0), (np.nan, 0.0), (0.0, np.inf)):
        rc, _ = raw_odometry(ctx, prm, [seq], T0, D, voxel=vox)
        assert rc == api.BAD_ARG, vox
        assert "voxel" in ctx.lib.dcreg_last_error(ctx._h).decode()
    assert ctx.launch_count == launches                                        # nothing launched
    # a frame with no finite point, and a frame outside the source filter's voxel range: found before the loop
    for bad_frame, why in ((np.full((50, 3), np.nan, np.float32), "no point"),
                           (np.array([[0.0, 0.0, 0.0], [4.0e5, 0.0, 0.0]], np.float32), "outside")):
        s2 = list(seq)
        s2[3] = bad_frame
        with pytest.raises(api.DcregError) as e:
            ctx.icp_run_odometry(prm, [seqs[0], s2], T_init[[0, 2]], np.concatenate([deltas[:1], D]), map_frames=3,
                                 cell_size=CELL, source_voxel=SV)
        msg = str(e.value)
        assert e.value.status == api.BAD_ARG and "sequence 1" in msg and "frame 4" in msg and why in msg, msg
    # the map leaves the map filter's voxel range at a later step: frame 3's prior is moved 1e6 m away, it aborts there,
    # and the map of frame 4 holds its points; frames 0 - 3 keep their outputs, the context stays usable
    D_far = D.copy()
    D_far[2, 0, 3] += 1.0e6
    rc, out = raw_odometry(ctx, prm, [seq], T0, D_far, voxel=(0.0, MV))
    msg = ctx.lib.dcreg_last_error(ctx._h).decode()
    assert rc == api.BAD_ARG and "sequence 0" in msg and "frame 4" in msg and "voxel" in msg, msg
    assert all(out["n_it"][k] >= 0 for k in range(4)) and out["n_it"][1] > 0
    assert out["n_it"][4] == -1 and out["n_it"][5] == -1 and np.all(out["T_out"][4:] == -1.0)
    assert out["st"][3] == api.NOT_ENOUGH_POINTS and out["T_out"][3, 0, 3] > 5e5
    rc, good = raw_odometry(ctx, prm, [seq], T0, D, voxel=(SV, MV))
    assert rc == api.OK
    from dcreg_b200 import Context
    with Context(0) as fresh:
        rc, ref = raw_odometry(fresh, prm, [seq], T0, D, voxel=(SV, MV))
        assert rc == api.OK
        for k in good:
            assert good[k].tobytes() == ref[k].tobytes(), k
