"""The capped voxel filter on the device: dcreg_voxel_downsample_n against its NumPy twin, and
dcreg_icp_run_odometry_voxel_n, scan-to-map odometry whose frame and map filters keep up to N points per voxel.

Every registered frame of a capped call is checked against its reconstruction with the twin, as in
tests/test_gpu_voxel.py: the frame's source is voxel_downsample(frame k, source_voxel, source_max_points), its map
voxel_downsample(concatenation of map_points(T_out[j], filtered frame j) over the window, map_voxel, map_max_points)."""
import numpy as np
import pytest

from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, assert_anchor, assert_priors, crowded_clouds, parking, raw_downsample,  # noqa: F401
                          raw_odometry, reconstruct, split, window_map)

pytestmark = pytest.mark.gpu

SV, MV = 0.3, 0.25            # source and map voxel sizes of the tests
VOXEL_N = "dcreg_icp_run_odometry_voxel_n"
CAPPED = "dcreg_voxel_downsample_n"


def capped(voxels, caps):
    """The filter settings of raw_odometry(VOXEL_N, ...) for voxel sizes (source, map) and caps (source, map)"""
    return dict(source_voxel=voxels[0], map_voxel=voxels[1], source_max_points=caps[0], map_max_points=caps[1])


@pytest.fixture(scope="module")
def odo():
    """20 frames of about 20 k points of one path with drifting odometry, in sequences of 1, 7 and 12 frames."""
    seqs, T_init, deltas, frames, T_true = parking()
    return seqs, frames, T_init, deltas, T_true


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
        rc, pts, kept, idx = raw_downsample(ctx, CAPPED, c4, voxel, stride=stride, max_points=max_points)
        assert rc == 0
        assert_equals_twin(pts, kept, idx, clouds, voxel, max_points)
    rc, pts2, kept2, _ = raw_downsample(ctx, CAPPED, c4, voxel, stride=4, want_index=False, max_points=max_points)
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
        a = raw_downsample(ctx, "dcreg_voxel_downsample", c, voxel, stride=stride)
        a1 = ctx.launch_count
        b = raw_downsample(ctx, CAPPED, c, voxel, stride=stride, max_points=1)
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


@pytest.mark.parametrize("voxels", [(SV, MV), (0.0, 0.0)], ids=["filtered", "unfiltered"])
def test_one_point_caps_are_the_voxel_call(ctx, odo, voxels):
    """(sv, 1, mv, 1): the same launches and the same bytes in every output as dcreg_icp_run_odometry_voxel(sv, mv)."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    a0 = ctx.launch_count
    rc_a, a = raw_odometry(ctx, "dcreg_icp_run_odometry_voxel", prm, seqs, T_init, deltas, source_voxel=voxels[0],
                           map_voxel=voxels[1], log_cap=30)
    a1 = ctx.launch_count
    rc_b, b = raw_odometry(ctx, VOXEL_N, prm, seqs, T_init, deltas, log_cap=30, **capped(voxels, (1, 1)))
    assert ctx.launch_count - a1 == a1 - a0
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k


def test_unreached_map_cap_is_the_unfiltered_map(ctx, odo):
    """A map cap above every voxel's occupancy keeps the whole map in order: the outputs of (sv, 0)."""
    from dcreg_b200.api import voxel_downsample
    seqs, frames, T_init, deltas, _ = odo
    prm = params()
    rc_a, a = raw_odometry(ctx, "dcreg_icp_run_odometry_voxel", prm, seqs, T_init, deltas, source_voxel=SV,
                           map_voxel=0.0, log_cap=30)
    rc_b, b = raw_odometry(ctx, VOXEL_N, prm, seqs, T_init, deltas, log_cap=30, **capped((SV, MV), (1, 1 << 30)))
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
        M = window_map(seq, rs, k, 3, SV, 0.0, (1, 1))
        assert voxel_downsample(M, MV, 1 << 30)[0].tobytes() == M.tobytes()


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
    rc_a, a = raw_odometry(ctx, VOXEL_N, prm, seqs, T_init, deltas, log_cap=30, **capped((SV, MV), (2, 8)))
    rc_b, b = raw_odometry(ctx, VOXEL_N, prm, seqs, T_init, deltas, log_cap=30, **capped((SV, MV), (2, 8)))
    assert rc_a == rc_b == 0
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    again = ctx.icp_run(prm, T_true[1])
    assert again.T.tobytes() == one.T.tobytes() and again.iterations == one.iterations
    assert [np.array(L.H27).tobytes() for L in again.logs] == [np.array(L.H27).tobytes() for L in one.logs]
    from dcreg_b200 import Context
    with Context(0) as fresh:                                                  # a fresh context: the same bytes
        rc, ref = raw_odometry(fresh, VOXEL_N, prm, seqs, T_init, deltas, log_cap=30, **capped((SV, MV), (2, 8)))
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
            rc, _ = raw_odometry(ctx, VOXEL_N, prm, ss, T0, None, **capped((SV, MV), caps))
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
            assert raw_downsample(ctx, CAPPED, good, v, max_points=n)[0] == api.BAD_ARG, (v, n)
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
            rc, out = raw_odometry(ctx, VOXEL_N, prm, [seq], T0, D, **capped(voxel, caps))
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
    rc, out = raw_odometry(ctx, VOXEL_N, prm, [seq], T0, D_far, **capped((0.0, MV), (1, 6)))
    msg = ctx.lib.dcreg_last_error(ctx._h).decode()
    assert rc == api.BAD_ARG and "frame 4" in msg and "voxel" in msg, msg
    assert all(out["n_it"][k] >= 0 for k in range(4)) and out["n_it"][4] == -1
    assert ctx.voxel_downsample(good, 0.5, 2)[1][1].tolist() == [0, 1]      # the context stays usable
