"""The voxel filter on the device: dcreg_voxel_downsample against its NumPy twin, and dcreg_icp_run_odometry_voxel, scan-to-
map odometry with voxel-filtered frames and local maps.

Every registered frame of a filtered call is checked against its reconstruction with the twin: the frame's source is
voxel_downsample(frame k, source_voxel), its map voxel_downsample(concatenation of map_points(T_out[j], filtered frame
j) over the window, map_voxel), then set_target + set_source + icp_run(T_prior[k]) with the tolerances of
tests/test_gpu_odometry.py."""
import numpy as np
import pytest

from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, assert_anchor, assert_priors, clouds_of_every_case, parking,  # noqa: F401
                          raw_downsample, raw_odometry, reconstruct, split)

pytestmark = pytest.mark.gpu

SV, MV = 0.3, 0.25            # source and map voxel sizes of the tests
VOXEL = "dcreg_icp_run_odometry_voxel"
FIRST = "dcreg_voxel_downsample"


@pytest.fixture(scope="module")
def odo():
    """20 frames of about 20 k points of one path with drifting odometry, in sequences of 1, 7 and 12 frames."""
    seqs, T_init, deltas, frames, T_true = parking()
    return seqs, frames, T_init, deltas, T_true


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
    rc, pts, kept, idx = raw_downsample(ctx, FIRST, c4, voxel, stride=4)
    assert rc == 0
    for b, c in enumerate(clouds):
        tp, ti = voxel_downsample(c, voxel)
        assert pts[kept[b]:kept[b + 1]].tobytes() == tp.tobytes() and np.array_equal(idx[kept[b]:kept[b + 1]], ti)
    rc, pts2, kept2, _ = raw_downsample(ctx, FIRST, c4, voxel, stride=4, want_index=False)
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
    rc, _, _, _ = raw_downsample(ctx, FIRST, far, 0.25)                      # 1.2e6 voxels > 2^20
    assert rc == api.BAD_ARG and "cloud 1" in ctx.lib.dcreg_last_error(ctx._h).decode()
    with pytest.raises(ValueError):
        api.voxel_downsample(far[1], 0.25)
    assert raw_downsample(ctx, FIRST, far, 1.0)[0] == api.OK
    launches = ctx.launch_count
    for v in (0.0, -0.5, np.nan, np.inf):
        assert raw_downsample(ctx, FIRST, good, v)[0] == api.BAD_ARG, v
    assert raw_downsample(ctx, FIRST, good, 0.5, stride=2)[0] == api.BAD_ARG
    assert raw_downsample(ctx, FIRST, [good[0], good[0][:0], good[1]], 0.5)[0] == api.BAD_ARG      # an empty cloud
    with pytest.raises(api.DcregError) as e:
        ctx.voxel_downsample([], 0.5)
    assert e.value.status == api.BAD_ARG
    assert ctx.launch_count == launches
    assert ctx.voxel_downsample(good, 0.5)[1][1].tolist() == [0]             # the context stays usable


def test_zero_voxels_are_the_existing_call(ctx, odo):
    """(0, 0): the same launches and the same bytes in every output as dcreg_icp_run_odometry."""
    seqs, _, T_init, deltas, _ = odo
    prm = params()
    a0 = ctx.launch_count
    rc_a, a = raw_odometry(ctx, "dcreg_icp_run_odometry", prm, seqs, T_init, deltas, log_cap=30)
    a1 = ctx.launch_count
    rc_b, b = raw_odometry(ctx, VOXEL, prm, seqs, T_init, deltas, source_voxel=0.0, map_voxel=0.0, log_cap=30)
    assert ctx.launch_count - a1 == a1 - a0
    assert rc_a == rc_b == 0
    for k in ("T_prior", "T_out", "n_it", "conv", "st", "cov", "log"):
        assert a[k].tobytes() == b[k].tobytes(), k
    assert b["npts"].tolist() == [len(f) for s in seqs for f in s]
    res = ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL)
    assert [r.n_points for r in res] == b["npts"].tolist()
    assert all(r.T.tobytes() == T.tobytes() for r, T in zip(res, a["T_out"]))


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
    rc_a, a = raw_odometry(ctx, VOXEL, prm, seqs, T_init, deltas, source_voxel=SV, map_voxel=MV, log_cap=30)
    rc_b, b = raw_odometry(ctx, VOXEL, prm, seqs, T_init, deltas, source_voxel=SV, map_voxel=MV, log_cap=30)
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
            entry, sizes = (VOXEL, dict(source_voxel=SV, map_voxel=MV)) if vox else ("dcreg_icp_run_odometry", {})
            rc, _ = raw_odometry(ctx, entry, prm, ss, T0, None, **sizes)
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
        rc, _ = raw_odometry(ctx, VOXEL, prm, [seq], T0, D, source_voxel=vox[0], map_voxel=vox[1])
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
    rc, out = raw_odometry(ctx, VOXEL, prm, [seq], T0, D_far, source_voxel=0.0, map_voxel=MV)
    msg = ctx.lib.dcreg_last_error(ctx._h).decode()
    assert rc == api.BAD_ARG and "sequence 0" in msg and "frame 4" in msg and "voxel" in msg, msg
    assert all(out["n_it"][k] >= 0 for k in range(4)) and out["n_it"][1] > 0
    assert out["n_it"][4] == -1 and out["n_it"][5] == -1 and np.all(out["T_out"][4:] == -1.0)
    assert out["st"][3] == api.NOT_ENOUGH_POINTS and out["T_out"][3, 0, 3] > 5e5
    rc, good = raw_odometry(ctx, VOXEL, prm, [seq], T0, D, source_voxel=SV, map_voxel=MV)
    assert rc == api.OK
    from dcreg_b200 import Context
    with Context(0) as fresh:
        rc, ref = raw_odometry(fresh, VOXEL, prm, [seq], T0, D, source_voxel=SV, map_voxel=MV)
        assert rc == api.OK
        for k in good:
            assert good[k].tobytes() == ref[k].tobytes(), k
