"""Scan-to-map odometry with the adaptive threshold (dcreg_icp_run_odometry_adaptive, dcreg_odometry_open_adaptive,
dcreg_odometry_push_adaptive): every frame's search radius follows its sequence's motion-model error on the device.

What is held: adaptive = NULL is the existing call, byte for byte and launch for launch; settings that keep every radius
at the ceiling give the existing call's bytes with one more launch per step; the returned radii follow the NumPy twin fed
with the call's own T_prior / T_out; every frame equals the single run set_target(map_k) + set_source(frame k) +
icp_run(T_prior[k]) at the radius the call RETURNED, also where the lanes of one step search different ring counts;
sessions equal the one call under any chunking, and a failed push leaves the threshold state as it was."""
import math

import numpy as np
import pytest

from harness import RADIUS, assert_same_run, ctx, params  # noqa: F401
from odom_harness import (CELL, RAGGED, assert_anchor, assert_priors, assert_same_flat, one_per_push,  # noqa: F401
                          parking, parking_sweeps, pushed, split, twin_maps, window_map)

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)
MV, DIST = 0.25, 10.0          # the voxel map's voxel and prune distance
CEILING = 2.0                  # four rings of cells: the ceiling of the tests whose radii move
MAPS = ["window", "voxel_map"]
C3_METHODS = ["Ours", "ME-TSVD"]
MAP_KW = {"window": dict(map_frames=3), "voxel_map": dict(map_voxel=MV, max_distance=DIST)}
# Under the 2 m ceiling with priors 0.3 to 0.6 m off, the first updates are far larger than with good priors at 0.5 m,
# and the solve passes the rounding of sums that agree to 1e-8 on in proportion (measured: 3e-7 of the update): a
# frame's steps may differ from its single run's by this fraction of the step; everything counted stays identical and
# the poses agree to 1e-8.
WIDE_STEPS = 1e-6


@pytest.fixture(scope="module")
def odo():
    """20 frames of one path (about 8 k points each, 20 m range) with drifting odometry, in sequences of 1, 7 and 12"""
    return parking(LENS, n_scan=8_000)[:3]


@pytest.fixture(scope="module")
def sweeps():
    """12 skewed sweeps with per-point timestamps in sequences of 5 and 7 frames (unskewed anchors)"""
    return parking_sweeps((5, 7), n_scan=8_000)


@pytest.fixture(scope="module")
def noisy():
    """Four sequences of 5 frames of one path whose increments are the true ones plus a translation error of a fixed
    size per sequence (0.03, 0.25, 0.42 and 0.6 m): under a ceiling of 2 m, with sigma starting at 2 / 3 m, their radii
    settle near three times those sizes, in four different rings of 0.5 m cells"""
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, _, _ = make_parking_sequence(20, seed=71, n_scan=6_000, max_range=20.0)
    rng = np.random.default_rng(9)
    deltas = np.empty((20, 4, 4))
    for k in range(20):
        D = np.linalg.inv(T_true[k]) @ T_true[min(k + 1, 19)]
        u = rng.normal(size=3) * [1.0, 1.0, 0.1]
        D[:3, 3] += u / np.linalg.norm(u) * (0.03, 0.25, 0.42, 0.6)[k // 5]
        deltas[k] = D
    seqs = [list(frames[a:a + 5]) for a in range(0, 20, 5)]
    return seqs, np.ascontiguousarray(T_true[0:20:5]), deltas


def threshold(*a):
    from dcreg_b200.api import AdaptiveThreshold
    return AdaptiveThreshold(*a)


def run(ctx, which, prm, seqs, T_init, deltas, **kw):
    kw.setdefault("want_log", True)
    kw.setdefault("want_cov", True)
    if which == "voxel_map":
        return ctx.icp_run_odometry_map(prm, seqs, T_init, deltas, map_voxel=MV, max_distance=DIST, cell_size=CELL, **kw)
    return ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=3, cell_size=CELL, **kw)


def open_session(ctx, which, prm, n_seqs, T_init, **kw):
    open_ = ctx.odometry_map_session if which == "voxel_map" else ctx.odometry_session
    return open_(prm, n_seqs, T_init, cell_size=CELL, **MAP_KW[which], **kw)


def counted(ctx, f):
    before = ctx.launch_count
    out = f()
    return out, ctx.launch_count - before


CONFIGS = [dict(), dict(motion="constant_velocity"), dict(source_voxel=0.3, map_max_points=4)]


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("method", C3_METHODS)
def test_null_is_the_existing_call(ctx, odo, sweeps, method, which):
    """adaptive = NULL: the bytes and the launches of dcreg_icp_run_odometry_deskew / _map; search_radius is the
    parameter's for every registered frame and 0 for the anchors"""
    seqs, T_init, deltas = odo
    prm = params(method)
    cases = [(seqs, T_init, deltas, kw) for kw in CONFIGS]
    sw = sweeps
    cases.append((sw["skewed"], sw["T_init"], sw["deltas"], dict(timestamps=sw["stamps"], want_deskewed=True, source_voxel=0.3)))
    for sq, T0, dl, kw in cases:
        D = None if kw.get("motion") == "constant_velocity" else dl
        ref, n_ref = counted(ctx, lambda: run(ctx, which, prm, sq, T0, D, **kw))
        got, n_got = counted(ctx, lambda: run(ctx, which, prm, sq, T0, D, want_radius=True, **kw))
        assert_same_flat(got, ref)
        assert n_got == n_ref
        for rs in split(got, sq):
            assert [r.search_radius for r in rs] == [0.0] + [RADIUS] * (len(rs) - 1)


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("method", C3_METHODS)
def test_radius_at_the_ceiling_gives_the_existing_bytes(ctx, odo, sweeps, method, which):
    """initial_threshold and min_motion at a third of the ceiling or more: sigma never falls below a third of it, every
    radius is the ceiling, and the outputs are the existing call's; the threshold kernel adds one launch per step"""
    seqs, T_init, deltas = odo
    prm = params(method)
    thr = threshold(RADIUS, RADIUS / 3.0, 100.0)
    cases = [(seqs, T_init, deltas, kw) for kw in CONFIGS]
    sw = sweeps
    cases.append((sw["skewed"], sw["T_init"], sw["deltas"], dict(timestamps=sw["stamps"], want_deskewed=True)))
    for sq, T0, dl, kw in cases:
        D = None if kw.get("motion") == "constant_velocity" else dl
        ref, n_ref = counted(ctx, lambda: run(ctx, which, prm, sq, T0, D, **kw))
        got, n_got = counted(ctx, lambda: run(ctx, which, prm, sq, T0, D, adaptive=thr, **kw))
        assert_same_flat(got, ref)
        assert n_got == n_ref + max(len(s) for s in sq) - 1
        for rs in split(got, sq):
            assert [r.search_radius for r in rs] == [0.0] + [RADIUS] * (len(rs) - 1)


def twin_radii(rs, thr, ceiling):
    """The twin's radii of one sequence, fed with the call's own priors and results; also the final state"""
    from dcreg_b200 import api
    state, out = (0.0, 0), [0.0]
    for r in rs[1:]:
        out.append(api.adaptive_threshold_radius(state, thr.initial_threshold, ceiling))
        state = api.adaptive_threshold_update(state, r.T_prior, r.T, thr.min_motion, thr.max_range)
    return out, state


def assert_radii_follow_twin(res, seqs, thr, ceiling, ulps=8):
    worst = 0.0
    for rs in split(res, seqs):
        want, _ = twin_radii(rs, thr, ceiling)
        assert rs[0].search_radius == 0.0
        for k in range(1, len(rs)):
            got = rs[k].search_radius
            assert 0.0 < got <= ceiling
            worst = max(worst, abs(got - want[k]) / np.spacing(want[k]))
    assert worst <= ulps, worst
    return worst


def reconstruct(ctx, which, method, seq, rs, k, frames=None, sv=0.0, cap=1, maps=None):
    """Frame k of a sequence as the single run at the radius the call returned"""
    from dcreg_b200.api import voxel_downsample
    assert rs[k].search_radius > 1e-6
    prm = params(method, search_radius=rs[k].search_radius)
    src = frames[k] if frames is not None else (voxel_downsample(seq[k], sv, 1)[0] if sv else seq[k])
    if which == "voxel_map":
        ctx.set_target(maps[k], CELL)
    else:
        fs = frames if frames is not None else [voxel_downsample(f, sv, 1)[0] if sv else f for f in seq]
        ctx.set_target(window_map(fs, rs, k, 3), CELL)
    ctx.set_source(src)
    return ctx.icp_run(prm, rs[k].T_prior)


def assert_reconstructions(ctx, which, method, res, seqs, T_init, sv=0.0, cap=1, deskewed=False, dx_rel=0.0):
    for s, (seq, rs) in enumerate(zip(seqs, split(res, seqs))):
        assert_anchor(rs[0], T_init[s])
        frames = [r.deskewed for r in rs] if deskewed else None
        maps = twin_maps(seq, rs, sv, MV, cap, DIST, frames=frames) if which == "voxel_map" else None
        for k in range(1, len(seq)):
            assert_same_run(rs[k], reconstruct(ctx, which, method, seq, rs, k, frames, sv, cap, maps), dx_rel=dx_rel)


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("method", C3_METHODS)
@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
def test_radii_follow_the_twin_and_frames_their_reconstruction(ctx, odo, method, which, motion):
    """Thresholds well under the ceiling: the radii move with the drifting odometry (or the constant-velocity model),
    follow the twin to a few ulp, and every frame is its single run at its returned radius"""
    seqs, T_init, deltas = odo
    D = deltas if motion == "increments" else None
    thr = threshold(0.12, 0.01, 20.0)
    res = run(ctx, which, params(method, search_radius=CEILING), seqs, T_init, D, motion=motion, adaptive=thr,
              map_max_points=4)
    assert_priors(res, seqs, T_init, D, motion)
    print("largest difference from the twin, in ulp of the radius:", assert_radii_follow_twin(res, seqs, thr, CEILING))
    # the radii do move (constant velocity predicts no motion for the first frame, 2.7 m off: soon at the ceiling)
    assert len({r.search_radius for r in res}) >= 4, sorted({r.search_radius for r in res})
    assert_reconstructions(ctx, which, method, res, seqs, T_init, cap=4, dx_rel=WIDE_STEPS)


@pytest.mark.parametrize("which", MAPS)
def test_timestamps_and_source_filter(ctx, sweeps, which):
    sw = sweeps
    thr = threshold(0.12, 0.01, 20.0)
    for method in C3_METHODS:
        res = run(ctx, which, params(method, search_radius=CEILING), sw["skewed"], sw["T_init"], sw["deltas"],
                  adaptive=thr, source_voxel=0.3, map_max_points=4, timestamps=sw["stamps"], want_deskewed=True)
        assert_radii_follow_twin(res, sw["skewed"], thr, CEILING)
        assert_reconstructions(ctx, which, method, res, sw["skewed"], sw["T_init"], sv=0.3, cap=4, deskewed=True,
                               dx_rel=WIDE_STEPS)


def rings(r):
    return max(1, math.ceil(r.search_radius / CELL - 1e-9))


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("method", C3_METHODS)
def test_lanes_of_one_step_search_different_ring_counts(ctx, noisy, method, which):
    """cell_size = ceiling / 4: the returned radii span all four ring counts, the lanes of a step differ in theirs (each
    lane's searches, the one-ring row tables included, key on the lane's own grid entry), and every frame is still its
    single run at its own radius"""
    seqs, T_init, deltas = noisy
    thr = threshold(2.0 / 3.0, 0.01, 20.0)
    prm = params(method, search_radius=2.0)
    res = run(ctx, which, prm, seqs, T_init, deltas, adaptive=thr, map_max_points=4)
    per_seq = split(res, seqs)
    seen = {rings(r) for r in res if r.search_radius > 0.0}
    # (the voxel map's first frames register against the anchor alone, pruned at 10 m: larger corrections, wider radii)
    assert seen == {1, 2, 3, 4} if which == "window" else len(seen) >= 2, [[rings(r) for r in rs] for rs in per_seq]
    assert all(rings(rs[1]) == 4 for rs in per_seq)                # sigma = 2 / 3 before any sample: the ceiling
    mixed = [k for k in range(2, 5) if len({rings(rs[k]) for rs in per_seq}) > 1]
    assert mixed
    if which == "window":                                           # ... next to one-ring lanes and their row tables
        assert any(1 in {rings(rs[k]) for rs in per_seq} for k in mixed)
    assert_radii_follow_twin(res, seqs, thr, 2.0)
    assert_reconstructions(ctx, which, method, res, seqs, T_init, cap=4, dx_rel=WIDE_STEPS)


def pushed_flat(ctx, which, prm, seqs, T_init, chunks, deltas, thr, stamps=None, **kw):
    """The recording pushed in chunks into a session with the threshold thr, with logs and covariances (deskewed points
    with stamps): one flat list of results"""
    res = pushed(ctx, prm, seqs, T_init, chunks, deltas, voxel_map=which == "voxel_map", stamps=stamps, want_log=True,
                 want_cov=True, want_deskewed=stamps is not None, adaptive=thr, **MAP_KW[which], **kw)
    return [r for rs in res for r in rs]


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
def test_chunkings_equal_one_call(ctx, odo, which, motion):
    """Three chunkings of the recording: the one call's bytes, search_radius included"""
    seqs, T_init, deltas = odo
    D = deltas if motion == "increments" else None
    thr = threshold(0.12, 0.01, 20.0)
    for method in C3_METHODS:
        prm = params(method, search_radius=CEILING)
        ref = run(ctx, which, prm, seqs, T_init, D, motion=motion, adaptive=thr, map_max_points=4)
        assert len({r.search_radius for r in ref}) >= 4
        for chunks in ([list(LENS)], one_per_push(LENS), RAGGED):
            got = pushed_flat(ctx, which, prm, seqs, T_init, chunks, D, thr, motion=motion, map_max_points=4)
            assert_same_flat(got, ref, radius=True)


@pytest.mark.parametrize("which", MAPS)
def test_mixed_deskew_and_plain_pushes(ctx, sweeps, which):
    """Pushes with and without timestamps: the one call whose frames of the plain pushes have every tau = 0.5"""
    sw = sweeps
    thr = threshold(0.12, 0.01, 20.0)
    prm = params(search_radius=CEILING)
    chunks = [[1, 1], [2, 2], [2, 4]]
    with_ts = lambda i: i != 1                                      # noqa: E731
    stamps = [[t if not 1 <= k < 3 else np.full_like(t, 0.5) for k, t in enumerate(ts)] for ts in sw["stamps"]]
    ref = run(ctx, which, prm, sw["skewed"], sw["T_init"], sw["deltas"], adaptive=thr, source_voxel=0.3,
              map_max_points=4, timestamps=stamps, want_deskewed=True)
    got = pushed_flat(ctx, which, prm, sw["skewed"], sw["T_init"], chunks, sw["deltas"], thr, stamps=sw["stamps"],
                      ts_push=with_ts, source_voxel=0.3, map_max_points=4)
    assert_same_flat(got, ref, radius=True)


@pytest.mark.parametrize("which", MAPS)
def test_failed_push_leaves_the_threshold_state(ctx, odo, which):
    """A push that fails at its second step (a far point enters that step's map) has already folded its first
    frame into the device's state; the session's committed state is untouched and the retry gives the one call's bytes"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    seq = [f[:6000] for f in seqs[2][:6]]
    # (the window's next map has no dense grid; the voxel map's next update has a voxel coordinate out of range)
    d = 3.0e4 if which == "window" else 1.0e6
    far = np.concatenate([seq[2], np.array([[d, d, 0.0]], np.float32)])
    thr = threshold(0.12, 0.01, 20.0)
    prm = params(search_radius=CEILING)
    ref = run(ctx, which, prm, [seq], T_init[2:3], deltas[8:14], adaptive=thr)
    with open_session(ctx, which, prm, 1, T_init[2:3], adaptive=thr) as sess:
        got = sess.push([seq[:2]], deltas[8:10], want_log=True, want_cov=True)[0]
        with pytest.raises(api.DcregError) as e:
            sess.push([[far, seq[3]]], deltas[10:12])
        assert e.value.status == api.BAD_ARG
        got += sess.push([seq[2:]], deltas[10:14], want_log=True, want_cov=True)[0]
    assert_same_flat(got, ref, radius=True)
    assert len({r.search_radius for r in ref}) > 3


def test_reproducible_and_context_untouched(ctx, odo):
    seqs, T_init, deltas = odo
    prm, wide = params(), params(search_radius=CEILING)
    thr = threshold(0.12, 0.01, 20.0)
    ctx.set_target(seqs[2][0], CELL)
    ctx.set_source(seqs[2][1])
    before = ctx.icp_run(prm, T_init[2])
    a = run(ctx, "window", wide, seqs, T_init, deltas, adaptive=thr)
    mid = ctx.icp_run(prm, T_init[2])
    b = run(ctx, "voxel_map", wide, seqs, T_init, deltas, adaptive=thr)
    a2 = run(ctx, "window", wide, seqs, T_init, deltas, adaptive=thr)
    b2 = run(ctx, "voxel_map", wide, seqs, T_init, deltas, adaptive=thr)
    after = ctx.icp_run(prm, T_init[2])
    assert_same_flat(a2, a, radius=True)
    assert_same_flat(b2, b, radius=True)
    for r in (mid, after):
        assert (r.status, r.iterations, r.converged) == (before.status, before.iterations, before.converged)
        assert r.T.tobytes() == before.T.tobytes()


@pytest.mark.parametrize("which", MAPS)
def test_launches_do_not_depend_on_the_number_of_sequences(ctx, odo, which):
    seqs, T_init, deltas = odo
    prm = params(fixed_iterations=1, max_iterations=4)
    thr = threshold(0.12, 0.01, 20.0)
    one = [seqs[1][:5]]
    three = [seqs[1][:5], seqs[2][:5], seqs[2][5:10]]
    T3 = np.stack([T_init[1], T_init[2], T_init[2]])
    run(ctx, which, prm, three, T3, None, adaptive=thr, want_log=False)         # buffers and graphs at their sizes
    _, n1 = counted(ctx, lambda: run(ctx, which, prm, one, T_init[1:2], None, adaptive=thr, want_log=False))
    _, n3 = counted(ctx, lambda: run(ctx, which, prm, three, T3, None, adaptive=thr, want_log=False))
    assert n1 == n3


def test_bad_settings(ctx, odo):
    """Each of the three settings not finite or out of range is BAD_ARG before anything is launched, in the one-shot call
    and at open; min_motion = 0 is allowed"""
    from dcreg_b200 import api
    seqs, T_init, deltas = odo
    prm = params()
    two = [seqs[1][:2]]
    bad = [(v, 0.1, 100.0) for v in (0.0, -1.0, math.nan, math.inf)]
    bad += [(2.0, v, 100.0) for v in (-0.1, math.nan, math.inf)]
    bad += [(2.0, 0.1, v) for v in (0.0, -5.0, math.nan, math.inf)]
    launches = ctx.launch_count
    for which in MAPS:
        for a in bad:
            with pytest.raises(api.DcregError) as e:
                run(ctx, which, prm, two, T_init[1:2], None, adaptive=threshold(*a))
            assert e.value.status == api.BAD_ARG and "adaptive" in str(e.value), a
            with pytest.raises(api.DcregError) as e:
                open_session(ctx, which, prm, 1, T_init[1:2], adaptive=threshold(*a))
            assert e.value.status == api.BAD_ARG, a
    assert ctx.launch_count == launches
    res = run(ctx, "window", prm, two, T_init[1:2], None, adaptive=threshold(0.12, 0.0, 20.0))
    assert res[1].search_radius == 3.0 * 0.12
    # the ceiling is still what the cell size is checked against
    with pytest.raises(api.DcregError):
        ctx.icp_run_odometry(params(search_radius=4.5), two, T_init[1:2], None, cell_size=1.0, adaptive=threshold())
    assert "(0, 4]" in ctx.lib.dcreg_last_error(ctx._h).decode()
