"""Motion compensation inside scan-to-map odometry (dcreg_icp_run_odometry_deskew, dcreg_odometry_push_deskew) on the
make_parking_sweeps scene: the NULL and mid-sweep cases against the calls without deskewing (bytes and launches), the
deskewed points against the NumPy twin with the increments the call returns, every registered frame against a single
run on the deskewed points, the end-to-end recovery of the unskewed result, sessions, and the errors."""
import numpy as np
import pytest

import dcreg_oracle as o

from odom_harness import CELL, RADIUS, ctx, params, pushed, result_bytes, sweeps  # noqa: F401

pytestmark = pytest.mark.gpu

LENS = (5, 7)


def flat(x):
    return [f for s in x for f in s]


def run(ctx, prm, sw, frames="skewed", stamps="stamps", **kw):
    kw.setdefault("map_frames", 3)
    kw.setdefault("deltas", sw["deltas"] if kw.get("motion", "increments") == "increments" else None)
    ts = None if stamps is None else (sw[stamps] if isinstance(stamps, str) else stamps)
    return ctx.icp_run_odometry(prm, sw[frames], sw["T_init"], cell_size=CELL, timestamps=ts, **kw)


def increments(res, sw, motion):
    """D_k of every frame from the call's own outputs (None for an anchor)"""
    from dcreg_b200.api import constant_velocity_increment
    D, k = [], 0
    for s in sw["skewed"]:
        for j in range(len(s)):
            if j == 0:
                D.append(None)
            elif motion == "increments":
                D.append(sw["deltas"][k + j - 1])
            else:
                D.append(np.eye(4) if j == 1 else constant_velocity_increment(res[k + j - 2].T, res[k + j - 1].T))
        k += len(s)
    return D


def kept(frame, stamps, source_voxel):
    from dcreg_b200.api import voxel_downsample
    if not source_voxel:
        return np.asarray(frame, np.float32)[:, :3], np.asarray(stamps, np.float32)
    pts, idx = voxel_downsample(frame, source_voxel)
    return pts, np.asarray(stamps, np.float32)[idx]


def within_contract(got, ref):
    ulp = np.spacing(np.abs(ref)).astype(np.float64)
    return bool((np.abs(got.astype(np.float64) - ref.astype(np.float64)) <= np.maximum(ulp, 1e-12)).all())


def test_null_timestamps_are_the_voxel_n_call(ctx, sweeps):
    prm = params()
    for kw in (dict(), dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)):
        a0 = ctx.launch_count
        ref = run(ctx, prm, sweeps, stamps=None, want_log=True, **kw)
        a1 = ctx.launch_count
        got = run(ctx, prm, sweeps, stamps=None, want_log=True, want_deskewed=True, **kw)
        assert ctx.launch_count - a1 == a1 - a0
        assert result_bytes(got) == result_bytes(ref)
        for r, f in zip(got, flat(sweeps["skewed"])):
            assert r.deskewed.tobytes() == kept(f, np.zeros(len(f)), kw.get("source_voxel"))[0].tobytes()


def test_mid_sweep_timestamps_change_nothing(ctx, sweeps):
    """tau = 0.5 everywhere: the bytes of the call without timestamps, every point copied, and one launch per call and
    two per step more"""
    prm = params()
    half = [[np.full(len(f), 0.5, np.float32) for f in s] for s in sweeps["skewed"]]
    for kw in (dict(), dict(source_voxel=0.25)):
        a0 = ctx.launch_count
        ref = run(ctx, prm, sweeps, stamps=None, want_cov=True, **kw)
        a1 = ctx.launch_count
        got = run(ctx, prm, sweeps, stamps=half, want_cov=True, want_deskewed=True, **kw)
        assert ctx.launch_count - a1 == (a1 - a0) + 1 + 2 * (max(LENS) - 1)
        assert result_bytes(got) == result_bytes(ref)
        for r, f in zip(got, flat(sweeps["skewed"])):
            assert r.deskewed.tobytes() == kept(f, np.zeros(len(f)), kw.get("source_voxel"))[0].tobytes()


@pytest.mark.parametrize("motion", ["increments", "constant_velocity"])
@pytest.mark.parametrize("source_voxel", [0.0, 0.25])
def test_deskewed_points_against_the_twin(ctx, sweeps, motion, source_voxel):
    from dcreg_b200.api import deskew_points
    prm = params()
    res = run(ctx, prm, sweeps, motion=motion, source_voxel=source_voxel, want_deskewed=True)
    D = increments(res, sweeps, motion)
    moved = 0
    for r, f, t, d in zip(res, flat(sweeps["skewed"]), flat(sweeps["stamps"]), D):
        pts, ts = kept(f, t, source_voxel)
        assert r.n_points == len(pts) == len(r.deskewed)
        if d is None:
            assert r.deskewed.tobytes() == pts.tobytes()
            continue
        twin = deskew_points(pts, ts, d)
        assert within_contract(r.deskewed, twin)
        moved += int((r.deskewed != pts).any(axis=1).sum())
    assert moved > 0


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_every_frame_is_a_single_run_on_its_deskewed_points(ctx, sweeps, method):
    from dcreg_b200.api import compose_prior, map_points
    prm = params(method)
    res = run(ctx, prm, sweeps, want_log=True, want_deskewed=True)
    D = increments(res, sweeps, "increments")
    k0 = 0
    for s in sweeps["skewed"]:
        rs = res[k0:k0 + len(s)]
        for k in range(1, len(s)):
            assert rs[k].T_prior.tobytes() == compose_prior(rs[k - 1].T, D[k0 + k]).tobytes()
            ctx.set_target(np.concatenate([map_points(rs[j].T, rs[j].deskewed) for j in range(max(0, k - 3), k)]), CELL)
            ctx.set_source(rs[k].deskewed)
            one = ctx.icp_run(prm, rs[k].T_prior)
            b = rs[k]
            assert (b.status, b.iterations, b.converged) == (one.status, one.iterations, one.converged)
            assert o.se3_log_distance(one.T, b.T) < 1e-8
            for x, y in zip(b.logs, one.logs):
                assert x.n_effective == y.n_effective and x.n_corr_pt == y.n_corr_pt
                assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)
        k0 += len(s)


def test_deskewing_recovers_the_unskewed_result(ctx, sweeps):
    """Skewed sweeps deskewed with the true increments register within 5 mm / 0.05 deg of the unskewed frames"""
    prm = params()
    got = run(ctx, prm, sweeps)
    ref = run(ctx, prm, sweeps, frames="unskewed", stamps=None)
    for a, b in zip(got, ref):
        dT = np.linalg.inv(b.T) @ a.T
        assert np.linalg.norm(dT[:3, 3]) < 5e-3
        assert np.degrees(np.arccos(np.clip((np.trace(dT[:3, :3]) - 1) / 2, -1, 1))) < 0.05


@pytest.mark.parametrize("filters", [dict(), dict(source_voxel=0.25, map_voxel=0.25, map_max_points=4)])
def test_sessions_equal_one_call(ctx, sweeps, filters):
    prm = params()
    ref = run(ctx, prm, sweeps, want_log=True, want_deskewed=True, **filters)
    for chunks in ([list(LENS)], [[1, 1]] * 5 + [[0, 1], [0, 1]], [[2, 3], [0, 1], [3, 3]]):
        got = flat(pushed(ctx, prm, sweeps["skewed"], sweeps["T_init"], chunks, sweeps["deltas"],
                          stamps=sweeps["stamps"], want_log=True, want_deskewed=True, map_frames=3, **filters))
        assert result_bytes(got) == result_bytes(ref)
        assert all(a.deskewed.tobytes() == b.deskewed.tobytes() for a, b in zip(got, ref))
    # pushes without timestamps are frames with tau = 0.5
    chunks = [[2, 3], [0, 1], [3, 3]]
    mixed = [[t.copy() for t in s] for s in sweeps["stamps"]]
    first = [0, 0]
    for i, cnt in enumerate(chunks):
        for s, c in enumerate(cnt):
            if i == 1:
                for j in range(first[s], first[s] + c):
                    mixed[s][j] = np.full(len(mixed[s][j]), 0.5, np.float32)
            first[s] += c
    ref = run(ctx, prm, sweeps, stamps=mixed, want_log=True, want_deskewed=True, **filters)
    got = flat(pushed(ctx, prm, sweeps["skewed"], sweeps["T_init"], chunks, sweeps["deltas"], stamps=sweeps["stamps"],
                      ts_push=lambda i: i != 1, want_log=True, want_deskewed=True, map_frames=3, **filters))
    assert result_bytes(got) == result_bytes(ref)
    assert all(a.deskewed.tobytes() == b.deskewed.tobytes() for a, b in zip(got, ref))


def test_reproducible_and_context_untouched(ctx, sweeps):
    prm = params()
    tgt = np.concatenate(sweeps["unskewed"][1][:3])
    ctx.set_target(tgt, RADIUS)
    ctx.set_source(sweeps["unskewed"][1][1])
    before = ctx.icp_run(prm, sweeps["T_true"][6])
    a = run(ctx, prm, sweeps, want_deskewed=True, want_log=True, motion="constant_velocity")
    b = run(ctx, prm, sweeps, want_deskewed=True, want_log=True, motion="constant_velocity")
    assert result_bytes(a) == result_bytes(b)
    assert all(x.deskewed.tobytes() == y.deskewed.tobytes() for x, y in zip(a, b))
    after = ctx.icp_run(prm, sweeps["T_true"][6])
    assert after.T.tobytes() == before.T.tobytes() and after.iterations == before.iterations


def test_nan_increment_adds_no_nonfinite_point(ctx, sweeps):
    prm = params()
    sw = dict(sweeps)
    sw["deltas"] = sweeps["deltas"].copy()
    sw["deltas"][3] = np.nan                       # the increment of sequence 0's last frame, which no later map holds
    res = run(ctx, prm, sw, want_deskewed=True)
    for r, f in zip(res, flat(sweeps["skewed"])):
        assert np.isfinite(r.deskewed).all() == np.isfinite(f).all()
    assert res[4].deskewed.tobytes() == flat(sweeps["skewed"])[4].tobytes()      # a NaN twist: copied


def test_bad_timestamps_before_any_launch(ctx, sweeps):
    from dcreg_b200 import api
    prm = params()
    for bad, what in ((np.nan, "not finite"), (1.5, "outside [0, 1]"), (-0.25, "outside [0, 1]")):
        ts = [[t.copy() for t in s] for s in sweeps["stamps"]]
        ts[1][3][17] = bad
        n = ctx.launch_count
        with pytest.raises(api.DcregError) as e:
            run(ctx, prm, sweeps, stamps=ts)
        assert e.value.status == api.BAD_ARG and ctx.launch_count == n
        msg = ctx.lib.dcreg_last_error(ctx._h).decode()
        assert "sequence 1" in msg and "frame 3 of the sequence" in msg and "point 17" in msg and what in msg, msg
    # a failed push leaves the session as it was
    ref = run(ctx, prm, sweeps, want_log=True, want_deskewed=True)
    first = np.concatenate([[0], np.cumsum(LENS)])
    out = [[] for _ in LENS]
    with ctx.odometry_session(prm, 2, sweeps["T_init"], cell_size=CELL, map_frames=3) as sess:
        for s, r in enumerate(sess.push([x[:2] for x in sweeps["skewed"]],
                                        np.concatenate([sweeps["deltas"][a:a + 2] for a in first[:-1]]), want_log=True,
                                        timestamps=[x[:2] for x in sweeps["stamps"]], want_deskewed=True)):
            out[s] += r
        bad = [x[2:] for x in sweeps["stamps"]]
        bad = [[t.copy() for t in s] for s in bad]
        bad[0][1][5] = np.inf
        n = ctx.launch_count
        rest_D = np.concatenate([sweeps["deltas"][a + 2:b] for a, b in zip(first[:-1], first[1:])])
        with pytest.raises(api.DcregError):
            sess.push([x[2:] for x in sweeps["skewed"]], rest_D, timestamps=bad)
        assert ctx.launch_count == n
        assert "frame 3 of the sequence since open" in ctx.lib.dcreg_last_error(ctx._h).decode()
        for s, r in enumerate(sess.push([x[2:] for x in sweeps["skewed"]], rest_D, want_log=True,
                                        timestamps=[x[2:] for x in sweeps["stamps"]], want_deskewed=True)):
            out[s] += r
    got = flat(out)
    assert result_bytes(got) == result_bytes(ref)
    assert all(a.deskewed.tobytes() == b.deskewed.tobytes() for a, b in zip(got, ref))
