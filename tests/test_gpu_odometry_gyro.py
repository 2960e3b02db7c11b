"""Scan-to-map odometry with gyroscope input (dcreg_icp_run_odometry_gyro, dcreg_odometry_open_gyro,
dcreg_odometry_push_gyro): every non-anchor frame's prior rotation and deskew rotation come from integrated rates.

What is held: gyro = NULL is the adaptive call, byte for byte and launch for launch; the returned T_prior follow the twin
(api.gyro_increment) recomputed from the returned T_out, and deskewed_xyz the twin (api.deskew_points_gyro) to one float32
ulp or 1e-12 m; every frame equals its single run from T_prior on its deskewed points; sessions equal the one call under
any chunking, with pushes that carry only the samples bracketing their frames, and a failed push commits nothing."""
import ctypes as C
import math

import numpy as np
import pytest

from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import CELL, assert_anchor, assert_same_flat, raw_odometry, split, window_map  # noqa: F401

pytestmark = pytest.mark.gpu

LENS = (5, 7)
MV, DIST = 0.25, 10.0
MAPS = ["window", "voxel_map"]
MAP_KW = {"window": dict(map_frames=3), "voxel_map": dict(map_voxel=MV, max_distance=DIST)}
R_SI = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])     # the IMU turned 90 degrees about z
BIAS = (0.002, -0.001, 0.003)


@pytest.fixture(scope="module")
def imu():
    """12 sweeps of make_parking_imu (about 8 k points, 20 m range; samples in an IMU frame turned against the LiDAR's,
    with a bias), in sequences of 5 and 7 frames whose anchors are unskewed; both sequences get every sample"""
    from dcreg_b200.scenes import make_parking_imu
    sk, ts, ft, smp, T, fr = make_parking_imu(sum(LENS), n_scan=8_000, max_range=20.0, R_sensor_imu=R_SI, bias=BIAS)
    b = np.concatenate([[0], np.cumsum(LENS)])
    for a in b[:-1]:
        sk[a] = fr[a]
    cut = lambda x: [list(x[p:q]) for p, q in zip(b[:-1], b[1:])]        # noqa: E731
    return dict(skewed=cut(sk), stamps=cut(ts), ft=ft, samples=[smp] * len(LENS), T_init=np.ascontiguousarray(T[b[:-1]]),
                T_true=T, unskewed=fr)


def gyro():
    from dcreg_b200.api import Gyro
    return Gyro(R_SI, BIAS)


def threshold():
    from dcreg_b200.api import AdaptiveThreshold
    return AdaptiveThreshold(0.12, 0.01, 20.0)


def run(ctx, which, prm, d, stamps=True, **kw):
    kw = dict(want_log=True, want_cov=True, motion="constant_velocity", cell_size=CELL, gyro=gyro(), frame_times=d["ft"],
              gyro_samples=d["samples"], timestamps=d["stamps"] if stamps else None, want_deskewed=True) | kw
    if which == "voxel_map":
        return ctx.icp_run_odometry_map(prm, d["skewed"], d["T_init"], None, map_voxel=MV, max_distance=DIST, **kw)
    return ctx.icp_run_odometry(prm, d["skewed"], d["T_init"], None, map_frames=3, **kw)


def counted(ctx, f):
    before = ctx.launch_count
    out = f()
    return out, ctx.launch_count - before


def mid(ft):
    return ft[:, 0] + 0.5 * ft[:, 1]


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("with_threshold", [False, True])
def test_null_gyro_is_the_adaptive_call(ctx, imu, which, with_threshold):
    """gyro = NULL: dcreg_icp_run_odometry_adaptive's bytes and launches, frame_times and samples not read"""
    from dcreg_b200 import api
    prm = params(search_radius=2.0 if with_threshold else 0.5)
    ts = np.ascontiguousarray(np.concatenate([t for s in imu["stamps"] for t in s]), np.float32)
    n = sum(LENS)
    values = dict(map_frames=3 if which == "window" else 0, motion=1, source_voxel=0.3, map_voxel=MV if which == "voxel_map" else 0.0,
                  source_max_points=1, map_max_points=4, max_distance=DIST,
                  adaptive=C.byref(threshold()) if with_threshold else None,
                  timestamps=ts.ctypes.data_as(C.POINTER(C.c_float)))
    nan = np.full((n, 2), math.nan)                 # frame times that would be refused, if they were read
    outs, launches = [], []
    for entry, extra in [("dcreg_icp_run_odometry_adaptive", {}),
                         ("dcreg_icp_run_odometry_gyro", dict(frame_times=nan.ctypes.data_as(C.POINTER(C.c_double))))]:
        desk = np.full((len(ts), 3), -1.0, np.float32)
        rad = np.full(n, -1.0)
        (rc, out), k = counted(ctx, lambda: raw_odometry(
            ctx, entry, prm, imu["skewed"], imu["T_init"], None, log_cap=30, **values, **extra,
            deskewed_xyz=desk.ctypes.data_as(C.POINTER(C.c_float)), search_radius=rad.ctypes.data_as(C.POINTER(C.c_double))))
        assert rc == api.OK
        outs.append([a.tobytes() for a in out.values()] + [desk.tobytes(), rad.tobytes()])
        launches.append(k)
    assert outs[0] == outs[1]
    assert launches[0] == launches[1]


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("stamps", [True, False])
def test_priors_and_deskew_follow_the_twin(ctx, imu, which, stamps):
    """T_prior = compose_prior(T_out[k-1], gyro_increment(..., T_out[k-2], T_out[k-1])) to FP64 rounding; deskewed_xyz =
    deskew_points_gyro with that increment's translation to one float32 ulp or 1e-12 m (timestamps NULL: the points
    themselves, bit for bit)"""
    from dcreg_b200.api import compose_prior, deskew_points_gyro, gyro_increment
    res = run(ctx, which, params(), imu, stamps=stamps)
    tm = mid(imu["ft"])
    k0 = 0
    for s, rs in enumerate(split(res, imu["skewed"])):
        assert_anchor(rs[0], imu["T_init"][s])
        for j in range(1, len(rs)):
            k = k0 + j
            D = gyro_increment(imu["samples"][s], tm[k - 1], tm[k], rs[j - 2].T if j >= 2 else None, rs[j - 1].T, R_SI,
                               BIAS)
            P = compose_prior(rs[j - 1].T, D)
            assert np.abs(rs[j].T_prior - P).max() < 1e-12, (s, j)
            P_in = imu["skewed"][s][j]
            if not stamps:
                assert rs[j].deskewed.tobytes() == P_in.tobytes()
                continue
            twin = deskew_points_gyro(P_in, imu["stamps"][s][j], imu["ft"][k], tm[k - 1], imu["samples"][s], D[:3, 3],
                                      R_SI, BIAS)
            err = np.abs(rs[j].deskewed.astype(np.float64) - twin.astype(np.float64))
            assert (err <= np.maximum(np.spacing(np.abs(twin)).astype(np.float64), 1e-12)).all(), (s, j)
            assert np.abs(twin - P_in).max() > 0.01                 # the sweep moved
        k0 += len(rs)


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_frames_equal_single_runs(ctx, imu, method):
    """Every registered frame is set_target(its window of deskewed frames) + set_source(its deskewed points) +
    icp_run(T_prior)"""
    prm = params(method)
    res = run(ctx, "window", prm, imu)
    for s, rs in enumerate(split(res, imu["skewed"])):
        frames = [r.deskewed for r in rs]
        for k in range(1, len(rs)):
            ctx.set_target(window_map(None, rs, k, 3, frames=frames), CELL)
            ctx.set_source(frames[k])
            assert_same_run(rs[k], ctx.icp_run(prm, rs[k].T_prior))


def bracket(smp, lo, hi):
    """The rows of smp from the last at or before lo to the first at or after hi"""
    a = np.searchsorted(smp[:, 0], lo, side="right") - 1
    b = np.searchsorted(smp[:, 0], hi, side="left")
    return smp[a:b + 1]


def pushed(ctx, which, prm, d, chunks, fail_at=None):
    """d pushed in chunks into a gyro session; each push carries only its frames' times and the samples that bracket its
    frames, from the previous mid-sweep (the anchor's start) to the last sweep's end.  fail_at: before that push, one
    whose samples stop short of its last sweep's end, which must fail"""
    from dcreg_b200 import api
    tm, ft = mid(d["ft"]), d["ft"]
    first = np.concatenate([[0], np.cumsum(LENS)])
    done = [0] * len(LENS)
    out = [[] for _ in LENS]
    open_ = ctx.odometry_map_session if which == "voxel_map" else ctx.odometry_session
    with open_(prm, len(LENS), d["T_init"], "constant_velocity", cell_size=CELL, adaptive=threshold(), gyro=gyro(),
               **MAP_KW[which]) as sess:
        for i, cnt in enumerate(chunks):
            def push(short=False):
                part, ts, fts, smp = [], [], [], []
                for s, c in enumerate(cnt):
                    g = first[s] + done[s]
                    part.append(d["skewed"][s][done[s]:done[s] + c])
                    ts.append(d["stamps"][s][done[s]:done[s] + c])
                    fts.append(ft[g:g + c])
                    lo = tm[g - 1] if done[s] else ft[g, 0]
                    hi = ft[g + c - 1, 0] + ft[g + c - 1, 1] - (0.02 if short else 0.0)
                    smp.append(bracket(d["samples"][s], min(lo, ft[g, 0]), hi) if c else np.zeros((0, 4)))
                return sess.push(part, want_log=True, want_cov=True, timestamps=ts, want_deskewed=True,
                                 frame_times=np.concatenate(fts), gyro_samples=smp)
            if i == fail_at:
                with pytest.raises(api.DcregError) as e:
                    push(short=True)
                assert e.value.status == api.BAD_ARG and "at or after" in str(e.value)
            for s, r in enumerate(push()):
                out[s].extend(r)
            done = [x + c for x, c in zip(done, cnt)]
    return [r for rs in out for r in rs]


@pytest.mark.parametrize("which", MAPS)
def test_chunkings_equal_one_call(ctx, imu, which):
    """Three chunkings, each push with only its bracketing samples (so a push's first frame integrates from a mid-sweep
    time of an earlier push), give the one call's bytes; a push that fails first commits nothing"""
    prm = params(search_radius=2.0)
    ref = run(ctx, which, prm, imu, adaptive=threshold())
    for chunks, fail_at in [([list(LENS)], None), ([[1, 1]] * 5 + [[0, 2]], 2), ([[2, 1], [0, 3], [3, 3]], 1)]:
        got = pushed(ctx, which, prm, imu, chunks, fail_at)
        assert_same_flat(got, ref, radius=True)


def test_plain_push_on_a_gyro_session(ctx, imu):
    """dcreg_odometry_push on a gyro session takes anchors only; the sequence's next frame then has no previous
    mid-sweep time and is refused, and neither refusal changes the session"""
    from dcreg_b200 import api
    d = imu
    with ctx.odometry_session(params(), 1, d["T_init"][:1], "constant_velocity", cell_size=CELL, gyro=gyro()) as sess:
        sess.push([d["skewed"][0][:1]])
        with pytest.raises(api.DcregError) as e:
            sess.push([d["skewed"][0][1:2]])
        assert "gyro samples" in str(e.value)
        with pytest.raises(api.DcregError) as e:
            sess.push([d["skewed"][0][1:2]], frame_times=d["ft"][1:2], gyro_samples=d["samples"][:1])
        assert "unknown" in str(e.value)


def test_reproducible_and_context_untouched(ctx, imu):
    prm = params()
    ctx.set_target(imu["unskewed"][3], CELL)
    ctx.set_source(imu["unskewed"][4])
    before = ctx.icp_run(prm, np.eye(4))
    a = run(ctx, "window", prm, imu)
    b = run(ctx, "voxel_map", prm, imu)
    a2 = run(ctx, "window", prm, imu)
    b2 = run(ctx, "voxel_map", prm, imu)
    after = ctx.icp_run(prm, np.eye(4))
    assert_same_flat(a2, a, radius=True)
    assert_same_flat(b2, b, radius=True)
    assert (after.status, after.iterations, after.converged) == (before.status, before.iterations, before.converged)
    assert after.T.tobytes() == before.T.tobytes()


@pytest.mark.parametrize("which", MAPS)
def test_launches_do_not_depend_on_the_number_of_sequences(ctx, imu, which):
    prm = params(fixed_iterations=1, max_iterations=4)
    d = imu
    one = dict(d, skewed=[d["skewed"][1][:4]], stamps=[d["stamps"][1][:4]], ft=d["ft"][5:9], samples=d["samples"][:1],
               T_init=d["T_true"][5:6])
    three = dict(d, skewed=[d["skewed"][1][:4], d["skewed"][0][:4], d["skewed"][1][3:7]],
                 stamps=[d["stamps"][1][:4], d["stamps"][0][:4], d["stamps"][1][3:7]],
                 ft=np.concatenate([d["ft"][5:9], d["ft"][0:4], d["ft"][8:12]]), samples=d["samples"][:1] * 3,
                 T_init=d["T_true"][[5, 0, 8]])
    run(ctx, which, prm, three, want_log=False)
    _, n1 = counted(ctx, lambda: run(ctx, which, prm, one, want_log=False))
    _, n3 = counted(ctx, lambda: run(ctx, which, prm, three, want_log=False))
    assert n1 == n3


def test_bad_arguments(ctx, imu):
    """Every gyro rule is BAD_ARG naming the sequence, frame or sample, before anything is launched"""
    from dcreg_b200 import api
    d = imu
    prm = params()
    two = dict(d, skewed=[d["skewed"][0][:3]], stamps=[d["stamps"][0][:3]], ft=d["ft"][:3], samples=d["samples"][:1],
               T_init=d["T_init"][:1])
    smp = d["samples"][0]

    def bad(expect, g=None, **over):
        with pytest.raises(api.DcregError) as e:
            run(ctx, "window", prm, dict(two, **{k: v for k, v in over.items() if k in two}),
                **{k: v for k, v in over.items() if k not in two}, **({} if g is None else dict(gyro=g)))
        assert e.value.status == api.BAD_ARG and expect in str(e.value), str(e.value)

    launches = ctx.launch_count
    for R in (np.diag([1.0, 1.0, math.nan]), np.diag([1.0, 1.0, 1.001]), np.ones((3, 3))):
        bad("R_sensor_imu", api.Gyro(R))
    bad("bias", api.Gyro(None, (0.0, math.inf, 0.0)))
    s2 = smp.copy(); s2[7, 2] = math.nan
    bad("sequence 0, sample 7", samples=[s2])
    s3 = smp.copy(); s3[9, 0] = s3[8, 0]
    bad("sample 9", samples=[s3])
    for span in (0.0, -0.1, math.nan, math.inf):
        f = d["ft"][:3].copy(); f[1, 1] = span
        bad("frame 1", ft=f)
    f = d["ft"][:3].copy(); f[2, 0] = f[1, 0] - 0.5 * f[1, 1]
    bad("not after", ft=f)
    t1 = mid(d["ft"])[0]
    bad("at or before", samples=[smp[smp[:, 0] > t1]])
    bad("at or after", samples=[smp[smp[:, 0] < d["ft"][2, 0] + d["ft"][2, 1] - 1e-3]])
    bad("CONSTANT_VELOCITY", motion="increments")
    assert ctx.launch_count == launches
    with pytest.raises(api.DcregError) as e:
        ctx.odometry_session(prm, 1, d["T_init"][:1], "constant_velocity", gyro=api.Gyro(np.ones((3, 3))))
    assert e.value.status == api.BAD_ARG
    with pytest.raises(api.DcregError) as e:
        with ctx.odometry_session(prm, 1, d["T_init"][:1], "constant_velocity", cell_size=CELL) as sess:
            sess.gyro = True        # gyro input pushed onto a session opened without it
            sess.push([two["skewed"][0][:1]], frame_times=two["ft"][:1], gyro_samples=two["samples"])
    assert "opened with gyro input" in str(e.value)
