"""Scan-to-map odometry with accelerometer input (dcreg_icp_run_odometry_imu, dcreg_odometry_open_imu,
dcreg_odometry_push_imu): every non-anchor frame's prior translation comes from the previous frame's velocity and the
preintegrated specific force, beside the gyro's rotation, and every frame's velocity is returned.

What is held: imu = NULL is the gyro call with gyro = NULL, byte for byte and launch for launch; the returned T_prior
follow the twin (api.imu_increment) recomputed from the returned T_out and velocities, the velocities the twin
(api.imu_velocity), and deskewed_xyz the gyro deskew (api.deskew_points_gyro) with the IMU translation, to one float32 ulp
or 1e-12 m; every frame equals its single run; window, voxel map and prior map; sessions equal the one call, velocity
included, under any chunking, and a failed push commits nothing."""
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
GB, AB = (0.002, -0.001, 0.003), (0.05, -0.02, 0.03)
GRAV = (0.0, 0.0, -9.80665)
N_MAP = 200_000


@pytest.fixture(scope="module")
def imu():
    """12 sweeps of make_parking_imu_accel (about 8 k points, 20 m range, 0.5 m a frame; samples in an IMU frame turned
    against the LiDAR's, with biases), in sequences of 5 and 7 frames whose anchors are unskewed; both sequences get
    every sample, and v_init is the true velocity of each sequence's first frame"""
    from dcreg_b200 import scenes
    sk, ts, ft, smp, T, v, fr = scenes.make_parking_imu_accel(sum(LENS), n_scan=8_000, max_range=20.0, n_map=N_MAP,
                                                              path_half_length=3.0, R_sensor_imu=R_SI, gyro_bias=GB,
                                                              accel_bias=AB)
    b = np.concatenate([[0], np.cumsum(LENS)])
    for a in b[:-1]:
        sk[a] = fr[a]
    cut = lambda x: [list(x[p:q]) for p, q in zip(b[:-1], b[1:])]        # noqa: E731
    return dict(skewed=cut(sk), stamps=cut(ts), ft=ft, samples=[smp] * len(LENS), T_init=np.ascontiguousarray(T[b[:-1]]),
                v_init=np.ascontiguousarray(v[b[:-1]]), T_true=T, v_true=v, unskewed=fr,
                map=scenes._parking_map(np.random.default_rng(43), N_MAP, 60.0))


def imu_settings():
    from dcreg_b200.api import Imu
    return Imu(R_SI, GB, AB, GRAV)


def threshold():
    from dcreg_b200.api import AdaptiveThreshold
    return AdaptiveThreshold(0.12, 0.01, 20.0)


def run(ctx, which, prm, d, stamps=True, **kw):
    kw = dict(want_log=True, want_cov=True, motion="constant_velocity", cell_size=CELL, imu=imu_settings(),
              frame_times=d["ft"], imu_samples=d["samples"], v_init=d["v_init"], want_velocity=True,
              timestamps=d["stamps"] if stamps else None, want_deskewed=True) | kw
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
def test_null_imu_is_the_null_gyro_call(ctx, imu, which, with_threshold):
    """imu = NULL: dcreg_icp_run_odometry_gyro's (gyro = NULL) bytes and launches; frame_times, samples and v_init not
    read, velocity not written"""
    from dcreg_b200 import api
    prm = params(search_radius=2.0 if with_threshold else 0.5)
    ts = np.ascontiguousarray(np.concatenate([t for s in imu["stamps"] for t in s]), np.float32)
    n = sum(LENS)
    values = dict(map_frames=3 if which == "window" else 0, motion=1, source_voxel=0.3,
                  map_voxel=MV if which == "voxel_map" else 0.0, source_max_points=1, map_max_points=4,
                  max_distance=DIST, adaptive=C.byref(threshold()) if with_threshold else None,
                  timestamps=ts.ctypes.data_as(C.POINTER(C.c_float)))
    nan = np.full((n, 2), math.nan)                 # inputs that would be refused, if they were read
    vel = np.full((n, 3), -1.0)
    outs, launches = [], []
    for entry, extra in [("dcreg_icp_run_odometry_gyro", {}),
                         ("dcreg_icp_run_odometry_imu", dict(frame_times=nan.ctypes.data_as(C.POINTER(C.c_double)),
                                                             v_init=nan.ctypes.data_as(C.POINTER(C.c_double)),
                                                             velocity=vel.ctypes.data_as(C.POINTER(C.c_double))))]:
        desk = np.full((len(ts), 3), -1.0, np.float32)
        rad = np.full(n, -1.0)
        (rc, out), k = counted(ctx, lambda: raw_odometry(
            ctx, entry, prm, imu["skewed"], imu["T_init"], None, log_cap=30, **values, **extra,
            deskewed_xyz=desk.ctypes.data_as(C.POINTER(C.c_float)),
            search_radius=rad.ctypes.data_as(C.POINTER(C.c_double))))
        assert rc == api.OK
        outs.append([a.tobytes() for a in out.values()] + [desk.tobytes(), rad.tobytes()])
        launches.append(k)
    assert outs[0] == outs[1]
    assert launches[0] == launches[1]
    assert (vel == -1.0).all()


def check_twin(res, d, starts, stamps=True, prior_map=False):
    """T_prior, velocity and deskewed points of every frame against the twin, from the returned T_out and velocities;
    starts: each sequence's first global frame index.  An anchor, or (prior map) a first frame, has v = v_init."""
    from dcreg_b200.api import compose_prior, deskew_points_gyro, imu_increment, imu_velocity
    tm = mid(d["ft"])
    moved = 0
    for s, rs in enumerate(split(res, d["skewed"])):
        if not prior_map:
            assert_anchor(rs[0], d["T_init"][s])
        assert rs[0].velocity.tobytes() == d["v_init"][s].tobytes()
        for j in range(1, len(rs)):
            k = starts[s] + j
            D = imu_increment(d["samples"][s], tm[k - 1], tm[k], rs[j - 1].T, rs[j - 1].velocity, GRAV, R_SI, GB, AB)
            assert np.abs(rs[j].T_prior - compose_prior(rs[j - 1].T, D)).max() < 1e-12, (s, j)
            v = imu_velocity(d["samples"][s], tm[k - 1], tm[k], rs[j - 1].T, rs[j].T, GRAV, R_SI, GB, AB)
            assert np.abs(rs[j].velocity - v).max() <= 1e-12 * max(1.0, np.abs(v).max()), (s, j)
            P_in = d["skewed"][s][j]
            if not stamps:
                assert rs[j].deskewed.tobytes() == P_in.tobytes()
                continue
            twin = deskew_points_gyro(P_in, d["stamps"][s][j], d["ft"][k], tm[k - 1], d["samples"][s][:, :4], D[:3, 3],
                                      R_SI, GB)
            err = np.abs(rs[j].deskewed.astype(np.float64) - twin.astype(np.float64))
            assert (err <= np.maximum(np.spacing(np.abs(twin)).astype(np.float64), 1e-12)).all(), (s, j)
            moved += np.abs(twin - P_in).max() > 0.01
    assert not stamps or moved > 0


@pytest.mark.parametrize("which", MAPS)
@pytest.mark.parametrize("stamps", [True, False])
@pytest.mark.parametrize("with_threshold", [False, True])
def test_priors_velocities_and_deskew_follow_the_twin(ctx, imu, which, stamps, with_threshold):
    prm = params(search_radius=2.0 if with_threshold else 0.5)
    res = run(ctx, which, prm, imu, stamps=stamps, adaptive=threshold() if with_threshold else None)
    check_twin(res, imu, np.concatenate([[0], np.cumsum(LENS)]), stamps)


def test_prior_map_follows_the_twin(ctx, imu):
    """dcreg_set_prior_map(1): first frames register from T_init and keep v_init; the frames after them follow the twin"""
    prm = params(search_radius=2.0)
    ctx.set_target(imu["map"], CELL)
    ctx.set_prior_map(True)
    try:
        res = run(ctx, "window", prm, imu, adaptive=threshold())
        res2 = run(ctx, "window", prm, imu, adaptive=threshold())
    finally:
        ctx.set_prior_map(False)
    check_twin(res, imu, np.concatenate([[0], np.cumsum(LENS)]), prior_map=True)
    assert_same_flat(res2, res, radius=True)


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
    """d pushed in chunks into an IMU session; each push carries only its frames' times and the samples that bracket
    its frames.  fail_at: before that push, one whose samples stop short of its last sweep's end, which must fail"""
    from dcreg_b200 import api
    tm, ft = mid(d["ft"]), d["ft"]
    first = np.concatenate([[0], np.cumsum(LENS)])
    done = [0] * len(LENS)
    out = [[] for _ in LENS]
    open_ = ctx.odometry_map_session if which == "voxel_map" else ctx.odometry_session
    with open_(prm, len(LENS), d["T_init"], "constant_velocity", cell_size=CELL, adaptive=threshold(),
               imu=imu_settings(), v_init=d["v_init"], **MAP_KW[which]) as sess:
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
                    smp.append(bracket(d["samples"][s], min(lo, ft[g, 0]), hi) if c else np.zeros((0, 7)))
                return sess.push(part, want_log=True, want_cov=True, timestamps=ts, want_deskewed=True,
                                 frame_times=np.concatenate(fts), imu_samples=smp, want_velocity=True)
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
    """Three chunkings, each push with only its bracketing samples, give the one call's bytes, velocities included; a
    push that fails first commits nothing"""
    prm = params(search_radius=2.0)
    ref = run(ctx, which, prm, imu, adaptive=threshold())
    for chunks, fail_at in [([list(LENS)], None), ([[1, 1]] * 5 + [[0, 2]], 2), ([[2, 1], [0, 3], [3, 3]], 1)]:
        got = pushed(ctx, which, prm, imu, chunks, fail_at)
        assert_same_flat(got, ref, radius=True)
        assert b"".join(r.velocity.tobytes() for r in got) == b"".join(r.velocity.tobytes() for r in ref)


def test_plain_push_on_an_imu_session(ctx, imu):
    """dcreg_odometry_push on an IMU session takes anchors only, which take v_init; gyro samples are refused"""
    from dcreg_b200 import api
    d = imu
    with ctx.odometry_session(params(), 1, d["T_init"][:1], "constant_velocity", cell_size=CELL, imu=imu_settings(),
                              v_init=d["v_init"][:1]) as sess:
        sess.push([d["skewed"][0][:1]])
        with pytest.raises(api.DcregError) as e:
            sess.push([d["skewed"][0][1:2]])
        assert "gyro samples" in str(e.value)
        sess.gyro, sess.imu = True, False       # 4-column samples pushed onto an IMU session
        with pytest.raises(api.DcregError) as e:
            sess.push([d["skewed"][0][1:2]], frame_times=d["ft"][1:2], gyro_samples=[d["samples"][0][:, :4]])
        assert "7-column" in str(e.value)


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
    for x, y in ((a, a2), (b, b2)):
        assert b"".join(r.velocity.tobytes() for r in x) == b"".join(r.velocity.tobytes() for r in y)
    assert (after.status, after.iterations, after.converged) == (before.status, before.iterations, before.converged)
    assert after.T.tobytes() == before.T.tobytes()


@pytest.mark.parametrize("which", MAPS)
def test_launches_do_not_depend_on_the_number_of_sequences(ctx, imu, which):
    prm = params(fixed_iterations=1, max_iterations=4)
    d = imu
    one = dict(d, skewed=[d["skewed"][1][:4]], stamps=[d["stamps"][1][:4]], ft=d["ft"][5:9], samples=d["samples"][:1],
               T_init=d["T_true"][5:6], v_init=d["v_true"][5:6])
    three = dict(d, skewed=[d["skewed"][1][:4], d["skewed"][0][:4], d["skewed"][1][3:7]],
                 stamps=[d["stamps"][1][:4], d["stamps"][0][:4], d["stamps"][1][3:7]],
                 ft=np.concatenate([d["ft"][5:9], d["ft"][0:4], d["ft"][8:12]]), samples=d["samples"][:1] * 3,
                 T_init=d["T_true"][[5, 0, 8]], v_init=d["v_true"][[5, 0, 8]])
    run(ctx, which, prm, three, want_log=False)
    _, n1 = counted(ctx, lambda: run(ctx, which, prm, one, want_log=False))
    _, n3 = counted(ctx, lambda: run(ctx, which, prm, three, want_log=False))
    _, ng = counted(ctx, lambda: run(ctx, which, prm, one, want_log=False, imu=None, imu_samples=None, v_init=None,
                                     want_velocity=False, gyro=__import__("dcreg_b200").Gyro(R_SI, GB),
                                     gyro_samples=[s[:, :4] for s in one["samples"]]))
    assert n1 == n3
    assert n1 == ng + 3                 # one velocity launch per registered step


def test_bad_arguments(ctx, imu):
    """Every new rule is BAD_ARG naming the sequence or sample, before anything is launched"""
    from dcreg_b200 import api
    d = imu
    prm = params()
    two = dict(d, skewed=[d["skewed"][0][:3]], stamps=[d["stamps"][0][:3]], ft=d["ft"][:3], samples=d["samples"][:1],
               T_init=d["T_init"][:1], v_init=d["v_init"][:1])

    def bad(expect, **over):
        with pytest.raises(api.DcregError) as e:
            run(ctx, "window", prm, dict(two, **{k: v for k, v in over.items() if k in two}),
                **{k: v for k, v in over.items() if k not in two})
        assert e.value.status == api.BAD_ARG and expect in str(e.value), str(e.value)

    launches = ctx.launch_count
    bad("accel_bias", imu=api.Imu(R_SI, GB, (0.0, math.nan, 0.0), GRAV))
    bad("gravity", imu=api.Imu(R_SI, GB, AB, (0.0, 0.0, -math.inf)))
    bad("v_init of sequence 0", v_init=np.array([[0.0, math.nan, 0.0]]))
    s2 = d["samples"][0].copy(); s2[7, 5] = math.inf
    bad("sequence 0, sample 7", samples=[s2])
    bad("R_sensor_imu", imu=api.Imu(np.ones((3, 3)), GB, AB, GRAV))
    bad("CONSTANT_VELOCITY", motion="increments")
    assert ctx.launch_count == launches
    with pytest.raises(api.DcregError) as e:
        ctx.odometry_session(prm, 2, d["T_init"], "constant_velocity", imu=imu_settings(),
                             v_init=np.array([[0.0, 0.0, 0.0], [math.inf, 0.0, 0.0]]))
    assert e.value.status == api.BAD_ARG and "v_init of sequence 1" in str(e.value)
    with pytest.raises(api.DcregError) as e:
        with ctx.odometry_session(prm, 1, d["T_init"][:1], "constant_velocity", cell_size=CELL,
                                  gyro=api.Gyro(R_SI, GB)) as sess:
            sess.gyro, sess.imu = False, True       # IMU samples pushed onto a gyro session
            sess.push([two["skewed"][0][:1]], frame_times=two["ft"][:1], imu_samples=two["samples"])
    assert "opened with IMU input" in str(e.value)
