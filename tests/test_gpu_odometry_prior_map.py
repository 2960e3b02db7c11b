"""Localisation in a prior map through the odometry front end (dcreg_set_prior_map): every frame registers against the
context's target instead of a local map, each sequence's first frame from its T_init.

What is held: 0 keeps every call's bytes and launches; with increments the calls return dcreg_icp_run_sequences' T_prior
bytes, statuses, iterations and masks, on a dense and on a sparse target; with constant velocity, a source filter,
deskewing (twist and gyro) and the adaptive threshold every frame equals its single run from its T_prior on its
deskewed points, and T_prior and the radii follow the twins; a sparse target gives a dense one's bytes; sessions equal
one call under any chunking, a failed push commits nothing, and a push reads the target at push time; the context's
source and target are untouched, launches do not depend on the number of sequences, and every refusal names the prior
map."""
import numpy as np
import pytest

import dcreg_oracle as o
from harness import assert_same_run, ctx, params  # noqa: F401
from odom_harness import CELL, one_per_push, result_bytes, split

pytestmark = pytest.mark.gpu

LENS = (1, 7, 12)
FAR = np.array([[2000.0, 1500.0, 400.0], [3000.0, 3000.0, 500.0]], dtype=np.float32)
R_SI = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
BIAS = (0.002, -0.001, 0.003)


@pytest.fixture(scope="module")
def seq():
    """20 frames of about 6 k points along the parking path, in sequences of 1, 7 and 12, with drifting increments;
    B: the parking map and four far-corner points (a dense grid), A: B and two far points (a sparse row index)"""
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, T_init, deltas, tgt = make_parking_sequence(sum(LENS), seed=71, n_map=300_000)
    b = np.concatenate([[0], np.cumsum(LENS)])
    corners = np.array([[-60, -60, -6], [60, 60, 5], [-60, 60, 5], [60, -60, -6]], dtype=np.float32)
    B = np.ascontiguousarray(np.concatenate([tgt, corners]))
    A = np.ascontiguousarray(np.concatenate([B, FAR]))
    seqs = [list(frames[p:q]) for p, q in zip(b[:-1], b[1:])]
    return dict(seqs=seqs, T_init=np.ascontiguousarray(T_true[b[:-1]]), deltas=deltas, A=A, B=B, T_true=T_true)


@pytest.fixture(scope="module")
def imu():
    """12 sweeps of make_parking_imu (about 8 k points), sequences of 5 and 7 frames, every sequence every sample,
    and the scene's own parking map"""
    from dcreg_b200.scenes import _parking_map, make_parking_imu
    lens = (5, 7)
    sk, ts, ft, smp, T, fr = make_parking_imu(sum(lens), n_scan=8_000, max_range=20.0, R_sensor_imu=R_SI, bias=BIAS)
    b = np.concatenate([[0], np.cumsum(lens)])
    cut = lambda x: [list(x[p:q]) for p, q in zip(b[:-1], b[1:])]        # noqa: E731
    return dict(skewed=cut(sk), stamps=cut(ts), ft=ft, samples=[smp] * len(lens), T_init=np.ascontiguousarray(T[b[:-1]]),
                T_true=T, map=_parking_map(np.random.default_rng(43), 500_000, 60.0), lens=lens)


def gyro():
    from dcreg_b200.api import Gyro
    return Gyro(R_SI, BIAS)


def threshold():
    from dcreg_b200.api import AdaptiveThreshold
    return AdaptiveThreshold(0.12, 0.01, 20.0)


def counted(ctx, f):
    before = ctx.launch_count
    out = f()
    return out, ctx.launch_count - before


def prior_map(ctx, f, enable=1):
    ctx.set_prior_map(enable)
    try:
        return f()
    finally:
        ctx.set_prior_map(0)


def twist_kw(d, **kw):
    return dict(motion="constant_velocity", cell_size=CELL, timestamps=d["stamps"], want_deskewed=True, want_log=True,
                want_cov=True, source_voxel=0.3) | kw


def gyro_kw(d, **kw):
    return twist_kw(d, gyro=gyro(), frame_times=d["ft"], gyro_samples=d["samples"], adaptive=threshold()) | kw


def test_off_means_off(ctx, imu):
    """set_prior_map(0) after 1: a window call, a deskew call and a gyro session give the bytes and launches of before"""
    prm = params(search_radius=2.0)
    ctx.set_target(imu["map"], CELL)

    def calls():
        out = []
        out.append(counted(ctx, lambda: result_bytes(ctx.icp_run_odometry(
            prm, imu["skewed"], imu["T_init"], None, map_frames=3, cell_size=CELL, want_log=True))))
        out.append(counted(ctx, lambda: result_bytes(ctx.icp_run_odometry(
            prm, imu["skewed"], imu["T_init"], None, map_frames=3, **twist_kw(imu)))))
        with ctx.odometry_session(prm, 2, imu["T_init"], "constant_velocity", map_frames=3, cell_size=CELL,
                                  adaptive=threshold(), gyro=gyro()) as sess:
            out.append(counted(ctx, lambda: [result_bytes(rs) for rs in sess.push(
                [imu["skewed"][0], imu["skewed"][1]], timestamps=imu["stamps"], frame_times=imu["ft"],
                gyro_samples=imu["samples"])]))
        return out

    before = calls()
    ctx.set_prior_map(1)
    ctx.set_prior_map(0)
    assert calls() == before


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
@pytest.mark.parametrize("target", ["dense", "sparse"])
@pytest.mark.parametrize("with_deltas", [True, False])
def test_increments_equal_sequences(ctx, seq, method, target, with_deltas):
    """Increments, no filter, no timestamps: _sequences' T_prior bytes, statuses, iterations and masks, T_out to 1e-8"""
    prm = params(method)
    ctx.set_target(seq["B"] if target == "dense" else seq["A"], CELL)
    D = seq["deltas"] if with_deltas else None
    ref = ctx.icp_run_sequences(prm, seq["seqs"], seq["T_init"], D, want_log=True, want_cov=True)
    got = prior_map(ctx, lambda: ctx.icp_run_odometry(prm, seq["seqs"], seq["T_init"], D, map_frames=1, cell_size=CELL,
                                                      want_log=True, want_cov=True))
    assert len(got) == len(ref) == sum(LENS)
    for k, (g, r) in enumerate(zip(got, ref)):
        assert g.T_prior.tobytes() == r.T_prior.tobytes(), k
        assert (g.status, g.iterations, g.converged) == (r.status, r.iterations, r.converged), k
        assert o.se3_log_distance(r.T, g.T) < 1e-8, k
        assert [list(x.analysis.degenerate_mask) for x in g.logs] == [list(x.analysis.degenerate_mask) for x in r.logs]
    for s, rs in enumerate(split(got, seq["seqs"])):
        assert rs[0].T_prior.tobytes() == seq["T_init"][s].tobytes()
        assert rs[0].iterations > 0


def single_runs(ctx, prm, res, radii=None):
    """every frame against set_source(its deskewed points) + icp_run(T_prior) on the context's target"""
    from dcreg_b200.api import IcpParams
    for k, r in enumerate(res):
        p = IcpParams.from_buffer_copy(prm)
        if radii is not None:
            p.search_radius = radii[k]
        ctx.set_source(r.deskewed)
        single = ctx.icp_run(p, r.T_prior)
        assert_same_run(r, single, dx_rel=1e-6)


def test_twist_deskew_equals_single_runs(ctx, imu):
    """Constant velocity and twist deskew: every frame is its single run; T_prior and deskewed_xyz follow the twins,
    the first frame of each sequence as given (the source filter's twin is the sessions' and the gyro test's concern)"""
    from dcreg_b200.api import compose_prior, constant_velocity_increment, deskew_points
    prm = params(search_radius=1.0)
    ctx.set_target(imu["map"], CELL)
    res = prior_map(ctx, lambda: ctx.icp_run_odometry(prm, imu["skewed"], imu["T_init"], None, map_frames=3,
                                                      **twist_kw(imu, source_voxel=0.0)))
    for s, rs in enumerate(split(res, imu["skewed"])):
        assert rs[0].T_prior.tobytes() == imu["T_init"][s].tobytes()
        for j, r in enumerate(rs):
            D = np.eye(4) if j < 2 else constant_velocity_increment(rs[j - 2].T, rs[j - 1].T)
            if j > 0:
                assert r.T_prior.tobytes() == compose_prior(rs[j - 1].T, D).tobytes(), (s, j)
            P = imu["skewed"][s][j]
            want = P if j == 0 else deskew_points(P, imu["stamps"][s][j], D)
            assert np.all(np.abs(r.deskewed - want) <= np.spacing(np.abs(want)) + 1e-12), (s, j)
    single_runs(ctx, prm, res)


def test_gyro_deskew_equals_single_runs(ctx, imu):
    """Gyro input, deskew and the adaptive threshold: every frame is its single run at its radius.  T_prior follows
    compose_prior(T_out[k-1], [G(tm_{k-1} -> tm_k) | t_D]) with the twin's D (api.gyro_increment) to FP64 rounding, the
    bound test_gpu_odometry_gyro holds it to (the device's sincos may differ from libm in the last bit); deskewed_xyz
    follows deskew_points_gyro to one float32 ulp or 1e-12 m and moved, and each sequence's first frame is as given; the
    radii follow the twin replayed with each sequence's first frame left out of its state, to the 8 ulps of
    test_gpu_odometry_adaptive (the model error's sine is the device's)"""
    from dcreg_b200.api import (adaptive_threshold_radius, adaptive_threshold_update, compose_prior, deskew_points_gyro,
                                gyro_increment)
    prm = params(search_radius=2.0)
    ctx.set_target(imu["map"], CELL)
    res = prior_map(ctx, lambda: ctx.icp_run_odometry(prm, imu["skewed"], imu["T_init"], None, map_frames=3,
                                                      **gyro_kw(imu, source_voxel=0.0)))
    th = threshold()
    tm = imu["ft"][:, 0] + 0.5 * imu["ft"][:, 1]
    k0 = 0
    for s, rs in enumerate(split(res, imu["skewed"])):
        assert rs[0].T_prior.tobytes() == imu["T_init"][s].tobytes()
        assert rs[0].deskewed.tobytes() == imu["skewed"][s][0].tobytes()
        state = (0.0, 0)
        for j, r in enumerate(rs):
            want = adaptive_threshold_radius(state, th.initial_threshold, prm.search_radius)
            assert abs(r.search_radius - want) <= 8 * np.spacing(want), (s, j)
            if j > 0:
                state = adaptive_threshold_update(state, r.T_prior, r.T, th.min_motion, th.max_range)
                k = k0 + j
                D = gyro_increment(imu["samples"][s], tm[k - 1], tm[k], rs[j - 2].T if j >= 2 else None, rs[j - 1].T,
                                   R_SI, BIAS)
                assert np.abs(r.T_prior - compose_prior(rs[j - 1].T, D)).max() < 1e-12, (s, j)
                P_in = imu["skewed"][s][j]
                twin = deskew_points_gyro(P_in, imu["stamps"][s][j], imu["ft"][k], tm[k - 1], imu["samples"][s],
                                          D[:3, 3], R_SI, BIAS)
                err = np.abs(r.deskewed.astype(np.float64) - twin.astype(np.float64))
                assert (err <= np.maximum(np.spacing(np.abs(twin)).astype(np.float64), 1e-12)).all(), (s, j)
                assert np.abs(twin - P_in).max() > 0.01                 # the sweep moved
        k0 += len(rs)
    single_runs(ctx, prm, res, [r.search_radius for r in res])


def test_gyro_session_first_push_without_gyro_input(ctx, imu):
    """A prior-map gyro session whose first push carries timestamps but no gyro input holds first frames alone: they
    register as the one call's first frames do, as given (not deskewed, no knot table read); the next frame then needs
    the first frame's mid-sweep time, which that push did not give, and its push is refused and commits nothing"""
    from dcreg_b200 import api
    prm = params(search_radius=2.0)
    ctx.set_target(imu["map"], CELL)
    one = prior_map(ctx, lambda: ctx.icp_run_odometry(prm, imu["skewed"], imu["T_init"], None, map_frames=3,
                                                      **gyro_kw(imu)))
    firsts = [rs[0] for rs in split(one, imu["skewed"])]
    ctx.set_prior_map(1)
    try:
        sess = ctx.odometry_session(prm, 2, imu["T_init"], "constant_velocity", map_frames=3, cell_size=CELL,
                                    source_voxel=0.3, adaptive=threshold(), gyro=gyro())
    finally:
        ctx.set_prior_map(0)
    with sess:
        got = sess.push([d[:1] for d in imu["skewed"]], want_log=True, want_cov=True,
                        timestamps=[t[:1] for t in imu["stamps"]], want_deskewed=True)
        assert [result_bytes(g) for g in got] == [result_bytes([f]) for f in firsts]
        for g, f in zip(got, firsts):
            assert g[0].deskewed.tobytes() == f.deskewed.tobytes()
            assert g[0].search_radius == f.search_radius
        with pytest.raises(api.DcregError) as e:
            sess.push([d[1:2] for d in imu["skewed"]], timestamps=[t[1:2] for t in imu["stamps"]],
                      frame_times=imu["ft"][[1, 6]], gyro_samples=imu["samples"])
        assert e.value.status == api.BAD_ARG and "unknown" in str(e.value)


def test_sparse_equals_dense(ctx, seq):
    """A prior-map call on A (a sparse row index) gives the bytes of the same call on B (a dense grid)"""
    prm = params()
    out = []
    for tgt in (seq["B"], seq["A"]):
        ctx.set_target(tgt, CELL)
        out.append(result_bytes(prior_map(ctx, lambda: ctx.icp_run_odometry(
            prm, seq["seqs"], seq["T_init"], None, "constant_velocity", map_frames=1, cell_size=CELL, want_log=True,
            want_cov=True))))
    assert out[0] == out[1]


def push_all(ctx, prm, d, chunks, gyro_on, fail_at=None, between=None):
    """d's sweeps pushed in chunks into a prior-map session (twist deskew, or gyro); fail_at: first a push without a
    target there, which must fail and commit nothing"""
    n = len(d["lens"])
    first = np.concatenate([[0], np.cumsum(d["lens"])])
    done, out = [0] * n, [[] for _ in range(n)]
    kw = dict(adaptive=threshold(), gyro=gyro()) if gyro_on else {}
    ctx.set_prior_map(1)
    try:
        sess = ctx.odometry_session(prm, n, d["T_init"], "constant_velocity", map_frames=3, cell_size=CELL,
                                    source_voxel=0.3, **kw)
    finally:
        ctx.set_prior_map(0)
    with sess:
        for i, cnt in enumerate(chunks):
            part = [d["skewed"][s][done[s]:done[s] + c] for s, c in enumerate(cnt)]
            ts = [d["stamps"][s][done[s]:done[s] + c] for s, c in enumerate(cnt)]
            gk = {}
            if gyro_on:
                rows = np.concatenate([np.arange(first[s] + done[s], first[s] + done[s] + c) for s, c in enumerate(cnt)])
                gk = dict(frame_times=d["ft"][rows.astype(int)], gyro_samples=d["samples"])

            def push():
                return sess.push(part, want_log=True, want_cov=True, timestamps=ts, want_deskewed=True, **gk)
            if i == fail_at:
                from dcreg_b200 import api
                bad = [[t.copy() for t in x] for x in ts]
                for x in bad:
                    if x:
                        x[0][0] = 2.0
                if any(bad):
                    with pytest.raises(api.DcregError):
                        sess.push(part, timestamps=bad, **gk)
            for s, r in enumerate(push()):
                out[s].extend(r)
            done = [a + c for a, c in zip(done, cnt)]
            if between:
                between(i)
    return out


@pytest.mark.parametrize("gyro_on", [False, True])
def test_sessions_equal_one_call(ctx, imu, gyro_on):
    """One frame per push, ragged pushes and sequences advancing unevenly give one call's bytes; a push with a bad
    timestamp fails and commits nothing"""
    prm = params(search_radius=2.0 if gyro_on else 1.0)
    ctx.set_target(imu["map"], CELL)
    kw = gyro_kw(imu) if gyro_on else twist_kw(imu)
    one = prior_map(ctx, lambda: ctx.icp_run_odometry(prm, imu["skewed"], imu["T_init"], None, map_frames=3, **kw))
    want = [result_bytes(rs) + [r.deskewed.tobytes() for r in rs] for rs in split(one, imu["skewed"])]
    if gyro_on:
        want = [w + [r.search_radius for r in rs] for w, rs in zip(want, split(one, imu["skewed"]))]
    lens = imu["lens"]
    for chunks in (one_per_push(lens), [[2, 0], [0, 3], [3, 4]], [[1, 1], [0, 4], [4, 0], [0, 2]]):
        got = push_all(ctx, prm, imu, chunks, gyro_on, fail_at=1)
        got_b = [result_bytes(rs) + [r.deskewed.tobytes() for r in rs] for rs in got]
        if gyro_on:
            got_b = [w + [r.search_radius for r in rs] for w, rs in zip(got_b, got)]
        assert got_b == want, chunks


def test_push_reads_the_target_at_push_time(ctx, seq):
    """A push without a target fails and commits nothing; a target swapped between pushes (B, then C: B without its
    points past x = 5 m, which changes the later frames' results) makes the later frames a call on C that starts from
    the carried pose.  Increments without deltas: frame 4's prior is T_out[3], so that call starts from the returned
    T_prior[4]; it sorts its frames under that pose rather than the session's dead-reckoned one, so it agrees to the
    rounding of FP64 sums grouped differently."""
    from dcreg_b200 import Context, api
    prm = params()
    s7 = seq["seqs"][1]
    C_map = np.ascontiguousarray(seq["B"][seq["B"][:, 0] < 5.0])
    with Context(0) as c2:
        c2.set_prior_map(1)
        with c2.odometry_session(prm, 1, seq["T_init"][1:2], map_frames=1, cell_size=CELL) as sess:
            with pytest.raises(api.DcregError) as e:
                sess.push([s7[:2]])
            assert e.value.status == api.BAD_ARG and "prior map" in str(e.value) and "target" in str(e.value)
            c2.set_target(seq["B"], CELL)
            a = sess.push([s7[:4]])[0]
            c2.set_target(C_map, CELL)
            b = sess.push([s7[4:]])[0]
        c2.set_target(seq["B"], CELL)
        full = c2.icp_run_odometry(prm, [s7], seq["T_init"][1:2], None, map_frames=1, cell_size=CELL)
        assert result_bytes(a) == result_bytes(full[:4])
        assert b[0].T_prior.tobytes() == full[4].T_prior.tobytes()
        assert any(x.T.tobytes() != y.T.tobytes() for x, y in zip(b, full[4:]))     # C is not B for these frames
        c2.set_target(C_map, CELL)
        on_c = c2.icp_run_odometry(prm, [s7[4:]], b[0].T_prior[None], None, map_frames=1, cell_size=CELL)
        assert len(on_c) == len(b)
        for x, y in zip(b, on_c):
            assert (x.status, x.iterations, x.converged) == (y.status, y.iterations, y.converged)
            assert o.se3_log_distance(y.T, x.T) < 1e-8


def test_context_costs_and_reproducibility(ctx, seq):
    """The context's source and target stay; launches do not depend on n_seqs; repeated calls give the same bytes"""
    prm = params()
    ctx.set_target(seq["B"], CELL)
    src = seq["seqs"][2][0]
    ctx.set_source(src)
    before = ctx.icp_run(prm, seq["T_init"][2])
    frames = seq["seqs"][2][:6]

    def call(n):
        return counted(ctx, lambda: prior_map(ctx, lambda: ctx.icp_run_odometry(
            prm, [frames] * n, np.repeat(seq["T_init"][2:3], n, 0), None, "constant_velocity", map_frames=1,
            cell_size=CELL, want_log=True)))
    (r1, l1), (r8, l8) = call(1), call(8)
    assert l1 == l8
    assert all(result_bytes(x) == result_bytes(r1) for x in split(r8, [frames] * 8))
    assert result_bytes(call(1)[0]) == result_bytes(r1)
    after = ctx.icp_run(prm, seq["T_init"][2])
    assert after.T.tobytes() == before.T.tobytes() and after.iterations == before.iterations


def test_bad_arguments(ctx, seq):
    """Every refusal of the prior map is DCREG_BAD_ARG and names it"""
    from dcreg_b200 import Context, api
    prm = params()
    s = [seq["seqs"][1][:3]]
    T0 = seq["T_init"][1:2]
    assert ctx.lib.dcreg_set_prior_map(ctx._h, 2) == api.BAD_ARG
    assert ctx.lib.dcreg_set_prior_map(ctx._h, -1) == api.BAD_ARG
    with pytest.raises(api.DcregError):
        ctx.set_prior_map(2)

    def refused(f, what="prior map"):
        with pytest.raises(api.DcregError) as e:
            prior_map(ctx, f)
        assert e.value.status == api.BAD_ARG and what in str(e.value), str(e.value)

    with Context(0) as c2:      # no target
        c2.set_prior_map(1)
        with pytest.raises(api.DcregError) as e:
            c2.icp_run_odometry(prm, s, T0, None, map_frames=1, cell_size=CELL)
        assert e.value.status == api.BAD_ARG and "prior map" in str(e.value)
    ctx.set_target(seq["B"], CELL)
    refused(lambda: ctx.icp_run_odometry(prm, s, T0, None, map_frames=1, cell_size=0.25))
    refused(lambda: ctx.icp_run_odometry_map(prm, s, T0, None, map_voxel=0.25, max_distance=10.0, cell_size=CELL))
    refused(lambda: ctx.icp_run_odometry(prm, s, T0, None, map_frames=0, cell_size=CELL, adaptive=threshold()))
    refused(lambda: ctx.odometry_map_session(prm, 1, T0, map_voxel=0.25, max_distance=10.0, cell_size=CELL))
    ctx.set_prior_map(1)
    try:
        sess = ctx.odometry_session(prm, 1, T0, map_frames=1, cell_size=CELL)
    finally:
        ctx.set_prior_map(0)
    with sess:
        sess.push(s)
        with pytest.raises(api.DcregError) as e:
            sess.local_map(0)
        assert e.value.status == api.BAD_ARG and "prior map" in str(e.value)
    with Context(0) as sharded:
        try:
            sharded.comm_init(sharded.comm_unique_id(), 0, 1)
        except api.DcregError:
            pytest.skip("no NCCL for the sharded-context case")
        sharded.set_target(seq["B"], CELL)
        sharded.set_prior_map(1)
        for f in (lambda: sharded.icp_run_odometry(prm, s, T0, None, map_frames=1, cell_size=CELL),
                  lambda: sharded.odometry_session(prm, 1, T0, map_frames=1, cell_size=CELL)):
            with pytest.raises(api.DcregError) as e:
                f()
            assert e.value.status == api.BAD_ARG and "prior map" in str(e.value) and "sharded" in str(e.value)
