"""What the odometry and voxel GPU tests share: the scenes, the solver settings, the asserts, the twins of the window and
voxel maps, one driver that pushes a recording into a session in chunks, and the raw callers of the C entry points.

Each test module keeps its own scenario (sequence lengths, points per frame, voxel sizes, caps, distances) and passes
it in; module-scoped fixtures imported from here are still set up once per module."""
import ctypes as C

import numpy as np
import pytest

import dcreg_oracle as o

RADIUS = 0.5
CELL = 0.5
RAGGED = [[1, 2, 0], [0, 0, 5], [0, 3, 1], [0, 2, 6]]     # sequences of 1, 7 and 12 frames at different rates


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


def parking(lens=(1, 7, 12), n_scan=20_000):
    """sum(lens) frames of one path (about n_scan points each, 20 m range) with drifting odometry, cut into sequences of
    lens frames: (seqs, T_init the true pose of each sequence's first frame, deltas, frames, T_true)"""
    from dcreg_b200.scenes import make_parking_sequence
    frames, T_true, _, deltas, _ = make_parking_sequence(sum(lens), seed=71, n_scan=n_scan, max_range=20.0)
    b = np.concatenate([[0], np.cumsum(lens)])
    seqs = [list(frames[p:q]) for p, q in zip(b[:-1], b[1:])]
    return seqs, np.ascontiguousarray(T_true[b[:-1]]), deltas, frames, T_true


def parking_sweeps(lens=(5, 7), n_scan=20_000):
    """sum(lens) skewed sweeps of one path with per-point timestamps, in sequences of lens frames whose anchors are
    unskewed (an anchor is never deskewed); T_init the true pose of each sequence's first frame"""
    from dcreg_b200.scenes import make_parking_sweeps
    skewed, stamps, T_true, deltas, frames = make_parking_sweeps(sum(lens), seed=71, n_scan=n_scan, max_range=20.0)
    b = np.concatenate([[0], np.cumsum(lens)])
    for a in b[:-1]:
        skewed[a] = frames[a]
    cut = lambda x: [list(x[p:q]) for p, q in zip(b[:-1], b[1:])]        # noqa: E731
    return dict(skewed=cut(skewed), stamps=cut(stamps), unskewed=cut(frames),
                T_init=np.ascontiguousarray(T_true[b[:-1]]), deltas=deltas, T_true=T_true)


@pytest.fixture(scope="module")
def odo():
    """parking(): 20 frames of about 20 k points in sequences of 1, 7 and 12: (seqs, T_init, deltas)"""
    return parking()[:3]


@pytest.fixture(scope="module")
def sweeps():
    """parking_sweeps(): 12 sweeps of about 20 k points in sequences of 5 and 7"""
    return parking_sweeps()


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


def crowded_clouds():
    """clouds_of_every_case() plus a cloud with one voxel holding 6000 points, interleaved with a sparse background and
    repeated at its end"""
    rng = np.random.default_rng(31)
    crowd = rng.uniform(0.01, 0.24, (6000, 3)).astype(np.float32)
    background = rng.uniform(-30, 30, (3000, 3)).astype(np.float32)
    crowded = np.concatenate([rng.permutation(np.concatenate([crowd, background])), crowd])
    return clouds_of_every_case() + [crowded]


def params(method="Ours", **over):
    from dcreg_b200 import default_params
    det, hand = ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG") if method == "Ours" else ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD")
    kw = dict(search_radius=RADIUS, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0,
              detection=det, handling=hand)
    kw.update(over)
    return default_params(**kw)


def one_per_push(lens):
    """Pushes of one frame per sequence while it has frames"""
    return [[1 if k < n else 0 for n in lens] for k in range(max(lens))]


# -- asserts --
def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def split(res, seqs):
    out, k = [], 0
    for s in seqs:
        out.append(res[k:k + len(s)])
        k += len(s)
    return out


def seq_results(res, seqs):
    return [list(r) for r in split(res, seqs)]


def assert_same_run(b, single, logs=True):
    assert (b.status, b.iterations, b.converged) == (single.status, single.iterations, single.converged)
    assert o.se3_log_distance(single.T, b.T) < 1e-8
    if not logs:
        return
    assert len(b.logs) == len(single.logs)
    for x, y in zip(b.logs, single.logs):
        assert x.n_effective == y.n_effective and x.n_corr_pt == y.n_corr_pt
        assert list(x.analysis.degenerate_mask) == list(y.analysis.degenerate_mask)
        if x.status == 0:
            assert rel_err(np.array(x.H27), np.array(y.H27)) < 1e-8
            assert np.max(np.abs(np.array(x.dx) - np.array(y.dx))) < 1e-8


def assert_anchor(r, T0):
    T0 = np.ascontiguousarray(T0, dtype=np.float64)
    assert r.T.tobytes() == T0.tobytes() and r.T_prior.tobytes() == T0.tobytes()
    assert (r.iterations, r.converged, r.status) == (0, 0, 0)
    assert len(r.logs) == 0
    if r.cov is not None:
        assert r.cov.tobytes() == (np.eye(6) * 1e6).tobytes()


def assert_priors(res, seqs, T_init, deltas, motion="increments"):
    from dcreg_b200.api import compose_prior, constant_velocity_increment
    k = 0
    for s, rs in enumerate(split(res, seqs)):
        assert rs[0].T_prior.tobytes() == np.ascontiguousarray(T_init[s]).tobytes()
        for j in range(1, len(rs)):
            if motion == "constant_velocity":
                D = np.eye(4) if j == 1 else constant_velocity_increment(rs[j - 2].T, rs[j - 1].T)
            else:
                D = np.eye(4) if deltas is None else deltas[k + j - 1]
            assert rs[j].T_prior.tobytes() == compose_prior(rs[j - 1].T, D).tobytes(), (s, j)
        k += len(rs)


def log_bytes(rec):
    r = type(rec).from_buffer_copy(bytes(rec))
    r.iter_time_ms = 0.0
    return bytes(r)


def result_bytes(res):
    return [(r.status, r.iterations, r.converged, r.n_points, r.T.tobytes(), r.T_prior.tobytes(),
             None if r.cov is None else r.cov.tobytes(), [log_bytes(x) for x in r.logs]) for r in res]


def assert_same(a_seqs, b_seqs):
    assert [len(x) for x in a_seqs] == [len(x) for x in b_seqs]
    for s, (xa, xb) in enumerate(zip(a_seqs, b_seqs)):
        for k, (a, b) in enumerate(zip(xa, xb)):
            where = (s, k)
            assert (a.status, a.iterations, a.converged, a.n_points) == (b.status, b.iterations, b.converged, b.n_points), where
            assert a.T.tobytes() == b.T.tobytes(), where
            assert a.T_prior.tobytes() == b.T_prior.tobytes(), where
            assert (a.cov is None) == (b.cov is None), where
            if a.cov is not None:
                assert a.cov.tobytes() == b.cov.tobytes(), where
            assert len(a.logs) == len(b.logs), where
            assert [log_bytes(x) for x in a.logs] == [log_bytes(y) for y in b.logs], where


def assert_same_flat(a, b, radius=False):
    """assert_same of two flat result lists, .deskewed byte for byte, and with radius .search_radius too"""
    assert_same([a], [b])
    for x, y in zip(a, b):
        assert (x.deskewed is None) == (y.deskewed is None)
        if x.deskewed is not None:
            assert x.deskewed.tobytes() == y.deskewed.tobytes()
        if radius:
            assert x.search_radius == y.search_radius


# -- twins --
def source_points(P, sv, cap=1):
    """F_s(P): the source filter voxel_downsample(P, sv, cap), or P itself for sv = 0"""
    from dcreg_b200.api import voxel_downsample
    return voxel_downsample(P, sv, cap)[0] if sv else P


def window_map(seq, rs, k, map_frames, sv=0.0, mv=0.0, caps=(1, 1), spacing=0.0, frames=None):
    """The twin's window map of frame k: voxel_downsample(M, mv, caps[1], spacing) (M itself for mv = 0) of M, the
    concatenation of map_points(T_out[j], F_s(frame j)) over the window (frames: the frames as they enter the maps,
    e.g. deskewed, instead of F_s(seq[j]))"""
    from dcreg_b200.api import map_points, voxel_downsample
    M = np.concatenate([map_points(rs[j].T, frames[j] if frames is not None else source_points(seq[j], sv, caps[0]))
                        for j in range(max(0, k - map_frames), k)])
    return voxel_downsample(M, mv, caps[1], spacing)[0] if mv else M


def twin_maps(seq, rs, sv, mv, cap, dist, spacing=0.0, frames=None):
    """The twin's voxel maps M_1 .. M_n of one sequence from its results: M_{k+1} = voxel_map_update(M_k, F_s(frame k),
    T_out[k], mv, cap, dist, spacing) (frames: the frames as inserted, e.g. deskewed; default F_s(seq[k]))"""
    from dcreg_b200.api import voxel_map_update
    M = np.zeros((0, 3), np.float32)
    out = [None]
    for k in range(len(rs)):
        P = frames[k] if frames is not None else source_points(seq[k], sv)
        M = voxel_map_update(M, P, rs[k].T, mv, cap, dist, spacing)
        out.append(M)
    return out


def reconstruct(ctx, prm, seq, rs, k, map_frames, sv=0.0, mv=0.0, caps=(1, 1), cell=CELL):
    """Frame k of a window call as the single run set_target(window map) + set_source(F_s(frame k)) + icp_run(T_prior)"""
    ctx.set_target(window_map(seq, rs, k, map_frames, sv, mv, caps), cell)
    ctx.set_source(source_points(seq[k], sv, caps[0]))
    return ctx.icp_run(prm, rs[k].T_prior)


def window_call(ctx, prm, seqs, T_init, deltas, **kw):
    """icp_run_odometry with a window longer than every sequence, logs and covariances"""
    return ctx.icp_run_odometry(prm, seqs, T_init, deltas, map_frames=max(len(s) for s in seqs) + 3, cell_size=CELL,
                                want_log=True, want_cov=True, **kw)


def map_call(ctx, prm, seqs, T_init, deltas, dist, **kw):
    """icp_run_odometry_map pruned at dist, logs and covariances"""
    return ctx.icp_run_odometry_map(prm, seqs, T_init, deltas, max_distance=dist, cell_size=CELL,
                                    want_log=True, want_cov=True, **kw)


# -- sessions --
def pushed(ctx, prm, seqs, T_init, chunks, deltas=None, *, voxel_map=False, stamps=None, ts_push=None, maps=None,
           between=None, want_log=False, want_cov=False, want_deskewed=False, **kw):
    """The recording pushed in `chunks` (per push, the frames of every sequence) into a session opened with kw and
    cell_size CELL (odometry_map_session with voxel_map, else odometry_session); returns one list of results per
    sequence.  deltas: the one call's deltas, cut into the pushes' entries.  stamps: per-frame timestamps nested like
    seqs, sent with push i where ts_push(i) (default: every push).  maps: a list that receives the local maps of every
    sequence after each push.  between(i): run after push i."""
    first = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
    done = [0] * len(seqs)
    out = [[] for _ in seqs]
    open_session = ctx.odometry_map_session if voxel_map else ctx.odometry_session
    with open_session(prm, len(seqs), T_init, cell_size=CELL, **kw) as sess:
        for i, cnt in enumerate(chunks):
            part = [seqs[s][done[s]:done[s] + c] for s, c in enumerate(cnt)]
            D = None
            if deltas is not None:
                D = np.concatenate([deltas[first[s] + done[s]:first[s] + done[s] + c] for s, c in enumerate(cnt)])
            ts = None
            if stamps is not None and (ts_push is None or ts_push(i)):
                ts = [stamps[s][done[s]:done[s] + c] for s, c in enumerate(cnt)]
            for s, r in enumerate(sess.push(part, D, want_log=want_log, want_cov=want_cov, timestamps=ts,
                                            want_deskewed=want_deskewed)):
                assert len(r) == cnt[s]
                out[s].extend(r)
            done = [d + c for d, c in zip(done, cnt)]
            if maps is not None:
                maps.append([sess.local_map(s) for s in range(len(seqs))])
            if between:
                between(i)
    assert done == [len(s) for s in seqs]
    return out


# -- the C entry points, for tables and outputs the Python binding would not build --
def _packed(clouds):
    xyz = np.ascontiguousarray(np.concatenate(clouds) if clouds else np.zeros((1, 3)), dtype=np.float32)
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int64)
    return xyz, off


def raw_odometry(ctx, entry, prm, seqs, T_init, deltas, log_cap=0, **values):
    """entry (a dcreg_icp_run_odometry* entry point) through api._odometry_call with every output filled with sentinels
    (-1) and the log records' iter_time_ms (a device clock reading) zeroed: (rc, dict of the output arrays).  values:
    the entry's other arguments by their C names (default cell_size CELL, map_frames 3, motion 0)."""
    from dcreg_b200 import api
    frames = [f for s in seqs for f in s]
    n = len(frames)
    xyz, off = _packed(frames)
    so = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int32)
    out = dict(T_prior=np.full((n, 4, 4), -1.0), T_out=np.full((n, 4, 4), -1.0), n_it=np.full(n, -1, np.int32),
               conv=np.full(n, -1, np.int32), st=np.full(n, -1, np.int32), cov=np.full((n, 36), -1.0),
               npts=np.full(n, -1, np.int64), log=np.zeros(max(n * log_cap, 1) * C.sizeof(api.IterLog), np.uint8))
    D = None if deltas is None else np.ascontiguousarray(deltas, dtype=np.float64)
    dp, ip = C.POINTER(C.c_double), lambda a: a.ctypes.data_as(C.POINTER(C.c_int))      # noqa: E731
    T0 = np.ascontiguousarray(T_init, dtype=np.float64)
    values = dict(cell_size=CELL, map_frames=3, motion=0) | values
    rc = api._odometry_call(
        ctx.lib, ctx._h, entry, params=C.byref(prm), n_seqs=len(seqs), seq_offsets=ip(so), n_frames=n,
        xyz=xyz.ctypes.data_as(C.POINTER(C.c_float)), frame_offsets=off.ctypes.data_as(C.POINTER(C.c_int64)), stride=3,
        T_init=T0.ctypes.data_as(dp), deltas=D.ctypes.data_as(dp) if D is not None else None,
        frame_points=out["npts"].ctypes.data_as(C.POINTER(C.c_int64)), T_prior=out["T_prior"].ctypes.data_as(dp),
        T_out=out["T_out"].ctypes.data_as(dp), n_iterations=ip(out["n_it"]), converged=ip(out["conv"]),
        status=ip(out["st"]), cov=out["cov"].ctypes.data_as(dp),
        log=C.cast(out["log"].ctypes.data, C.POINTER(api.IterLog)) if log_cap else None, log_cap=log_cap, **values)
    for rec in (api.IterLog * (n * log_cap)).from_buffer(out["log"]):
        rec.iter_time_ms = 0.0
    return rc, out


def raw_push(ctx, seq_off, frames, deltas=None, stride=3, offsets=None, n=None):
    """dcreg_odometry_push with T_out alone (the other outputs NULL): its return code"""
    from dcreg_b200 import api
    dp = C.POINTER(C.c_double)
    so = np.ascontiguousarray(seq_off, dtype=np.int32)
    n = int(so[-1]) if n is None else n
    xyz, off = _packed(frames)
    off = np.ascontiguousarray(off if offsets is None else offsets, np.int64)
    T_out = np.empty((max(n, 1), 4, 4))
    D = None if deltas is None else np.ascontiguousarray(deltas, dtype=np.float64)
    return api._odometry_call(ctx.lib, ctx._h, "dcreg_odometry_push", seq_offsets=so.ctypes.data_as(C.POINTER(C.c_int)),
                              n_frames=n, xyz=xyz.ctypes.data_as(C.POINTER(C.c_float)),
                              frame_offsets=off.ctypes.data_as(C.POINTER(C.c_int64)), stride=stride,
                              deltas=D.ctypes.data_as(dp) if D is not None else None, T_out=T_out.ctypes.data_as(dp),
                              log_cap=0)


def raw_downsample(ctx, entry, clouds, voxel, stride=3, want_index=True, **values):
    """entry (a dcreg_voxel_downsample* entry point) on (N_b, stride) clouds: (rc, points, offsets, index).  values:
    max_points and min_spacing, for the entry points that take them."""
    from dcreg_b200 import api
    xyz, off = _packed([np.asarray(c, np.float32)[:, :stride] for c in clouds])
    pts = np.empty((max(int(off[-1]), 1), 3), np.float32)
    kept = np.zeros(len(clouds) + 1, np.int64)
    idx = np.empty(max(int(off[-1]), 1), np.int64)
    i64 = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))                            # noqa: E731
    rc = api._odometry_call(ctx.lib, ctx._h, entry, n_clouds=len(clouds), xyz=xyz.ctypes.data_as(C.POINTER(C.c_float)),
                            offsets=i64(off), stride=stride, voxel=float(voxel),
                            out_xyz=pts.ctypes.data_as(C.POINTER(C.c_float)), out_offsets=i64(kept),
                            out_index=i64(idx) if want_index else None, **values)
    return rc, pts, kept, idx
