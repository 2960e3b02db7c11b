"""Which C entry point each odometry and voxel-downsample method of the Python binding calls, and with which arguments.

A Context on a fake library records every call, checks its arguments as ctypes would against the real library's
argtypes, and names them after include/dcreg_b200.h.  The entry point names itself in dcreg_last_error, so the choice
is part of what a caller sees.  No GPU: the library is loaded, never called."""
import ctypes as C
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_arguments():
    """{function: its argument names in C order} for every dcreg_* function include/dcreg_b200.h declares"""
    txt = open(os.path.join(ROOT, "include", "dcreg_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return {name: [re.findall(r"\w+", a)[-1] for a in args.split(",")]
            for name, args in re.findall(r"\bint\s+(dcreg_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", txt)}


class FakeLib:
    """Records (function, {argument name: value}) for every call and returns DCREG_OK"""

    def __init__(self, real):
        self.real, self.calls, self.names = real, [], header_arguments()

    def __getattr__(self, name):
        argtypes = getattr(self.real, name).argtypes

        def call(*args):
            assert len(args) == len(argtypes) == len(self.names[name]), name
            for t, a in zip(argtypes, args):
                t.from_param(a)                                  # raises where ctypes would
            self.calls.append((name, dict(zip(self.names[name][1:], args[1:]))))
            return 0
        call.argtypes = argtypes
        return call


def is_pointer(t):
    return issubclass(t, (C._Pointer, C.c_void_p))


@pytest.fixture(scope="module")
def real():
    from dcreg_b200 import build, api
    build.build()                      # cross-compiles sm_90a with nvcc if stale
    return api.load_library()


@pytest.fixture
def ctx(real):
    from dcreg_b200 import api
    c = api.Context.__new__(api.Context)
    c.lib, c._h, c.n_source, c._lane_params = FakeLib(real), C.c_void_p(0x1000), 0, False
    yield c
    c._h = None


def scene():
    rng = np.random.default_rng(5)
    seqs = [[rng.random((5, 3), np.float32), rng.random((6, 3), np.float32)], [rng.random((4, 3), np.float32)]]
    stamps = [[np.full(len(f), 0.5, np.float32) for f in s] for s in seqs]
    return seqs, stamps, np.stack([np.eye(4)] * 2), np.stack([np.eye(4)] * 3)


def params():
    from dcreg_b200 import api
    return api.default_params(search_radius=0.5)


def assert_call(ctx, entry, scalars, null):
    """The last call: entry, exactly these non-pointer arguments, and exactly these pointer arguments NULL"""
    name, args = ctx.lib.calls[-1]
    assert name == entry
    types = dict(zip(ctx.lib.names[name][1:], getattr(ctx.lib.real, name).argtypes[1:]))
    assert {k: v for k, v in args.items() if not is_pointer(types[k])} == scalars
    assert {k for k, v in args.items() if v is None} == set(null)


RUN = dict(n_seqs=2, n_frames=3, stride=3, cell_size=0.5, map_frames=4, motion=0, log_cap=0)
FILTERS = dict(source_voxel=0.0, map_voxel=0.0, source_max_points=1, map_max_points=1)
DESKEW_NULL = {"timestamps", "cov", "deskewed_xyz", "log"}

ODOMETRY = {
    "plain": (dict(), "dcreg_icp_run_odometry", RUN, {"cov", "log"}),
    "logs_and_covariances": (dict(want_log=True, want_cov=True), "dcreg_icp_run_odometry", RUN | dict(log_cap=30),
                             set()),
    "constant_velocity": (dict(motion="constant_velocity"), "dcreg_icp_run_odometry", RUN | dict(motion=1),
                          {"deltas", "cov", "log"}),
    "voxels": (dict(source_voxel=0.3, map_voxel=0.25), "dcreg_icp_run_odometry_voxel",
               RUN | dict(source_voxel=0.3, map_voxel=0.25), {"cov", "log"}),
    "caps": (dict(map_voxel=0.25, map_max_points=3), "dcreg_icp_run_odometry_voxel_n",
             RUN | FILTERS | dict(map_voxel=0.25, map_max_points=3), {"cov", "log"}),
    "source_cap": (dict(source_voxel=0.3, source_max_points=2), "dcreg_icp_run_odometry_voxel_n",
                   RUN | FILTERS | dict(source_voxel=0.3, source_max_points=2), {"cov", "log"}),
    "timestamps": (dict(timestamps=True, map_voxel=0.25), "dcreg_icp_run_odometry_deskew",
                   RUN | FILTERS | dict(map_voxel=0.25), {"cov", "deskewed_xyz", "log"}),
    "want_deskewed": (dict(want_deskewed=True), "dcreg_icp_run_odometry_deskew", RUN | FILTERS,
                      {"timestamps", "cov", "log"}),
    "adaptive": (dict(adaptive=True, timestamps=True, map_max_points=4), "dcreg_icp_run_odometry_adaptive",
                 RUN | FILTERS | dict(map_max_points=4, max_distance=0.0), {"cov", "deskewed_xyz", "log"}),
    "want_radius": (dict(want_radius=True), "dcreg_icp_run_odometry_adaptive", RUN | FILTERS | dict(max_distance=0.0),
                    {"adaptive"} | DESKEW_NULL),
}


def settle(kw, stamps):
    """kw with timestamps = True and adaptive = True made real"""
    from dcreg_b200 import api
    kw = dict(kw)
    if kw.get("timestamps"):
        kw["timestamps"] = stamps
    if kw.get("adaptive"):
        kw["adaptive"] = api.AdaptiveThreshold()
    return kw


@pytest.mark.parametrize("case", sorted(ODOMETRY))
def test_icp_run_odometry(ctx, case):
    kw, entry, scalars, null = ODOMETRY[case]
    seqs, stamps, T_init, deltas = scene()
    D = None if kw.get("motion") == "constant_velocity" else deltas
    res = ctx.icp_run_odometry(params(), seqs, T_init, D, map_frames=4, cell_size=0.5, **settle(kw, stamps))
    assert len(res) == 3 and len(ctx.lib.calls) == 1
    assert_call(ctx, entry, scalars, null)


MAP = dict(n_seqs=2, n_frames=3, stride=3, cell_size=0.5, motion=0, log_cap=0) | FILTERS | dict(map_voxel=0.25,
                                                                                              max_distance=7.0)


@pytest.mark.parametrize("adaptive", [False, True], ids=["map", "adaptive"])
def test_icp_run_odometry_map(ctx, adaptive):
    seqs, stamps, T_init, deltas = scene()
    kw = dict(adaptive=True) if adaptive else dict()
    ctx.icp_run_odometry_map(params(), seqs, T_init, deltas, map_voxel=0.25, max_distance=7.0, cell_size=0.5,
                             **settle(kw, stamps))
    if adaptive:
        assert_call(ctx, "dcreg_icp_run_odometry_adaptive", MAP | dict(map_frames=0), DESKEW_NULL)
    else:
        assert_call(ctx, "dcreg_icp_run_odometry_map", MAP, DESKEW_NULL)


OPEN = dict(n_seqs=2, cell_size=0.5, motion=0) | FILTERS
SESSIONS = {
    "window": ("dcreg_odometry_open", OPEN | dict(map_frames=4, source_voxel=0.3)),
    "window_adaptive": ("dcreg_odometry_open_adaptive", OPEN | dict(map_frames=4, source_voxel=0.3, max_distance=0.0)),
    "map": ("dcreg_odometry_open_map", OPEN | dict(map_voxel=0.25, max_distance=7.0)),
    "map_adaptive": ("dcreg_odometry_open_adaptive", OPEN | dict(map_frames=0, map_voxel=0.25, max_distance=7.0)),
}


@pytest.mark.parametrize("timestamps", [False, True], ids=["plain", "timestamps"])
@pytest.mark.parametrize("kind", sorted(SESSIONS))
def test_session_open_and_push(ctx, kind, timestamps):
    from dcreg_b200 import api
    seqs, stamps, T_init, deltas = scene()
    adaptive = api.AdaptiveThreshold() if kind.endswith("adaptive") else None
    if kind.startswith("window"):
        sess = ctx.odometry_session(params(), 2, T_init, map_frames=4, cell_size=0.5, source_voxel=0.3,
                                    adaptive=adaptive)
    else:
        sess = ctx.odometry_map_session(params(), 2, T_init, map_voxel=0.25, max_distance=7.0, cell_size=0.5,
                                        adaptive=adaptive)
    entry, scalars = SESSIONS[kind]
    assert_call(ctx, entry, scalars, set())
    out = sess.push(seqs, deltas, timestamps=stamps if timestamps else None)
    assert [len(r) for r in out] == [2, 1]
    push = dict(n_frames=3, stride=3, log_cap=0)
    if adaptive is not None:
        null = {"cov", "deskewed_xyz", "log"} | (set() if timestamps else {"timestamps"})
        assert_call(ctx, "dcreg_odometry_push_adaptive", push, null)
    elif timestamps:
        assert_call(ctx, "dcreg_odometry_push_deskew", push, {"cov", "deskewed_xyz", "log"})
    else:
        assert_call(ctx, "dcreg_odometry_push", push, {"cov", "log"})
    sess.close()
    assert ctx.lib.calls[-1][0] == "dcreg_odometry_close"


@pytest.mark.parametrize("max_points,min_spacing,entry", [(1, 0.0, "dcreg_voxel_downsample_n"),
                                                          (4, 0.0, "dcreg_voxel_downsample_n"),
                                                          (4, 0.1, "dcreg_voxel_downsample_spaced")])
def test_voxel_downsample(ctx, max_points, min_spacing, entry):
    seqs, _, _, _ = scene()
    out = ctx.voxel_downsample([f for s in seqs for f in s], 0.5, max_points, min_spacing)
    assert len(out) == 3
    scalars = dict(n_clouds=3, stride=3, voxel=0.5, max_points=max_points)
    if entry == "dcreg_voxel_downsample_spaced":
        scalars["min_spacing"] = min_spacing
    assert_call(ctx, entry, scalars, set())
