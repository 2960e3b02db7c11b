"""dcreg_b200/csrc/se3.cuh (the device's SE(3) log / exp of the odometry's motion compensation) built as host C++ and
held against the NumPy twin on random motions: at most 4 FP64 ulp on every twist entry (of the twist's largest entry),
and every deskewed point within the accuracy contract (one float32 ulp or 1e-12 m) of the twin."""
import subprocess

import numpy as np

from dcreg_b200 import api
from harness import tool_program


def random_motions(rng, n):
    """Twists with angles spread from 0 to pi (log-uniform small ones, a few at the ends), exponentiated by the twin"""
    ang = np.concatenate([[0.0, 1e-12, 1e-9, 1e-6, 1e-3, 0.5, 2.0, np.pi - 1e-6, np.pi - 1e-3],
                          10.0 ** rng.uniform(-8, 0, n // 2), rng.uniform(0, np.pi, n - n // 2 - 9)])
    axis = rng.normal(size=(len(ang), 3))
    axis /= np.linalg.norm(axis, axis=1, keepdims=True)
    xi = np.concatenate([rng.uniform(-2, 2, (len(ang), 3)), axis * ang[:, None]], axis=1)
    D = np.array([api.se3_exp(x) for x in xi])
    D[0] = np.eye(4)                                        # the exact identity
    D[1, :3, 3] = [0.5, -0.25, 0.0]                         # a pure translation
    return D


def test_host_build_matches_the_twin(tmp_path):
    exe = tool_program(tmp_path, "test_se3.cpp", compiler="c++")
    rng = np.random.default_rng(2024)
    D = random_motions(rng, 400)
    n_pts = 20_000
    m = rng.integers(0, len(D), n_pts).astype(np.int32)
    tau = rng.uniform(0, 1, n_pts).astype(np.float32)
    tau[:50] = 0.5
    P = rng.uniform(-40, 40, (n_pts, 3)).astype(np.float32)
    rec = np.zeros(n_pts, dtype=[("m", "<i4"), ("tau", "<f4"), ("p", "<f4", 3)])
    rec["m"], rec["tau"], rec["p"] = m, tau, P
    inp, out = tmp_path / "in.bin", tmp_path / "out.bin"
    with open(inp, "wb") as f:
        f.write(np.int32(len(D)).tobytes() + np.ascontiguousarray(D).tobytes() + np.int32(n_pts).tobytes() + rec.tobytes())
    res = subprocess.run([str(exe), str(inp), str(out)], capture_output=True, text=True)
    assert res.returncode == 0 and "SE3_HOST_OK" in res.stdout, res.stdout + res.stderr
    raw = np.fromfile(out, dtype=np.uint8)
    xi_host = raw[:len(D) * 48].view(np.float64).reshape(-1, 6)
    pts_host = raw[len(D) * 48:].view(np.float32).reshape(-1, 3)
    xi_twin = np.array([api.se3_log(d) for d in D])
    assert (xi_host[0] == 0.0).all() and (xi_twin[0] == 0.0).all()
    scale = np.spacing(np.abs(xi_twin).max(axis=1, keepdims=True))
    assert (np.abs(xi_host - xi_twin) <= 4 * scale).all(), np.max(np.abs(xi_host - xi_twin) / scale)
    twin = np.empty_like(P)
    for k in range(len(D)):
        rows = np.nonzero(m == k)[0]
        twin[rows] = api.deskew_points(P[rows], tau[rows], D[k])
    ulp = np.spacing(np.abs(twin)).astype(np.float64)
    err = np.abs(pts_host.astype(np.float64) - twin.astype(np.float64))
    assert (err <= np.maximum(ulp, 1e-12)).all(), float(np.max(err / ulp))
    assert pts_host[:50].tobytes() == P[:50].tobytes()      # tau = 0.5: copied
