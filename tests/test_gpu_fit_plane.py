"""The loop's plane fit with correctly rounded FP64 primitives (dcreg_b200/csrc/cr_fp64.cuh), built for sm_90a with the
library's flags and run on the device:
  * crf::div / crf::sqrt equal __ddiv_rn / __dsqrt_rn bit for bit wherever their range flag is clear (2^27 operands
    each), and the flag is set on zero, subnormal, huge, infinite and NaN operands;
  * corr::fit_plane_reg equals the fit as it was with plain `/` and `sqrt` (kept in tools/test_fit_plane.cu) in ok, n
    and d, bit for bit, on the QR check's 400 k systems, lattices, pivot ties, all row orders of five-point sets,
    neighbourhoods that must take the fallback, and the 5-NN neighbourhoods of C2 and corridor clouds."""
import subprocess

import numpy as np
import pytest

from harness import tool_program


@pytest.mark.gpu
def test_correctly_rounded_primitives_on_the_device(tmp_path):
    exe = tool_program(tmp_path, "test_cr_fp64.cu", compiler="device", skip_missing=False)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    print(res.stdout)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "CR_FP64_OK" in res.stdout


def _neighbourhoods(pts, n_queries, seed):
    """Rows of the five nearest target points (in distance order) around jittered target points."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(seed)
    q = pts[rng.integers(0, len(pts), n_queries)] + rng.normal(0.0, 0.05, (n_queries, 3)).astype(np.float32)
    _, idx = cKDTree(pts.astype(np.float64)).query(q.astype(np.float64), k=5)
    return idx.astype(np.int32)


@pytest.mark.gpu
def test_plane_fit_is_bit_identical_to_the_plain_fit(tmp_path):
    from dcreg_b200.scenes import make_cylinder, make_corridor
    exe = tool_program(tmp_path, "test_fit_plane.cu", compiler="device", skip_missing=False)
    cyl = np.asarray(make_cylinder(100_000, seed=42), dtype=np.float32)
    cor = np.asarray(make_corridor(100_000, seed=44), dtype=np.float32)
    pts = np.concatenate([cyl, cor])
    keys = np.concatenate([_neighbourhoods(cyl, 200_000, 1), len(cyl) + _neighbourhoods(cor, 200_000, 2)])
    p4 = np.zeros((len(pts), 4), dtype=np.float32)
    p4[:, :3] = pts
    p4.tofile(tmp_path / "pts.f32")
    keys.tofile(tmp_path / "keys.i32")
    res = subprocess.run([str(exe), str(tmp_path / "pts.f32"), str(tmp_path / "keys.i32")], capture_output=True, text=True)
    print(res.stdout)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "FIT_PLANE_OK" in res.stdout
    assert "qr_reg systems: 400000 systems x 2 gates, 0 mismatches" in res.stdout
