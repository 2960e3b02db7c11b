"""Host-side check of the register-resident pivoted QR used by the loop's plane fits: it must agree bit for bit with the
generic local-memory version (the one the seams and the legacy kernel use) on random, ill-conditioned and rank-deficient
5x3 systems.  Compiles tools/test_qr_reg.cu as HOST code with nvcc (no GPU involved)."""
import os
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def device_program_flags():
    """The library's nvcc flags for a standalone sm_90a program: without the shared-library and ptxas-report options,
    each dropped with its argument."""
    from dcreg_b200.build import NVCC_FLAGS
    flags, skip = [], False
    for f in NVCC_FLAGS:
        if skip:
            skip = False
        elif f in ("-Xcompiler", "-Xptxas"):
            skip = True
        elif f != "--shared":
            flags.append(f)
    assert "arch=compute_90a,code=sm_90a" in flags and "--fmad=true" in flags
    return flags


def test_register_qr_is_bit_identical_to_the_generic_qr(tmp_path):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = tmp_path / "test_qr_reg"
    subprocess.run([nvcc, "-O2", "-o", str(exe), os.path.join(ROOT, "tools", "test_qr_reg.cu")], check=True,
                   capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "400000 systems, 0 mismatches" in res.stdout


def test_fast_solve_step_pieces_on_the_host(tmp_path):
    """k2_fast.cuh (warm-started 3x3 Jacobi, pivoted L D L^T inverse with the FullPivLU invertibility decision) compiled
    as host code: residuals, orthogonality, warm == cold to rounding, decisions against a plain full-pivot LU."""
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = tmp_path / "test_k2_fast"
    subprocess.run([nvcc, "-O2", "-o", str(exe), os.path.join(ROOT, "tools", "test_k2_fast.cu")], check=True,
                   capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "K2_FAST_OK" in res.stdout


@pytest.mark.gpu
def test_fast_solve_step_pieces_on_the_device(tmp_path):
    """The same k2_fast.cuh checks built for sm_90a with the library's flags and run in a kernel, so the MUFU-seeded
    reciprocals are the ones the solve step uses; plus fast_rcp / fast_div against __drcp_rn / __ddiv_rn over
    [1e-300, 1e300] and fast_rsqrt against mpmath on a sample: at most the documented 2 ulp."""
    import mpmath
    import numpy as np
    from dcreg_b200.build import _nvcc
    exe = tmp_path / "test_k2_fast_dev"
    subprocess.run([_nvcc()] + device_program_flags() + ["-DK2F_DEVICE_TEST", "-o", str(exe), os.path.join(ROOT, "tools", "test_k2_fast.cu")],
                   check=True, capture_output=True, text=True)
    out = tmp_path / "rsqrt.bin"
    res = subprocess.run([str(exe), str(out)], capture_output=True, text=True)
    print(res.stdout)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "K2_FAST_OK" in res.stdout
    xy = np.fromfile(out, dtype=np.float64).reshape(-1, 2)
    assert len(xy) > 20_000 and xy[:, 0].min() <= 1e-300 and xy[:, 0].max() >= 1e300
    worst = 0
    with mpmath.workdps(40):
        for x, y in xy:
            ref = float(1 / mpmath.sqrt(mpmath.mpf(x)))
            worst = max(worst, abs(int(np.float64(y).view(np.int64)) - int(np.float64(ref).view(np.int64))))
    print(f"fast_rsqrt: max {worst} ulp from the correctly rounded 1/sqrt(x) on {len(xy)} points")
    assert worst <= 2


def test_loop_tile_plan(tmp_path):
    """loop_plan.hpp (how a run's source slots are cut into blocks of the iteration kernel) as plain host C++: coverage,
    tile bounds, resident-block cap, the small-cloud rule and the values used for the shipped cloud / C2 / C4 / C5; and
    which iteration-kernel instantiation and shared memory a plan runs, against launch_plan's former if-ladder."""
    gxx = shutil.which("g++")
    if not gxx:
        pytest.skip("g++ not available")
    exe = tmp_path / "test_loop_plan"
    subprocess.run([gxx, "-O2", "-std=c++17", "-o", str(exe), os.path.join(ROOT, "tools", "test_loop_plan.cpp")], check=True,
                   capture_output=True, text=True)
    res = subprocess.run([str(exe)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "LOOP_PLAN_OK" in res.stdout
