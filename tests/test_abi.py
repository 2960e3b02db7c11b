"""The C-ABI library must exist in-tree, load, and export every symbol include/dcreg_b200.h declares.
No compute calls here (no GPU on the build box)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from dcreg_b200 import build, api
    build.build()                      # cross-compiles sm_90a with nvcc if stale
    return api.load_library()


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "dcreg_b200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(dcreg_[a-z0-9_]+)\s*\(", txt)) - {"dcreg_plane_callback"})


def test_header_and_binding_agree(lib):
    from dcreg_b200 import api
    assert header_symbols() == sorted(api.EXPORTS)


def test_every_symbol_exported(lib):
    for name in header_symbols():
        assert hasattr(lib, name), name


def test_abi_version_and_struct_sizes(lib):
    from dcreg_b200 import api
    assert lib.dcreg_abi_version() == 2
    p = api.default_params()
    assert p.search_radius == 1.0 and p.max_iterations == 30 and p.pcg_max_iter == 10
    assert p.cond_thresh == 10.0 and p.eig_thresh == 120.0 and p.kappa_target == 1.0 and p.std_reg_gamma == 0.01
    assert p.plane_thickness == 0.2 and p.weight_slope == 0.9 and p.weight_gate == 0.1 and p.min_effective_points == 10
    # sizes of the C structs as compiled by g++/nvcc (checked in test_struct_sizes_match_c below)
    assert ctypes.sizeof(api.IcpParams) == 128
    assert ctypes.sizeof(api.Analysis) == 1184 and ctypes.sizeof(api.IterLog) == 1672


def test_struct_sizes_match_c(tmp_path):
    import subprocess
    src = tmp_path / "sz.c"
    src.write_text('#include "dcreg_b200.h"\n#include <stdio.h>\nint main(){printf("%zu %zu %zu\\n",'
                   'sizeof(dcreg_icp_params),sizeof(dcreg_analysis),sizeof(dcreg_iter_log));return 0;}\n')
    exe = tmp_path / "sz"
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    out = subprocess.check_output([str(exe)], text=True).split()
    from dcreg_b200 import api
    assert [int(x) for x in out] == [ctypes.sizeof(api.IcpParams), ctypes.sizeof(api.Analysis),
                                     ctypes.sizeof(api.IterLog)]


def test_no_device_fails_loudly(lib):
    """Without a GPU the product refuses to run (no CPU fallback)."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from dcreg_b200 import api
    with pytest.raises(api.DcregError) as e:
        api.Context(0)
    assert e.value.status == api.NO_DEVICE


def test_sass_is_sm90a():
    import subprocess
    from dcreg_b200 import api
    out = subprocess.run(["cuobjdump", "--list-elf", api.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out
