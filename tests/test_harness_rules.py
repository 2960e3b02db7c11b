"""The test modules share one harness: no module imports a test module, the helpers every module needs are defined once
in harness.py, and harness.params builds the C3 settings for exactly the method it is given."""
import ast
import glob
import os

import pytest

import harness

TESTS = os.path.dirname(os.path.abspath(__file__))
SHARED = {"ctx", "rel_err", "assert_same_run", "c3_params", "log_bytes", "device_program_flags"}
FAKE_CTX = "test_odometry_binding.py"          # its ctx is a context over a fake library, not the device fixture
C3 = dict(search_radius=0.5, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0)


def modules():
    return sorted(glob.glob(os.path.join(TESTS, "**", "*.py"), recursive=True))


@pytest.fixture(scope="module")
def lib():
    from dcreg_b200 import api, build
    build.build()                      # cross-compiles sm_90a with nvcc if stale
    return api.load_library()


def test_no_module_imports_a_test_module():
    for path in modules():
        imported = set()
        for node in ast.walk(ast.parse(open(path).read(), path)):
            if isinstance(node, ast.Import):
                imported.update(a.name.split(".")[0] for a in node.names)
            elif isinstance(node, ast.ImportFrom) and node.module:
                imported.add(node.module.split(".")[0])
        assert not [m for m in imported if m.startswith("test_")], os.path.relpath(path, TESTS)


def test_shared_helpers_are_defined_only_in_the_harness():
    for path in modules():
        name = os.path.basename(path)
        if name == "harness.py":
            continue
        defined = set()
        for node in ast.parse(open(path).read(), path).body:
            if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
                defined.add(node.name)
            elif isinstance(node, (ast.Assign, ast.AnnAssign)):
                targets = node.targets if isinstance(node, ast.Assign) else [node.target]
                for t in targets:
                    if isinstance(t, ast.Name) and (t.id in SHARED or t.id == "METHODS" and isinstance(node.value, ast.Dict)):
                        defined.add(t.id)
        if name == FAKE_CTX:
            defined.discard("ctx")
        assert not defined & (SHARED | {"METHODS"}), (os.path.relpath(path, TESTS), sorted(defined & (SHARED | {"METHODS"})))


@pytest.mark.parametrize("method", ["Ours", "ME-TSVD"])
def test_params_are_the_c3_settings(lib, method):
    """Byte for byte the library's defaults with the C3 fields and the method's detection and handling"""
    from dcreg_b200.api import default_params
    ref = default_params()
    detection, handling = {"Ours": (1, 3), "ME-TSVD": (2, 5)}[method]       # SCHUR + PCG; FULL_EVD + TRUNCATED_SVD
    for k, v in (C3 | dict(detection=detection, handling=handling)).items():
        setattr(ref, k, v)
    assert bytes(harness.params(method)) == bytes(ref)


def test_params_run_the_method_named(lib):
    p = harness.params("FCN-SR")
    assert (p.detection, p.handling) == (4, 4)                  # FULL_SVD_CONDITION, SOLUTION_REMAPPING
    with pytest.raises(KeyError):
        harness.params("ME-SVD")
