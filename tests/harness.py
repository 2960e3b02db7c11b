"""What the test modules share: the context, the six SO(3) methods and the C3 solver settings, the comparisons of two
runs, the programs of tools/ built on the host, and the small point sets and helpers more than one module uses.

Module-scoped fixtures imported from here are still set up once per module."""
import csv
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

import dcreg_oracle as o

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
RADIUS = 0.5
F = np.float32

METHODS = {                       # the six methods the CLI's SO(3) path recognises (icp_test_runner's test_methods)
    "Ours": ("SCHUR_CONDITION_NUMBER", "PRECONDITIONED_CG"),
    "NONE": ("NONE_DETE", "NONE_HAND"),
    "ME-SR": ("FULL_EVD_MIN_EIGENVALUE", "SOLUTION_REMAPPING"),
    "FCN-SR": ("FULL_SVD_CONDITION", "SOLUTION_REMAPPING"),
    "ME-TSVD": ("FULL_EVD_MIN_EIGENVALUE", "TRUNCATED_SVD"),
    "ME-TReg": ("FULL_EVD_MIN_EIGENVALUE", "STANDARD_REGULARIZATION"),
}


@pytest.fixture(scope="module")
def ctx():
    from dcreg_b200 import Context
    c = Context(0)
    yield c
    c.close()


# -- solver settings --
def params(method="Ours", radius=RADIUS, **over):
    """The C3 settings: 30 iterations, convergence at 1e-5 rad and 1e-3 m, kappa 10, and the method's detection and
    handling (an unknown name is a KeyError)"""
    from dcreg_b200 import default_params
    det, hand = METHODS[method]
    kw = dict(search_radius=radius, max_iterations=30, conv_thresh_rot=1e-5, conv_thresh_trans=1e-3, kappa_target=10.0,
              detection=det, handling=hand)
    kw.update(over)
    return default_params(**kw)


def oracle_method(method):
    """METHODS[method] as the oracle's DET_ / HAND_ constants"""
    det, hand = METHODS[method]
    return getattr(o, "DET_" + det.removesuffix("_DETE")), getattr(o, "HAND_" + hand.removesuffix("_HAND"))


def params_from(setup, method, **over):
    """The oracle's settings of a golden.json setup"""
    det, hand = oracle_method(method)
    p = o.Params(search_radius=setup["search_radius"], max_iterations=setup["max_iterations"],
                 conv_rot=setup["conv_rot"], conv_trans=setup["conv_trans"], cond_thresh=setup["cond_thresh"],
                 eig_thresh=setup["eig_thresh"], kappa_target=setup["kappa_target"],
                 std_reg_gamma=setup["std_reg_gamma"], use_weight_derivative=setup["use_weight_derivative"],
                 detection=det, handling=hand)
    for k, v in over.items():
        setattr(p, k, v)
    return p


def init_T(setup):
    x, y, z = setup["init_xyz"]
    r, p, yw = [math.radians(a) for a in setup["init_rpy_deg"]]
    return o.pose6d_to_matrix(x, y, z, r, p, yw)


# -- comparisons --
def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64); b = np.asarray(b, dtype=np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-300))


def assert_same_run(b, single, logs=True, dx_rel=0.0):
    """b is the run single to the rounding of FP64 sums grouped differently.  dx_rel widens the step's tolerance by that
    fraction of the step, for runs whose first updates are large enough to pass the sums' rounding on in proportion."""
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
            assert np.max(np.abs(np.array(x.dx) - np.array(y.dx))) < 1e-8 + dx_rel * np.max(np.abs(np.array(y.dx)))


def log_bytes(rec, fitness=True):
    """a log record's bytes with iter_time_ms (a device clock reading) zeroed, and without fitness its fitness too"""
    r = type(rec).from_buffer_copy(bytes(rec))
    r.iter_time_ms = 0.0
    if not fitness:
        r.fitness = 0.0
    return bytes(r)


# -- programs of tools/ built on the host --
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


def tool_program(dest, source, *flags, compiler="g++", skip_missing=True):
    """tools/<source> built into the directory dest; returns the executable.  compiler: "g++" (g++ -O2 -std=c++17),
    "c++" (the same with g++ or else c++), "nvcc" (nvcc -O2, host code) or "device" (device_program_flags()); flags
    follow these.  A missing compiler skips the test, or with skip_missing=False fails it."""
    if compiler in ("g++", "c++"):
        cxx = shutil.which("g++") or (shutil.which("c++") if compiler == "c++" else None)
        missing = None if cxx else ("g++ not available" if compiler == "g++" else "no host C++ compiler")
        cmd = [cxx, "-O2", "-std=c++17"]
    elif compiler == "nvcc":
        nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
        missing = None if os.path.exists(nvcc) else "nvcc not available"
        cmd = [nvcc, "-O2"]
    else:
        from dcreg_b200.build import _nvcc
        try:
            cmd, missing = [_nvcc()] + device_program_flags(), None
        except RuntimeError:
            cmd, missing = None, "nvcc not available"
    if missing:
        if skip_missing:
            pytest.skip(missing)
        raise RuntimeError(missing)
    exe = os.path.join(dest, os.path.splitext(source)[0])
    res = subprocess.run(cmd + list(flags) + ["-o", exe, os.path.join(ROOT, "tools", source)], capture_output=True,
                         text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    return exe


# -- the CLI's configuration --
def write_config(path, out_dir, setup, methods, extra_methods="", extra=""):
    x, y, z = setup["init_xyz"]
    r, p, w = setup["init_rpy_deg"]
    lines = "\n".join(f'  "{m}": [ "{METHODS[m][0]}", "{METHODS[m][1]}" ]' for m in methods)
    with open(path, "w") as f:
        f.write(f"""
test:
  num_runs: 1     # Number of test runs (set to 1 for single run)
  save_pcd: true  # Save aligned point clouds
  save_error_pcd: false
  visualize: false  # Enable visualization

# Output Options
output:
  save_csv: true

paths:
  folder_path: "{GOLD}/"
  output_folder: "{out_dir}/"
  source_pcd: "cylinder_7562.pcd"
  target_pcd: "cylinder_7562.pcd"

icp:
  search_radius: {setup['search_radius']}
  max_iterations: {setup['max_iterations']}
  error_threshold: 0.2  # Error threshold (m)

  CONVERGENCE_THRESH_TRANS: {setup['conv_trans']}
  CONVERGENCE_THRESH_ROT: {setup['conv_rot']}

  normal_nn: 5
  use_weight_derivative: {'true' if setup['use_weight_derivative'] else 'false'}

initial_noise:
  # x: 9.0
  x: {x}
  y: {y}
  z: {z}
  roll_deg: {r}
  pitch_deg: {p}
  yaw_deg: {w}

gt_pose:
  x: 0.0
  y: 0.0
  z: 0.0
  roll_deg: 0.0
  pitch_deg: 0.0
  yaw_deg: 0.

degeneracy:
  condition_threshold: {setup['cond_thresh']}  # DEGENERACY_THRES_COND
  eigenvalue_threshold: {setup['eig_thresh']}

method_params:

  standard_reg:
    gamma: {setup['std_reg_gamma']}  # STD_REG_GAMMA

  pcg:
    kappa_target: {setup['kappa_target']}
    tolerance: 1e-6
    max_iter: 10

  tsvd:
    singular_threshold: 120.0

icp_params:
  XICP_ENOUGH_INFO_THRESHOLD: 300.0      # ignored

test_methods:
#  "None": [ "NONE_DETE", "NONE_HAND" ]
{lines}
{extra_methods}
{extra}
""")


def dump(runner, cfg):
    out = subprocess.run([runner, "--dump-config", cfg], capture_output=True, text=True, check=True).stdout
    kv, methods = {}, []
    for line in out.splitlines():
        if line.startswith("method="):
            methods.append(line[len("method="):].split("|"))
        elif "=" in line and not line.startswith("="):
            k, v = line.split("=", 1)
            kv[k] = v
    return kv, methods


def read_csv(path):
    with open(path) as f:
        return list(csv.DictReader(f))


# -- point sets --
def dist2(q, pts, pairwise=False):
    """corr::dist2: float32 differences, products and sums, x then y then z, no fused operations.  Every query against
    every point ((m, n) result), or with pairwise=True query i against point i."""
    if not pairwise:
        q, pts = q[:, None, :], pts[None, :, :]
    ex = (q[..., 0] - pts[..., 0]).astype(F)
    ey = (q[..., 1] - pts[..., 1]).astype(F)
    ez = (q[..., 2] - pts[..., 2]).astype(F)
    return ((ex * ex).astype(F) + (ey * ey).astype(F)).astype(F) + (ez * ez).astype(F)


def ties_lattice():
    """the target of test_gpu_parity.py::test_loop_reuse_on_a_lattice_with_duplicates_and_ties: 0.25 m lattices,
    exact duplicates (floor[::5]) and a 0.05 m patch with ~300 points within 0.5 m of its inside"""
    g = np.arange(-6, 6, 0.25, dtype=F)
    X, Y = np.meshgrid(g, g)
    floor = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, F)], axis=1)
    wall = np.stack([X.ravel(), np.full(X.size, 6.0, F), (Y.ravel() + 6.0) * 0.5], axis=1)
    wall2 = np.stack([np.full(X.size, -6.0, F), X.ravel(), (Y.ravel() + 6.0) * 0.5], axis=1)
    d = np.arange(-1, 1, 0.05, dtype=F)
    DX, DY = np.meshgrid(d, d)
    dense = np.stack([DX.ravel(), DY.ravel(), np.zeros(DX.size, F)], axis=1)
    return np.concatenate([floor, wall, wall2, dense, floor[::5]]).astype(F)


def voxel_lattice(voxel):
    """Points on voxel faces on both sides of 0, their float32 neighbours below, and their mirror images"""
    g = np.arange(-6, 6, dtype=np.float64) * voxel
    P = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3).astype(np.float32)
    return np.concatenate([P, np.nextafter(P, np.float32(-np.inf)), -P])


def holes(rng, n=600):
    """(n, 4) points with NaN and infinite coordinates"""
    P = rng.uniform(-3, 3, (n, 4)).astype(np.float32)
    P[::7, 0] = np.nan
    P[3::11, 1] = np.inf
    P[5::13, 2] = -np.inf
    P[::17, 3] = np.nan                                                      # a 4th column does not matter
    return P


def direct(P, voxel):
    """The voxel filter's rule read literally: walk the points in order, the voxel of a finite point is
    floor(float64(c) * (1 / voxel)) per axis, and the first point to reach a voxel keeps it."""
    from dcreg_b200.api import VOXEL_LIMIT
    inv = 1.0 / voxel
    first = {}
    for i, p in enumerate(np.asarray(P, dtype=np.float32)):
        c = [float(np.float64(v)) for v in p[:3]]
        if not all(math.isfinite(v) for v in c):
            continue
        key = tuple(math.floor(v * inv) for v in c)
        assert all(-VOXEL_LIMIT <= k < VOXEL_LIMIT for k in key)
        first.setdefault(key, i)
    return np.array(sorted(first.values()), dtype=np.int64)


# -- designed systems through the host-plane loop (K1 + k2_step_kernel) --
def designed(kind, rng_seed=5, n=900, tilt=0.0):
    """Source points and world planes whose normal equations do not depend on the pose (to rounding): each point keeps
    its normal (rotated with the pose) and its residual rho.  Returns (points f32, normals, rho)."""
    rng = np.random.default_rng(rng_seed)
    if kind == "generic":                       # anisotropic translation and rotation blocks, all ratios distinct
        p = rng.uniform(-5.0, 5.0, (n, 3)) * np.array([1.0, 0.6, 0.3])
        u = rng.standard_normal((n, 3)) * np.array([1.0, 0.35, 0.12])
        nrm = u / np.linalg.norm(u, axis=1, keepdims=True)
        rho = rng.uniform(-2e-3, 2e-3, n)
    elif kind in ("box2", "box3"):              # axis-aligned faces of a symmetric box: equal Schur eigenvalues
        # every face point comes with its reflections in the face's two other coordinates, so the coupling H_Rt and
        # the off-diagonal entries vanish; box3: the same count per axis (H_tt = c I), box2: fewer on the z faces
        per = n // 24
        ext = np.array([4.0, 4.0, 0.5])
        p, nrm = [], []
        for ax in range(3):
            cnt = per if kind == "box3" or ax < 2 else max(1, per // 20)
            for sgn in (-1.0, 1.0):
                q = rng.uniform(-1.0, 1.0, (cnt, 3)) * ext
                q[:, ax] = sgn * ext[ax]
                for f in ((1, 1), (1, -1), (-1, 1), (-1, -1)):
                    s = np.ones(3); s[[a for a in range(3) if a != ax]] = f
                    p.append(q * s); nrm.append(np.tile(np.eye(3)[ax] * sgn, (cnt, 1)))
        p, nrm = np.concatenate(p), np.concatenate(nrm)
        rho = 1e-3 * rng.choice([-1.0, 1.0], len(p))                    # |rho| equal: every point has the same weight
    elif kind in ("rank2", "rank2_rot", "tilt"):   # translation block of rank 2 (+ tilt out of the plane)
        p = rng.uniform(-5.0, 5.0, (n, 3))
        ang = rng.uniform(0.0, 2.0 * math.pi, n)
        nrm = np.stack([np.cos(ang), np.sin(ang), np.zeros(n)], axis=1)
        if kind == "tilt":
            nrm[:, 2] = tilt * np.where(np.arange(n) % 2 == 0, 1.0, -1.0)
            nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        if kind == "rank2_rot":
            Rg = o.pose6d_to_matrix(0, 0, 0, 0.7, -0.4, 1.1)[:3, :3]
            nrm = nrm @ Rg.T
        rho = rng.uniform(-2e-3, 2e-3, n)
    else:
        raise ValueError(kind)
    return p.astype(np.float32), nrm, rho


def run_designed(ctx, sysd, prm, T0=None):
    p, nrm, rho = sysd
    p64 = p.astype(np.float64)

    def plane_fn(T):
        R, t = T[:3, :3], T[:3, 3]
        q = (p64 @ R.T + t).astype(np.float32).astype(np.float64)          # fl32(R p + t), as K1 forms it
        nw = nrm @ R.T
        planes = np.empty((len(p), 4))
        planes[:, :3] = nw
        planes[:, 3] = rho - np.einsum("kj,kj->k", nw, q)
        return planes, len(p)

    ctx.set_source(p)
    return ctx.icp_run_host_planes(prm, np.eye(4) if T0 is None else T0, plane_fn)
