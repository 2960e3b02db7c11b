"""CPU oracle (NumPy/SciPy twin) for the DCReg hot path.  TEST INFRASTRUCTURE ONLY.

This file restates, in plain FP64 NumPy, the one path of JokerJohn/DCReg that the
CUDA engine accelerates.  It is a *checker*: only ``tests/``, ``__graft_entry__.smoke()``
and ``bench.py``'s cpu_baseline / ``--impl reference`` leg may import it.  The product
(``dcreg_b200``) never imports anything from ``oracle/``.

Parity status: PINNED.  ``tests/test_oracle_golden.py`` checks this restatement against
the reference's own shipped dumps (SURVEY.md §8c: G1 = DCReg/dataset/icp_results,
G2 = results/simulation/table3_fig9_fig10, extracted into tests/golden/golden.json by
tests/golden/make_golden.py).  The reference binary itself cannot be built here
(Eigen/PCL/yaml-cpp/Ceres/TBB/Open3D absent; its "Ours" path is a stub in the released
source), see DESIGN.md.

Every function cites the reference file:line (relative to a checkout of the reference) it follows.
The stubbed "Ours" stages (Schur detection, preconditioner, PCG) follow the paper's
Alg. 1/3, Eq. 18-21, 43-46 as summarised in SURVEY.md §3.4 and are pinned by the shipped
per-iteration ``dx`` / ``T`` of the authors' own run (G2).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import numpy as np

# ----------------------------------------------------------------------------
# enums (DCReg/include/utils.hpp:106-121) - integer values are the C-ABI values
# ----------------------------------------------------------------------------
DET_NONE = 0
DET_SCHUR_CONDITION_NUMBER = 1
DET_FULL_EVD_MIN_EIGENVALUE = 2
DET_EVD_SUB_CONDITION = 3
DET_FULL_SVD_CONDITION = 4

HAND_NONE = 0
HAND_STANDARD_REGULARIZATION = 1
HAND_ADAPTIVE_REGULARIZATION = 2
HAND_PRECONDITIONED_CG = 3
HAND_SOLUTION_REMAPPING = 4
HAND_TRUNCATED_SVD = 5


@dataclass
class Params:
    """ICPParameters / Config defaults, DCReg/include/utils.hpp:82-103,132-171."""
    search_radius: float = 1.0
    max_iterations: int = 30
    conv_rot: float = 1e-5
    conv_trans: float = 1e-3
    cond_thresh: float = 10.0          # DEGENERACY_THRES_COND
    eig_thresh: float = 120.0          # DEGENERACY_THRES_EIG
    kappa_target: float = 1.0          # KAPPA_TARGET (yaml: method_params.pcg.kappa_target)
    pcg_tol: float = 1e-6
    pcg_max_iter: int = 10
    std_reg_gamma: float = 0.01
    use_weight_derivative: bool = False  # icp_test_runner.cpp:1691
    detection: int = DET_SCHUR_CONDITION_NUMBER
    handling: int = HAND_PRECONDITIONED_CG


# ----------------------------------------------------------------------------
# SE(3) helpers
# ----------------------------------------------------------------------------
def pose6d_to_matrix(x, y, z, roll, pitch, yaw):
    """Pose6D2Matrix, DCReg/include/utils.hpp:452-460: T = Trans * Rz * Ry * Rx (radians)."""
    cr, sr = math.cos(roll), math.sin(roll)
    cp, sp = math.cos(pitch), math.sin(pitch)
    cy, sy = math.cos(yaw), math.sin(yaw)
    Rx = np.array([[1, 0, 0], [0, cr, -sr], [0, sr, cr]], dtype=np.float64)
    Ry = np.array([[cp, 0, sp], [0, 1, 0], [-sp, 0, cp]], dtype=np.float64)
    Rz = np.array([[cy, -sy, 0], [sy, cy, 0], [0, 0, 1]], dtype=np.float64)
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = [x, y, z]
    return T


def skew(v):
    """MathUtils::skew, DCReg/include/math_utils.hpp:11-17."""
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]], dtype=np.float64)


def so3_exp(omega):
    """MathUtils::exp, math_utils.hpp:20-33 (Rodrigues; I + [w]x below 1e-10)."""
    omega = np.asarray(omega, dtype=np.float64)
    theta = float(np.linalg.norm(omega))
    if theta < 1e-10:
        return np.eye(3) + skew(omega)
    K = skew(omega / theta)
    return np.eye(3) + math.sin(theta) * K + (1.0 - math.cos(theta)) * (K @ K)


def so3_log(R):
    """Rotation vector of R (robust variant of math_utils.hpp:36-46; test metric only)."""
    c = max(-1.0, min(1.0, (np.trace(R) - 1.0) / 2.0))
    theta = math.acos(c)
    if abs(theta) < 1e-12:
        return 0.5 * np.array([R[2, 1] - R[1, 2], R[0, 2] - R[2, 0], R[1, 0] - R[0, 1]])
    w = theta / (2.0 * math.sin(theta)) * (R - R.T)
    return np.array([w[2, 1], w[0, 2], w[1, 0]])


def se3_log_distance(Ta, Tb):
    """|| log(Ta^-1 Tb) ||: rotation-vector norm and translation norm stacked (test metric)."""
    E = np.linalg.inv(Ta) @ Tb
    return float(np.linalg.norm(np.concatenate([so3_log(E[:3, :3]), E[:3, 3]])))


def boxplus(R, t, dx):
    """SE3State::boxplus, math_utils.hpp:158-166: R <- R exp(w), t <- t + R_old v."""
    return R @ so3_exp(dx[:3]), t + R @ dx[3:]


def pose_error(gt, T):
    """calculatePoseError, utils.hpp:497-535 (translation norm, |angle| in degrees)."""
    E = np.linalg.inv(gt) @ T
    c = max(-1.0, min(1.0, (np.trace(E[:3, :3]) - 1.0) / 2.0))
    return float(np.linalg.norm(E[:3, 3])), math.degrees(abs(math.acos(c)))


# ----------------------------------------------------------------------------
# PCD v0.7 binary reader (x y z intensity float32) - SURVEY.md Appendix B.3
# ----------------------------------------------------------------------------
def read_pcd_xyz(path):
    with open(path, "rb") as f:
        raw = f.read()
    pos = 0
    npts = None
    fields = sizes = None
    while True:
        end = raw.index(b"\n", pos)
        line = raw[pos:end].decode("ascii", "replace").strip()
        pos = end + 1
        tok = line.split()
        if not tok:
            continue
        if tok[0] == "FIELDS":
            fields = tok[1:]
        elif tok[0] == "SIZE":
            sizes = [int(s) for s in tok[1:]]
        elif tok[0] == "POINTS":
            npts = int(tok[1])
        elif tok[0] == "DATA":
            if tok[1] != "binary":
                raise ValueError("only DATA binary supported")
            break
    stride = sum(sizes)
    assert all(s == 4 for s in sizes)
    arr = np.frombuffer(raw, dtype=np.float32, count=npts * (stride // 4), offset=pos)
    arr = arr.reshape(npts, stride // 4)
    ix, iy, iz = fields.index("x"), fields.index("y"), fields.index("z")
    return np.ascontiguousarray(arr[:, [ix, iy, iz]])


# ----------------------------------------------------------------------------
# Stage S1: correspondences + plane fit + residual + weight
# ----------------------------------------------------------------------------
def transform_points_f32(src_f32, R, t):
    """pointBodyToGlobal, DCReg/include/utils.hpp:630-636: FP64 math, float32 store."""
    q = src_f32.astype(np.float64) @ R.T + t
    return q.astype(np.float32)


def build_tree(tgt_f32):
    from scipy.spatial import cKDTree
    return cKDTree(tgt_f32.astype(np.float64))


def fit_planes(nb):
    """icp_test_runner.cpp:1727-1773.  nb: (K,5,3) float64 neighbour coords.

    Least-squares solve of nb @ x = -1 (reference: 5x3 colPivHouseholderQr).  Here: batched
    pseudo-inverse (agrees with the QR solution to rounding for full-rank systems and yields a
    zero component for an all-zero column, like Eigen's pivoted solve).  On other rank-deficient
    neighbourhoods (collinear or duplicated points) the minimum-norm solution differs from the
    pivoted QR's basic one; those are pinned by dcreg_oracle_rows.qr53, the operation-for-operation
    restatement of the kernel's QR.  This whole-loop oracle keeps pinv: it is a fast, independent
    route to the shipped golden runs, whose neighbourhoods are full rank or have zero columns.
    Returns n (K,3), d (K,), ok (K,) [norm >= 1e-6 and thickness gate passed].
    """
    K = nb.shape[0]
    b = -np.ones((K, 5, 1))
    x = (np.linalg.pinv(nb) @ b)[:, :, 0]
    ps = np.linalg.norm(x, axis=1)
    ok = ps >= 1e-6
    ps_safe = np.where(ok, ps, 1.0)
    n = x / ps_safe[:, None]
    d = 1.0 / ps_safe
    dist = np.einsum("kj,kij->ki", n, nb) + d[:, None]
    ok &= np.max(dist * dist, axis=1) < 0.2 * 0.2
    return n, d, ok


@dataclass
class Correspondences:
    """Per-source-slot outputs of S1 (before compaction), all length N."""
    valid: np.ndarray        # bool: s > 0.1 and all gates passed  (laserCloudOriSurfFlag)
    n: np.ndarray            # (N,3) unit normal (FP64)
    d: np.ndarray            # (N,) plane offset
    r: np.ndarray            # (N,) raw residual n.q + d
    s: np.ndarray            # (N,) weight
    ds_dr: np.ndarray        # (N,) weight derivative (0 unless use_weight_derivative)
    n_pt: int                # correspondence_pt_count (5th NN within radius)
    has_plane: np.ndarray = None   # bool: plane fit passed the norm + thickness gates


def find_correspondences(src_f32, tgt_f32, tree, R, t, radius, use_wd):
    """icp_test_runner.cpp:1714-1813."""
    N = src_f32.shape[0]
    q32 = transform_points_f32(src_f32, R, t)
    dist, idx = tree.query(q32.astype(np.float64), k=5)
    # FLANN returns float32 squared distances; the gate compares d2[4] < radius^2 (line 1726)
    d2 = (dist[:, 4] * dist[:, 4]).astype(np.float32)
    near = np.isfinite(dist[:, 4]) & (d2.astype(np.float64) < radius * radius)
    n = np.zeros((N, 3)); d = np.zeros(N); r = np.zeros(N); s = np.zeros(N); ds = np.zeros(N)
    valid = np.zeros(N, dtype=bool)
    has_plane = np.zeros(N, dtype=bool)
    sel = np.nonzero(near)[0]
    if sel.size:
        nb = tgt_f32[idx[sel]].astype(np.float64)          # (K,5,3)
        nn, dd, ok = fit_planes(nb)
        q = q32[sel].astype(np.float64)
        rr = np.einsum("kj,kj->k", nn, q) + dd             # line 1774
        ss = np.maximum(0.0, 1.0 - 0.9 * np.abs(rr))       # line 1776
        dsdr = np.zeros_like(rr)
        if use_wd:                                         # lines 1780-1783
            m = (ss > 0.0) & (ss < 1.0)
            dsdr[m] = np.where(rr[m] > 0, -0.9, 0.9)
        keep = ok & (ss > 0.1)                             # line 1785
        n[sel] = nn; d[sel] = dd; r[sel] = rr; s[sel] = ss; ds[sel] = dsdr
        valid[sel] = keep
        has_plane[sel] = ok
    return Correspondences(valid, n, d, r, s, ds, int(near.sum()), has_plane)


# ----------------------------------------------------------------------------
# Stages S4-S5: Jacobian + normal equations
# ----------------------------------------------------------------------------
def build_rows(src_f32, corr: Correspondences, R):
    """icp_test_runner.cpp:1863-1907 + math_utils.hpp:102-121.

    The reference stores coeff = (s*n, s*r) in a float32 PointT (lines 1786-1790) and rebuilds
    the normal as float32(s*n)/s (line 1889) and b = -float32(s*r) (line 1906).  Both roundings
    are reproduced here.
    """
    v = corr.valid
    p = src_f32[v].astype(np.float64)
    s = corr.s[v]; r = corr.r[v]; ds = corr.ds_dr[v]
    wn32 = (s[:, None] * corr.n[v]).astype(np.float32).astype(np.float64)
    sr32 = (s * r).astype(np.float32).astype(np.float64)
    nu = wn32 / s[:, None]                                   # normal_unweighted
    nR = nu @ R                                              # n^T R           (translation block)
    # with a = R^T n:  a^T [p]x = (a x p)^T, hence  -n^T R [p]x = (p x a)^T
    Jrot = np.cross(p, nR)
    Jr = np.concatenate([Jrot, nR], axis=1)                  # (K,6), rotation first
    A = (s + r * ds)[:, None] * Jr                           # line 1898
    b = -sr32                                                # line 1906
    return A, b


def normal_equations(A, b):
    """icp_test_runner.cpp:1910-1919: H = A^T A, g = A^T b."""
    return A.T @ A, A.T @ b


def pack27(H, g):
    """SymmetricHessianComputer layout, DCReg/include/hessian_computer.h:62-123:
    21 upper-triangular entries row-major ((0,0),(0,1)..(5,5)) followed by the 6 rhs."""
    out = np.empty(27)
    k = 0
    for i in range(6):
        for j in range(i, 6):
            out[k] = H[i, j]; k += 1
    out[21:] = g
    return out


def unpack27(v):
    H = np.zeros((6, 6)); k = 0
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = v[k]; k += 1
    return H, np.array(v[21:27], dtype=np.float64)


def reduce_normal_equations(src4, plane4, R, t, use_wd):
    """Oracle for the K1 seam (include/dcreg_b200.h: dcreg_reduce_normal_equations).

    Inputs are what the kernel reads: src4 (N,4) float32 body-frame points, plane4 (N,4)
    float32 or float64 (nx,ny,nz,d); a slot whose normal is all-zero is an empty slot.
    Per slot (icp_test_runner.cpp:1718,1774-1803,1863-1915): q = fl32(R p + t), r = n.q + d,
    s = max(0, 1-0.9|r|), gate s > 0.1, J = (s + r ds_dr)[(p x R^T n), R^T n], b = -fl32(s r),
    with the float32 round trip of s*n.  Returns out27 and stats (sum r^2, N_eff, N_with_plane).
    """
    p = src4[:, :3].astype(np.float64)
    n = plane4[:, :3].astype(np.float64)
    d = plane4[:, 3].astype(np.float64)
    q = (p @ R.T + t).astype(np.float32).astype(np.float64)
    has = np.any(n != 0.0, axis=1)
    r = np.einsum("kj,kj->k", n, q) + d
    s = np.maximum(0.0, 1.0 - 0.9 * np.abs(r))
    ds = np.zeros_like(r)
    if use_wd:
        m = (s > 0.0) & (s < 1.0)
        ds[m] = np.where(r[m] > 0, -0.9, 0.9)
    valid = has & (s > 0.1)
    corr = Correspondences(valid, n, d, r, s, ds, int(has.sum()), has)
    A, b = build_rows(src4[:, :3], corr, R)
    H, g = normal_equations(A, b)
    stats = np.array([float(np.sum(r[valid] ** 2)), float(valid.sum()), float(has.sum())])
    return pack27(H, g), stats


# ----------------------------------------------------------------------------
# Stage S6: degeneracy analysis
# ----------------------------------------------------------------------------
@dataclass
class Analysis:
    """DegeneracyAnalysisResult, DCReg/include/utils.hpp:427-448."""
    is_degenerate: bool = False
    mask: list = field(default_factory=lambda: [False] * 6)
    eigenvalues_full: np.ndarray = None
    eigenvectors_full: np.ndarray = None
    singular_values: np.ndarray = None
    cond_full: float = float("nan")
    cond_full_sub_rot: float = float("nan")
    cond_full_sub_trans: float = float("nan")
    cond_schur_rot: float = float("nan")
    cond_schur_trans: float = float("nan")
    cond_diag_rot: float = float("nan")
    cond_diag_trans: float = float("nan")
    lambda_schur_rot: np.ndarray = None
    lambda_schur_trans: np.ndarray = None
    lambda_sub_rot: np.ndarray = None
    lambda_sub_trans: np.ndarray = None
    schur_V_rot: np.ndarray = None
    schur_V_trans: np.ndarray = None
    P: np.ndarray = None
    pcg_iterations: int = 0


def schur_blocks(H):
    """icp_test_runner.cpp:2418-2469 (the only released Schur code) + paper Eq. 18."""
    H_RR, H_tt, H_Rt, H_tR = H[:3, :3], H[3:, 3:], H[:3, 3:], H[3:, :3]
    S_R = H_RR - H_Rt @ np.linalg.inv(H_tt) @ H_tR
    S_t = H_tt - H_tR @ np.linalg.inv(H_RR) @ H_Rt
    return 0.5 * (S_R + S_R.T), 0.5 * (S_t + S_t.T)


def _cond(lam):
    return float(np.max(lam) / max(float(np.min(lam)), 1e-12))


def analyze_degeneracy(H, prm: Params) -> Analysis:
    """DCReg::analyzeDegeneracy, DCReg/include/dcreg.hpp:45-166, plus the Schur detection that
    the release stubs out (dcreg.hpp:96-98): paper Eq. 18-21 / Alg. 1, SURVEY.md §3.4."""
    a = Analysis()
    lam, V = np.linalg.eigh(H)                                  # ascending (dcreg.hpp:66)
    a.eigenvalues_full, a.eigenvectors_full = lam, V
    a.cond_full_sub_trans = abs(lam[2]) / max(abs(lam[0]), 1e-12)   # dcreg.hpp:70-72
    a.cond_full_sub_rot = abs(lam[5]) / max(abs(lam[3]), 1e-12)     # dcreg.hpp:73-75
    sv = np.sort(np.abs(lam))[::-1]                             # JacobiSVD of symmetric H
    a.singular_values = sv
    a.cond_full = sv[0] / sv[5] if sv[5] > 1e-12 else float("inf")  # dcreg.hpp:85-89
    # diagonal blocks + Schur complements (icp_test_runner.cpp:2418-2469)
    a.lambda_sub_rot = np.linalg.eigvalsh(H[:3, :3])
    a.lambda_sub_trans = np.linalg.eigvalsh(H[3:, 3:])
    a.cond_diag_rot, a.cond_diag_trans = _cond(a.lambda_sub_rot), _cond(a.lambda_sub_trans)
    S_R, S_t = schur_blocks(H)
    a.lambda_schur_rot, a.schur_V_rot = np.linalg.eigh(S_R)
    a.lambda_schur_trans, a.schur_V_trans = np.linalg.eigh(S_t)
    a.cond_schur_rot, a.cond_schur_trans = _cond(a.lambda_schur_rot), _cond(a.lambda_schur_trans)
    a.P = np.eye(6)

    det = prm.detection
    if det == DET_SCHUR_CONDITION_NUMBER:
        # kappa_i = lambda_max / lambda_i per block, degenerate iff > threshold (Eq. 20-21)
        for blk, lamb in ((0, a.lambda_schur_rot), (3, a.lambda_schur_trans)):
            for i in range(3):
                k = lamb[2] / max(lamb[i], 1e-12)
                if k > prm.cond_thresh:
                    a.mask[blk + i] = True
        a.is_degenerate = any(a.mask)
        # preconditioner, Eq. 43-46: clamp eigenvalues at lambda_max / kappa_target
        P = np.zeros((6, 6))
        for blk, lamb, Vb in ((0, a.lambda_schur_rot, a.schur_V_rot),
                              (3, a.lambda_schur_trans, a.schur_V_trans)):
            lt = np.maximum(lamb, lamb[2] / prm.kappa_target)
            P[blk:blk + 3, blk:blk + 3] = Vb @ np.diag(1.0 / lt) @ Vb.T
        a.P = P
    elif det == DET_FULL_EVD_MIN_EIGENVALUE:                    # dcreg.hpp:100-110
        for i in range(6):
            if lam[i] < prm.eig_thresh:
                a.mask[i] = True
        a.is_degenerate = any(a.mask)
    elif det == DET_EVD_SUB_CONDITION:
        # dcreg.hpp:112-126 reads cond_diag_* which the released analyzeDegeneracy never fills
        # (NaN) -> never degenerate.  Kept as released.
        a.is_degenerate = False
    elif det == DET_FULL_SVD_CONDITION:                         # dcreg.hpp:128-143
        a.is_degenerate = bool(a.cond_full > prm.cond_thresh)
        if a.is_degenerate:
            mx = float(np.max(lam))
            for i in range(6):
                if mx / lam[i] > prm.cond_thresh:
                    a.mask[i] = True
    return a


# ----------------------------------------------------------------------------
# Stage S7: solve
# ----------------------------------------------------------------------------
def qr_solve(H, g):
    """H.colPivHouseholderQr().solve(g) (dcreg.hpp:182,190,197): full-rank 6x6 direct solve."""
    return np.linalg.lstsq(H, g, rcond=None)[0]


def pcg(H, g, P, max_iter, tol):
    """Paper Alg. 3 (stub at dcreg.hpp:279-287): PCG on H x = g, x0 = 0, stop on ||r||_2 < tol."""
    x = np.zeros(6)
    r = g.copy()
    z = P @ r
    p = z.copy()
    rz = float(r @ z)
    it = 0
    for it in range(1, max_iter + 1):
        Hp = H @ p
        alpha = rz / float(p @ Hp)
        x = x + alpha * p
        r = r - alpha * Hp
        if float(np.linalg.norm(r)) < tol:
            break
        z = P @ r
        rz_new = float(r @ z)
        p = z + (rz_new / rz) * p
        rz = rz_new
    return x, it


def solve_degenerate_system(H, g, prm: Params, a: Analysis):
    """DCReg::solveDegenerateSystem, dcreg.hpp:168-264 (+ PCG branch from paper Alg. 3)."""
    h = prm.handling
    if h == HAND_STANDARD_REGULARIZATION:                       # dcreg.hpp:177-184
        Hr = H.copy()
        if a.is_degenerate:
            Hr[np.diag_indices(6)] += prm.std_reg_gamma
        return qr_solve(Hr, g)
    if h == HAND_PRECONDITIONED_CG:                             # dcreg.hpp:186-193
        if a.is_degenerate:
            x, a.pcg_iterations = pcg(H, g, a.P, prm.pcg_max_iter, prm.pcg_tol)
            return x
        return qr_solve(H, g)
    if h == HAND_SOLUTION_REMAPPING:                            # dcreg.hpp:195-221
        x = qr_solve(H, g)
        if a.is_degenerate:
            V = a.eigenvectors_full
            Pp = np.zeros((6, 6)); good = 0
            for i in range(6):
                if not a.mask[i]:
                    Pp += np.outer(V[:, i], V[:, i]); good += 1
            x = Pp @ x if good > 0 else np.zeros(6)
        return x
    if h == HAND_TRUNCATED_SVD:                                 # dcreg.hpp:223-248
        # singular values are DEScending while the mask is indexed by AScending eigen-index:
        # the reference pairs mask[i] with sigma_i as-is (quirk kept).
        lam, V = a.eigenvalues_full, a.eigenvectors_full
        order = np.argsort(-np.abs(lam), kind="stable")
        x = np.zeros(6); kept = 0
        for i in range(6):
            sig = a.singular_values[i]
            if (not a.mask[i]) and sig > 1e-9:
                v = V[:, order[i]]
                # U_i = sign(lambda) V_i for a symmetric matrix; H is PSD so sign = +
                x += (1.0 / sig) * v * float(v @ g) * (1.0 if lam[order[i]] >= 0 else -1.0)
                kept += 1
        return x if kept else np.zeros(6)
    return qr_solve(H, g)                                       # NONE_HAND / default


# ----------------------------------------------------------------------------
# The outer loop
# ----------------------------------------------------------------------------
@dataclass
class IterLog:
    rmse: float
    fitness: float
    n_eff: int
    n_pt: int
    objective: float
    gradient: np.ndarray
    H: np.ndarray
    g: np.ndarray
    dx: np.ndarray
    T: np.ndarray
    analysis: Analysis


def icp_so3(src_f32, tgt_f32, T_init, prm: Params, tree=None):
    """TestRunner::Point2PlaneICP_SO3_OpenMP, icp_test_runner.cpp:1611-2060.
    Returns (converged, T_final, [IterLog...], status) with status in {"ok","not_enough_points",
    "nonfinite"}."""
    if tree is None:
        tree = build_tree(tgt_f32)
    R = T_init[:3, :3].copy(); t = T_init[:3, 3].copy()
    logs = []
    converged = False
    status = "ok"
    N = src_f32.shape[0]
    for _ in range(prm.max_iterations):
        corr = find_correspondences(src_f32, tgt_f32, tree, R, t, prm.search_radius,
                                    prm.use_weight_derivative)
        n_eff = int(corr.valid.sum())
        if n_eff < 10:                                          # lines 1847-1854
            status = "not_enough_points"
            break
        fitness = corr.n_pt / N                                 # line 1856
        rmse = math.sqrt(float(np.sum(corr.r[corr.valid] ** 2)) / n_eff)  # line 1858
        A, b = build_rows(src_f32, corr, R)
        H, g = normal_equations(A, b)
        a = analyze_degeneracy(H, prm)
        dx = solve_degenerate_system(H, g, prm, a)
        if not np.all(np.isfinite(dx)):                         # lines 1942-1950
            status = "nonfinite"
            break
        R, t = boxplus(R, t, dx)                                # line 1953
        T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
        logs.append(IterLog(rmse, fitness, n_eff, corr.n_pt, 0.5 * float(b @ b), -g, H, g, dx, T, a))
        if np.linalg.norm(dx[:3]) < prm.conv_rot and np.linalg.norm(dx[3:]) < prm.conv_trans:
            converged = True                                    # lines 1998-2002
            break
    T = np.eye(4); T[:3, :3] = R; T[:3, 3] = t
    return converged, T, logs, status


# ----------------------------------------------------------------------------
# Post-run metrics
# ----------------------------------------------------------------------------
def point_to_point_metrics(src_f32, tgt_f32, T, error_threshold, tree_tgt=None):
    """calculatePointToPointError, DCReg/include/utils.hpp:538-589 (+ pcl::transformPointCloud: FP64 math, float32
    store).  Returns dict(rmse, fitness, chamfer, n_valid).  FLANN reports float32 squared distances."""
    from scipy.spatial import cKDTree
    aligned = transform_points_f32(src_f32, T[:3, :3], T[:3, 3])
    if tree_tgt is None:
        tree_tgt = build_tree(tgt_f32)

    def nn_d2(tree, data_f32, queries_f32):
        _, idx = tree.query(queries_f32.astype(np.float64), k=1)
        e = queries_f32 - data_f32[idx]                              # float32 differences
        return (e[:, 0] * e[:, 0] + e[:, 1] * e[:, 1] + e[:, 2] * e[:, 2]).astype(np.float32)

    d2 = nn_d2(tree_tgt, tgt_f32, aligned).astype(np.float64)
    dist = np.sqrt(d2)
    ok = dist < error_threshold
    n = len(aligned)
    rmse = math.sqrt(float(d2[ok].sum()) / n)
    fitness = float(ok.sum()) / n
    d2b = nn_d2(cKDTree(aligned.astype(np.float64)), aligned, tgt_f32).astype(np.float64)
    chamfer = 0.5 * (float(dist.sum()) / n + float(np.sqrt(d2b).sum()) / len(tgt_f32))
    return {"rmse": rmse, "fitness": fitness, "chamfer": chamfer, "n_valid": int(ok.sum())}
