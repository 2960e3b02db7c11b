"""High-precision reference of the "Ours" solve step (Schur detection + PCG handling).  TEST INFRASTRUCTURE ONLY.

The device step (k2_solve.cuh: icp_step_warp_ours) computes the same mathematics as dcreg_oracle.analyze_degeneracy /
solve_degenerate_system in FP64 with its own arithmetic (MUFU-seeded reciprocals, a warm-started Jacobi, an L D L^T
block inverse, a lane-parallel PCG with FMAs).  This module evaluates the step in mpmath at DPS digits from a
record's H27, taken as exact doubles, and reports, besides every intermediate quantity, the MARGIN of every decision
the step takes, so a test can tell a decision that FP64 rounding cannot flip (clear) from one it can (inside the band).

Margins and the band
  * eigenvalue decisions (mask: lambda_max / lambda_i > cond_thresh, i.e. lambda_i < lambda_max / cond_thresh; the
    Eq. 46 clamp: lambda_i < lambda_max / kappa_target) are measured as |lambda_i - lambda_max / c| / scale, with
    lambda_i floored at 1e-12 for the mask as the step floors it (max is 1-Lipschitz, so the floored value carries the
    same absolute error and the same band applies below the floor).  scale is
    the size of what the FP64 Schur complement is computed from, lambda_max(S) + ||H_Rt||_2^2 ||H_tt^-1||_2 for S_R
    (and the mirror for S_t): FP64 eigenvalues of S are off by ~2e-15 * scale (a few ulp of the entries, the Jacobi
    adds ~1 ulp of lambda_max).  EIG_BAND = 1e-12 leaves a factor ~500 over that.
  * the PCG stop rule ||r_k|| < tol: margin | ||r_k|| - tol |.  The FP64 recurrence drifts from the exact one by
    ~eps cond(H) ||g|| in absolute terms (a corridor with cond(H) 1.2e5 and ||g|| 3.6e4 ends its 6th FP64 iteration
    at ||r|| = 8.3e-7 where the exact residual is 1e-52), so the stop is clear when the margin exceeds
    PCG_BAND_ABS * cond(H) * ||g|| with PCG_BAND_ABS = 8 eps, and PCG_BAND = 1e-6 of tol.
  * FullPivLU's invertibility (every pivot > 3 eps * largest pivot): the exact pivot ratio min|p| / max|p| is clear
    when it exceeds PIVOT_CLEAR = 16 eps (the FP64 pivots are off by a few eps of the largest), and clearly singular only
    when the block has an exactly zero row (the FP64 pivot is then exactly zero too).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import mpmath

EPS = 2.220446049250313e-16
EIG_BAND = 1e-12
PCG_BAND = 1e-6
PCG_BAND_ABS = 8 * EPS
PIVOT_CLEAR = 16 * EPS
DPS = 60


@dataclass
class StepRef:
    H: object = None                      # mp 6x6
    g: object = None                      # mp 6
    pivot_ratio: list = field(default_factory=list)     # [H_RR, H_tt]: exact min|pivot| / max|pivot| of FullPivLU
    pivot_margin: list = field(default_factory=list)    # pivot_ratio / (3 eps) - 1
    block_invertible: list = field(default_factory=list)  # FullPivLU's decision in exact arithmetic
    block_clear: list = field(default_factory=list)     # that decision is clear of rounding
    schur_ok: bool = False
    S: list = field(default_factory=list)               # [S_R, S_t] (mp 3x3)
    lam: list = field(default_factory=list)             # [rot, trans]: ascending eigenvalues (mp)
    V: list = field(default_factory=list)               # eigenvectors in columns (mp 3x3)
    scale: list = field(default_factory=list)           # eigenvalue error scale per block (see the module docstring)
    cond_ratio: list = field(default_factory=list)      # 6: lambda_max / max(lambda_i, 1e-12), rot then trans
    cond_margin: list = field(default_factory=list)     # 6: cond_ratio / cond_thresh - 1 (relative distance)
    mask_margin: list = field(default_factory=list)     # 6: |max(lambda_i, 1e-12) - lambda_max / cond_thresh| / scale
    clamp_margin: list = field(default_factory=list)    # 6: |lambda_i - lambda_max / kappa_target| / scale
    mask: list = field(default_factory=lambda: [0] * 6)
    is_degenerate: int = 0
    P: object = None                                    # mp 6x6, clamped preconditioner (identity unless schur_ok)
    pcg_x: list = field(default_factory=list)           # iterates x_1 .. x_max_iter (mp 6), never stopped early
    pcg_rnorm: list = field(default_factory=list)       # ||r_1|| .. ||r_max_iter||
    pcg_stop: int = 0                                   # iterations under the stop rule ||r_k|| < tol (0: QR branch)
    pcg_margin: list = field(default_factory=list)      # | ||r_k|| - tol | / band, k = 1 .. pcg_stop (clear: > 1)
    pcg_band: float = 0.0                               # max(PCG_BAND tol, PCG_BAND_ABS cond(H) ||g||)
    x_qr: object = None                                 # H^-1 g (None when H is singular)
    cond_H: float = math.inf                            # 2-norm condition number of H
    dx: object = None                                   # the step's reference dx (PCG iterate or H^-1 g)
    clear: bool = True                                  # every decision that shaped dx is outside its band


def _mat(rows):
    return mpmath.matrix(rows)


def _unpack27(v27):
    H = mpmath.matrix(6, 6)
    k = 0
    for i in range(6):
        for j in range(i, 6):
            H[i, j] = H[j, i] = mpmath.mpf(float(v27[k]))
            k += 1
    g = mpmath.matrix([mpmath.mpf(float(v27[21 + i])) for i in range(6)])
    return H, g


def _block(H, r0, c0):
    return _mat([[H[r0 + i, c0 + j] for j in range(3)] for i in range(3)])


def fullpiv_pivots(A):
    """Pivots of Eigen's FullPivLU (largest |entry| of the remaining block), in the working precision."""
    A = A.copy()
    n = A.rows
    piv = []
    for k in range(n):
        br, bc, bv = k, k, mpmath.mpf(-1)
        for i in range(k, n):
            for j in range(k, n):
                if abs(A[i, j]) > bv:
                    br, bc, bv = i, j, abs(A[i, j])
        piv.append(bv)
        if bv == 0:
            piv.extend([mpmath.mpf(0)] * (n - k - 1))
            break
        if br != k:
            for j in range(n):
                A[k, j], A[br, j] = A[br, j], A[k, j]
        if bc != k:
            for i in range(n):
                A[i, k], A[i, bc] = A[i, bc], A[i, k]
        for i in range(k + 1, n):
            f = A[i, k] / A[k, k]
            for j in range(k + 1, n):
                A[i, j] -= f * A[k, j]
    return piv


def _norm2(A):
    return max(abs(s) for s in mpmath.svd_r(A, compute_uv=False))


def _vnorm(v):
    return mpmath.sqrt(sum(v[i] ** 2 for i in range(len(v))))


def _pcg(H, g, P, max_iter):
    x = mpmath.matrix(6, 1)
    r = g.copy()
    z = P * r
    p = z.copy()
    rz = (r.T * z)[0]
    xs, rns = [], []
    for _ in range(max_iter):
        Hp = H * p
        pHp = (p.T * Hp)[0]
        if pHp == 0:
            break
        alpha = rz / pHp
        x = x + alpha * p
        r = r - alpha * Hp
        xs.append(x.copy())
        rns.append(_vnorm(r))
        z = P * r
        rz_new = (r.T * z)[0]
        if rz == 0:
            break
        p = z + (rz_new / rz) * p
        rz = rz_new
    return xs, rns


def step_reference(v27, cond_thresh=10.0, kappa_target=1.0, pcg_tol=1e-6, pcg_max_iter=10, dps=DPS) -> StepRef:
    """The "Ours" analysis + solve of one record at `dps` digits, with the margin of every decision."""
    with mpmath.workdps(dps):
        a = StepRef()
        H, g = _unpack27(v27)
        a.H, a.g = H, g
        HRR, Htt, HRt, HtR = _block(H, 0, 0), _block(H, 3, 3), _block(H, 0, 3), _block(H, 3, 0)
        for B in (HRR, Htt):
            piv = fullpiv_pivots(B)
            mx = max(abs(p) for p in piv)
            ratio = min(abs(p) for p in piv) / mx if mx > 0 else mpmath.mpf(0)
            a.pivot_ratio.append(float(ratio))
            a.pivot_margin.append(float(ratio / (3 * EPS) - 1))
            a.block_invertible.append(bool(mx > 0 and ratio > 3 * EPS))
            zero_row = any(all(B[i, j] == 0 for j in range(3)) for i in range(3))
            a.block_clear.append(bool(ratio > PIVOT_CLEAR or zero_row))
        a.schur_ok = a.block_invertible[0] and a.block_invertible[1]
        a.cond_H = _cond2(H)
        a.x_qr = mpmath.lu_solve(H, g) if math.isfinite(a.cond_H) else None
        a.P = mpmath.eye(6)
        if a.schur_ok:
            HRRi, Htti = mpmath.inverse(HRR), mpmath.inverse(Htt)
            SR = HRR - HRt * Htti * HtR
            St = Htt - HtR * HRRi * HRt
            a.scale = [None, None]
            for blk, (S, Hoff, Hinv) in enumerate(((SR, HRt, Htti), (St, HtR, HRRi))):
                S = (S + S.T) / 2
                E, Q = mpmath.eigsy(S)
                order = sorted(range(3), key=lambda i: E[i])
                lam = [E[i] for i in order]
                V = _mat([[Q[r, i] for i in order] for r in range(3)])
                a.S.append(S); a.lam.append(lam); a.V.append(V)
                a.scale[blk] = abs(lam[2]) + _norm2(Hoff) ** 2 * _norm2(Hinv)
            a.P = mpmath.matrix(6, 6)
            for blk in range(2):
                lam, V, sc = a.lam[blk], a.V[blk], a.scale[blk]
                lt = []
                for i in range(3):
                    ratio = lam[2] / max(lam[i], mpmath.mpf(1e-12))
                    a.cond_ratio.append(float(ratio))
                    a.cond_margin.append(float(ratio / cond_thresh - 1))
                    a.mask_margin.append(float(abs(max(lam[i], mpmath.mpf(1e-12)) - lam[2] / cond_thresh) / sc))
                    # lambda_max is its own clamp's reference: max(lambda_max, lambda_max / kappa) is lambda_max for any
                    # kappa >= 1, so that comparison decides nothing
                    a.clamp_margin.append(float(abs(lam[i] - lam[2] / kappa_target) / sc) if i < 2 else math.inf)
                    if ratio > cond_thresh:
                        a.mask[blk * 3 + i] = 1
                    lt.append(max(lam[i], lam[2] / kappa_target))
                for i in range(3):
                    for j in range(3):
                        a.P[blk * 3 + i, blk * 3 + j] = sum(V[i, k] * V[j, k] / lt[k] for k in range(3))
            a.is_degenerate = int(any(a.mask))
        if a.is_degenerate:
            a.pcg_x, a.pcg_rnorm = _pcg(H, g, a.P, pcg_max_iter)
            stop = len(a.pcg_x)
            a.pcg_band = max(PCG_BAND * pcg_tol, PCG_BAND_ABS * a.cond_H * float(_vnorm(g)))
            for k, rn in enumerate(a.pcg_rnorm):
                a.pcg_margin.append(float(abs(rn - pcg_tol) / a.pcg_band) if a.pcg_band > 0 else math.inf)
                if rn < pcg_tol:
                    stop = k + 1
                    break
            a.pcg_stop = stop
            a.dx = a.pcg_x[stop - 1] if stop > 0 else mpmath.matrix(6, 1)
        else:
            a.dx = a.x_qr
        # the decisions that shaped dx: block invertibility, the mask (only whether any flag is set matters for dx, but a
        # flag inside the band changes the logged mask), the clamps (they shape P, hence the PCG iterates), the stops
        a.clear = all(a.block_clear)
        if a.schur_ok:
            a.clear = a.clear and all(m > EIG_BAND for m in a.mask_margin)
            if a.is_degenerate:
                a.clear = a.clear and all(m > EIG_BAND for m in a.clamp_margin)
                a.clear = a.clear and all(m > 1.0 for m in a.pcg_margin)
        return a


def _cond2(H):
    s = mpmath.svd_r(H, compute_uv=False)
    smax = max(abs(v) for v in s)
    smin = min(abs(v) for v in s)
    return float(smax / smin) if smin > 0 else math.inf


def to_float(v):
    """mp vector / list -> list of Python floats."""
    return [float(v[i]) for i in range(len(v))]


# ==================================================================================================================
# Every dcreg_analysis field, the baseline methods' detections and handlers, the pose update and the covariance.
#
# Each reference value comes with the error an FP64 computation of it may carry (an absolute bound, K_* eps times the
# quantity's own scale), and each decision with its margin in units of the error of the quantities it compares.  A
# decision is clear when that margin exceeds 1; a value whose bound is math.inf is not compared (inside the band).
#   * eigenvalues of H, singular values (|lambda| of the symmetric H): dH = K_EIG eps ||H||_2 (Weyl);
#   * lambda_sub_*: K_EIG eps ||block||_2; lambda_schur_*: dS = K_EIG eps (|lambda_max(S)| + ||H_off||^2 ||B^-1|| cond(B))
#     with B the block the Schur complement inverts (its FP64 inverse is off by cond(B) eps relative);
#   * ratios (conditions) by their derivative: d(a / b) <= (a / b) (da / |a| + db / |b|), doubled for second order;
#   * eigenvectors, compared without their sign: 2 dS / gap (Davis-Kahan), not compared when that exceeds 1/4;
#   * P = f(S) with f(lambda) = 1 / max(lambda, lambda_max / kappa): f is Lipschitz with 1 / lt_min^2 and the clamp
#     level moves with lambda_max, so |dP| <= 2 (sqrt(3) + 1 / kappa) dS / lt_min^2;
#   * dx of the QR solve: K_DX cond(H) eps |x|_max; of TReg the same with H + gamma I; of SR and TSVD, which apply
#     f(H) with f(lambda) = kept(lambda) / lambda: K_DX eps ||H|| |x| (1 / lambda_min,kept + 2 / gap) with gap the
#     distance between a kept and a dropped eigenvalue (the projector's Davis-Kahan term); x is the QR solution for SR
#     and g / lambda_min,kept for TSVD (f's divided differences are 1 / (lambda_a lambda_b) and 1 / (lambda_a gap)).
# ==================================================================================================================
K_EIG = 64
K_DX = 64
K_POSE = 16
K_COV = 64
QR_RANK_CLEAR = 256 * EPS       # colpiv QR: a column set is clearly of full rank when sigma_min > this * ||H||
COV_PIVOT_CLEAR = 64 * EPS      # FullPivLU 6x6 (cut at 6 eps of the largest pivot): clearly invertible above this ratio

DET_NONE, DET_SCHUR, DET_EVD_MIN, DET_EVD_SUB, DET_SVD_COND = 0, 1, 2, 3, 4
HAND_NONE, HAND_STD_REG, HAND_ADAPTIVE, HAND_PCG, HAND_SR, HAND_TSVD = 0, 1, 2, 3, 4, 5

ANALYSIS_FIELDS = ("eigenvalues_full", "singular_values", "cond_full", "cond_full_sub_rot", "cond_full_sub_trans",
                   "lambda_sub_rot", "lambda_sub_trans", "cond_diag_rot", "cond_diag_trans", "lambda_schur_rot",
                   "lambda_schur_trans", "cond_schur_rot", "cond_schur_trans", "schur_V_rot", "schur_V_trans",
                   "aligned_V_rot", "aligned_V_trans", "P_preconditioner")
SIGNFREE = ("schur_V_rot", "schur_V_trans")     # eigenvectors in columns, compared without their sign
INT_FIELDS = ("degenerate_mask", "is_degenerate", "schur_singular", "rot_indices", "trans_indices")


@dataclass
class AnalysisRef:
    vals: dict = field(default_factory=dict)      # field -> reference values (floats; NaN / inf where the device writes them)
    bound: dict = field(default_factory=dict)     # field -> absolute bound per value (math.inf: not compared)
    ints: dict = field(default_factory=dict)      # integer field -> values, compared exactly (absent: inside the band)
    margins: dict = field(default_factory=dict)   # decision -> [margin / band] (clear when > 1)
    lam: list = field(default_factory=list)       # eigenvalues of H, ascending (mp)
    V: object = None                              # their eigenvectors in columns (mp 6x6)
    normH: float = 0.0
    dH: float = 0.0                               # eigenvalue bound of H
    order: list = field(default_factory=list)     # singular index -> eigen index (descending |lambda|)
    mask: list = field(default_factory=lambda: [0] * 6)
    is_degenerate: int = 0
    schur_ok: bool = False
    clear: bool = True                            # every decision that shapes mask, branch and dx is outside its band
    dx: object = None                             # reference dx (floats), None for the "Ours" handler (step_reference)
    dx_bound: float = math.inf                    # absolute, max-norm
    branch: str = ""


def _eigsy_sorted(A):
    E, Q = mpmath.eigsy((A + A.T) / 2)
    n = A.rows
    idx = sorted(range(n), key=lambda i: E[i])
    return [E[i] for i in idx], _mat([[Q[r, i] for i in idx] for r in range(n)])


def _ratio(num, den, dnum, dden, floor):
    """|num| / max(|den|, floor) and its bound (max and |.| are 1-Lipschitz: no decision to band)"""
    d = max(abs(den), mpmath.mpf(floor))
    v = abs(num) / d
    if dden >= 0.5 * d:
        return float(v), math.inf
    return float(v), float(2 * v * (dnum / max(abs(num), mpmath.mpf(1e-300)) + dden / d))


def _gaps(lam):
    return [min([abs(lam[i] - lam[j]) for j in range(len(lam)) if j != i]) for i in range(len(lam))]


def align_reference(V, dV):
    """Alg. 2 on the exact eigenvectors V (mp 3x3, columns): (aligned V, indices, margins of every greedy pick and
    sign fix in units of 2 dV).  Same rule as k2_solve.cuh's align_axes: largest |V[j][i]| over unused (i, j), then
    v <- -v when v[j] < 0, then Gram-Schmidt in slot order."""
    used_v, used_e, ind, margins = set(), set(), [0, 0, 0], []
    for _ in range(3):
        cand = sorted(((abs(V[j, i]), i, j) for j in range(3) if j not in used_e for i in range(3) if i not in used_v),
                      key=lambda c: -c[0])
        if len(cand) > 1:
            margins.append(float((cand[0][0] - cand[1][0]) / (2 * dV)) if dV > 0 else math.inf)
        _, bi, bj = cand[0]
        used_v.add(bi); used_e.add(bj); ind[bj] = bi
    Va = mpmath.matrix(3, 3)
    for j in range(3):
        v = [V[r, ind[j]] for r in range(3)]
        margins.append(float(abs(v[j]) / (2 * dV)) if dV > 0 else math.inf)
        if v[j] < 0:
            v = [-x for x in v]
        for k in range(j):
            d = sum(v[r] * Va[r, k] for r in range(3))
            v = [v[r] - d * Va[r, k] for r in range(3)]
        n = mpmath.sqrt(sum(x * x for x in v))
        for r in range(3):
            Va[r, j] = v[r] / n if n > 0 else 0
    return Va, ind, margins


def _flat(M):
    return [float(M[i, j]) for i in range(M.rows) for j in range(M.cols)]


def qr_reference(H, g):
    """colPivHouseholderQr().solve(g) in exact arithmetic: exactly zero columns (rows) get a zero component, the rest
    is the solution of the remaining block.  Returns (x mp, cond of the remaining block, clear): clear when that
    block is of full rank far above the QR's rank cut (sigma_min > QR_RANK_CLEAR ||H||)."""
    n = H.rows
    keep = [j for j in range(n) if any(H[i, j] != 0 for i in range(n))]
    x = mpmath.matrix(n, 1)
    if not keep:
        return x, 1.0, True
    B = _mat([[H[i, j] for j in keep] for i in keep])
    s = [abs(v) for v in mpmath.eigsy((B + B.T) / 2)[0]]
    nH = max(s)
    if min(s) <= QR_RANK_CLEAR * nH:
        return None, math.inf, False
    xb = mpmath.lu_solve(B, _mat([[g[i]] for i in keep]))
    for k, j in enumerate(keep):
        x[j] = xb[k]
    return x, float(nH / min(s)), True


def analysis_reference(v27, prm, dps=DPS) -> AnalysisRef:
    """Every dcreg_analysis field of analyze_and_solve<true> for the record H27 v27 and settings prm (any object with
    dcreg_icp_params' field names), with the baseline detections and handlers as released (dcreg_oracle.py,
    k2_solve.cuh): FULL_SVD's mask uses signed lambda; TSVD pairs mask[i] with sigma_i in descending order, cuts at
    sigma > 1e-9 and takes sign(lambda); SR with no kept vector returns 0; TReg adds gamma only when degenerate;
    EVD_SUB never flags; ADAPTIVE and NONE are the QR solve.  For the Schur detection dx is left to step_reference."""
    det, hand = int(prm.detection), int(prm.handling)
    with mpmath.workdps(dps):
        a = AnalysisRef()
        H, g = _unpack27(v27)
        lam, V = _eigsy_sorted(H)
        a.lam, a.V = lam, V
        nH = max(abs(x) for x in lam)
        a.normH = float(nH)
        dH = K_EIG * EPS * nH
        a.dH = float(dH)
        a.vals["eigenvalues_full"] = [float(x) for x in lam]
        a.bound["eigenvalues_full"] = [float(dH)] * 6
        order = sorted(range(6), key=lambda i: -abs(lam[i]))
        a.order = order
        sv = [abs(lam[e]) for e in order]
        a.vals["singular_values"] = [float(s) for s in sv]
        a.bound["singular_values"] = [float(dH)] * 6
        # cond_full: sigma_1 / sigma_6 when sigma_6 > 1e-12, else inf: a decision
        m_sv = float(abs(sv[5] - mpmath.mpf(1e-12)) / dH) if dH > 0 else math.inf
        a.margins["sigma6 vs 1e-12"] = [m_sv]
        if sv[5] > 1e-12:
            a.vals["cond_full"] = [float(sv[0] / sv[5])]
            a.bound["cond_full"] = [_ratio(sv[0], sv[5], dH, dH, 0.0)[1] if m_sv > 1 else math.inf]
        else:
            a.vals["cond_full"] = [math.inf]
            a.bound["cond_full"] = [0.0 if m_sv > 1 else math.inf]
        for name, num, den in (("cond_full_sub_trans", lam[2], lam[0]), ("cond_full_sub_rot", lam[5], lam[3])):
            v, b = _ratio(num, den, dH, dH, 1e-12)
            a.vals[name], a.bound[name] = [v], [b]
        # diagonal blocks
        HRR, Htt, HRt, HtR = _block(H, 0, 0), _block(H, 3, 3), _block(H, 0, 3), _block(H, 3, 0)
        blk_eig = {}
        for nm, B in (("rot", HRR), ("trans", Htt)):
            lb, Vb = _eigsy_sorted(B)
            blk_eig[nm] = (lb, Vb)
            db = K_EIG * EPS * max(abs(x) for x in lb)
            a.vals["lambda_sub_" + nm] = [float(x) for x in lb]
            a.bound["lambda_sub_" + nm] = [float(db)] * 3
            v, b = (float(lb[2] / max(lb[0], mpmath.mpf(1e-12))),
                    _ratio(lb[2], max(lb[0], mpmath.mpf(1e-12)), db, db, 1e-12)[1])
            a.vals["cond_diag_" + nm], a.bound["cond_diag_" + nm] = [v], [b]
        # Schur complements: FullPivLU's invertibility of both blocks decides whether they exist
        blocks_clear, inv_ok = [], []
        for B in (HRR, Htt):
            piv = fullpiv_pivots(B)
            mx = max(abs(p) for p in piv)
            ratio = min(abs(p) for p in piv) / mx if mx > 0 else mpmath.mpf(0)
            inv_ok.append(bool(mx > 0 and ratio > 3 * EPS))
            zero_row = any(all(B[i, j] == 0 for j in range(3)) for i in range(3))
            blocks_clear.append(bool(ratio > PIVOT_CLEAR or zero_row))
        a.schur_ok = inv_ok[0] and inv_ok[1]
        a.margins["FullPivLU 3x3"] = [1.0 if all(blocks_clear) else 0.0]
        eye9 = [1.0, 0, 0, 0, 1.0, 0, 0, 0, 1.0]
        for nm in ("rot", "trans"):
            a.vals["aligned_V_" + nm] = list(eye9)
            a.bound["aligned_V_" + nm] = [0.0] * 9
            a.ints[nm + "_indices"] = [0, 1, 2]
        a.vals["P_preconditioner"] = [1.0 if i % 7 == 0 else 0.0 for i in range(36)]
        a.bound["P_preconditioner"] = [0.0] * 36
        schur = []                                                 # (lam, V, dS) per block
        if not all(blocks_clear):                                  # inside the band: nothing of the Schur part compared
            for nm in ("rot", "trans"):
                for f in ("lambda_schur_", "cond_schur_", "schur_V_", "aligned_V_"):
                    n = {"lambda_schur_": 3, "cond_schur_": 1}.get(f, 9)
                    a.vals[f + nm], a.bound[f + nm] = [math.nan] * n, [math.inf] * n
                a.ints.pop(nm + "_indices", None)
            if det == DET_SCHUR:
                a.bound["P_preconditioner"] = [math.inf] * 36
        elif not a.schur_ok:
            a.ints["schur_singular"] = [1]
            for nm in ("rot", "trans"):
                a.vals["lambda_schur_" + nm], a.bound["lambda_schur_" + nm] = [math.nan] * 3, [0.0] * 3
                a.vals["cond_schur_" + nm], a.bound["cond_schur_" + nm] = [math.inf], [0.0]
                a.vals["schur_V_" + nm], a.bound["schur_V_" + nm] = list(eye9), [0.0] * 9
        else:
            a.ints["schur_singular"] = [0]
            HRRi, Htti = mpmath.inverse(HRR), mpmath.inverse(Htt)
            condB = {nm: float(max(abs(x) for x in blk_eig[nm][0]) / min(abs(x) for x in blk_eig[nm][0]))
                     for nm in ("rot", "trans")}
            for nm, S, Hoff, Hinv, cb in (("rot", HRR - HRt * Htti * HtR, HRt, Htti, condB["trans"]),
                                          ("trans", Htt - HtR * HRRi * HRt, HtR, HRRi, condB["rot"])):
                ls, Vs = _eigsy_sorted((S + S.T) / 2)
                dS = K_EIG * EPS * (abs(ls[2]) + _norm2(Hoff) ** 2 * _norm2(Hinv) * cb)
                schur.append((ls, Vs, dS))
                a.vals["lambda_schur_" + nm] = [float(x) for x in ls]
                a.bound["lambda_schur_" + nm] = [float(dS)] * 3
                v, b = _ratio(ls[2], max(ls[0], mpmath.mpf(1e-12)), dS, dS, 1e-12)
                a.vals["cond_schur_" + nm], a.bound["cond_schur_" + nm] = [float(ls[2] / max(ls[0], 1e-12))], [b]
                gaps = _gaps(ls)
                colb = [float(2 * dS / gp) if gp > 0 and 2 * dS / gp < 0.25 else math.inf for gp in gaps]
                a.vals["schur_V_" + nm] = _flat(Vs)
                a.bound["schur_V_" + nm] = [colb[k % 3] for k in range(9)]
                dV = max(colb)
                Va, ind, marg = align_reference(Vs, dV) if math.isfinite(dV) else (None, None, [0.0])
                a.margins["alignment " + nm] = marg
                if math.isfinite(dV) and min(marg) > 1:
                    a.vals["aligned_V_" + nm], a.bound["aligned_V_" + nm] = _flat(Va), [8 * dV] * 9
                    a.ints[nm + "_indices"] = ind
                else:
                    a.vals["aligned_V_" + nm], a.bound["aligned_V_" + nm] = [math.nan] * 9, [math.inf] * 9
                    a.ints.pop(nm + "_indices", None)
        # ---- detection ----
        mask = [0] * 6
        mm = []
        if det == DET_SCHUR and schur:
            kap = mpmath.mpf(float(prm.kappa_target))
            P = mpmath.matrix(6, 6)
            lt_min, dS_max = None, max(s[2] for s in schur)
            for blk, (ls, Vs, dS) in enumerate(schur):
                for i in range(3):
                    li = max(ls[i], mpmath.mpf(1e-12))
                    if ls[2] / li > prm.cond_thresh:
                        mask[blk * 3 + i] = 1
                    mm.append(float(abs(li - ls[2] / prm.cond_thresh) / (dS * (1 + 1 / mpmath.mpf(prm.cond_thresh)))))
                lt = [max(ls[i], ls[2] / kap) for i in range(3)]
                lt_min = min([lt_min] + lt) if lt_min is not None else min(lt)
                for i in range(3):
                    for j in range(3):
                        P[blk * 3 + i, blk * 3 + j] = sum(Vs[i, k] * Vs[j, k] / lt[k] for k in range(3))
            a.vals["P_preconditioner"] = _flat(P)
            bP = 2 * (math.sqrt(3) + 1 / float(kap)) * float(dS_max / lt_min ** 2) if lt_min > 0 else math.inf
            a.bound["P_preconditioner"] = [bP] * 36
        elif det == DET_EVD_MIN:
            for i in range(6):
                mask[i] = int(lam[i] < prm.eig_thresh)
                mm.append(float(abs(lam[i] - mpmath.mpf(prm.eig_thresh)) / dH) if dH > 0 else math.inf)
        elif det == DET_SVD_COND:
            cf = sv[0] / sv[5] if sv[5] > 1e-12 else mpmath.inf
            deg = bool(cf > prm.cond_thresh)
            if mpmath.isinf(cf):
                mm.append(m_sv)
            else:
                dcf = 2 * cf * dH * (1 / sv[0] + 1 / sv[5])
                mm.append(min(m_sv, float(abs(cf - prm.cond_thresh) / dcf) if dcf > 0 else math.inf))
            if deg:
                ct = mpmath.mpf(prm.cond_thresh)
                for i in range(6):
                    if abs(lam[i]) <= dH:                          # the sign of lambda_i decides mx / lambda_i
                        mm.append(float(abs(lam[i]) / dH) if dH > 0 else 0.0)
                        mask[i] = int(lam[i] == 0 or (lam[i] > 0 and lam[5] / lam[i] > ct))
                        continue
                    mask[i] = int(lam[i] > 0 and lam[5] / lam[i] > ct)
                    if lam[i] > 0:
                        mm.append(float(abs(lam[i] - lam[5] / ct) / (dH * (1 + 1 / ct))))
        a.margins["mask"] = mm
        a.mask, a.is_degenerate = mask, int(any(mask))
        a.ints["degenerate_mask"], a.ints["is_degenerate"] = list(mask), [a.is_degenerate]
        a.clear = all(m > 1 for m in mm) and all(blocks_clear)
        if not a.clear:                                            # the decisions themselves are inside the band
            a.ints.pop("degenerate_mask"); a.ints.pop("is_degenerate")
        # ---- handling ----
        if det == DET_SCHUR and hand == HAND_PCG:
            a.branch = "ours"
            return a
        if hand == HAND_PCG and a.is_degenerate:
            raise NotImplementedError("PCG without the Schur preconditioner")
        gnorm = mpmath.sqrt(sum(g[i] ** 2 for i in range(6)))

        def qr_branch(Hs):
            x, cond, ok = qr_reference(Hs, g)
            if not ok:
                return None, math.inf
            return x, K_DX * cond * EPS * float(max(abs(x[i]) for i in range(6)))

        def kept_bound(kept_e, x_norm):
            """f(H) with f = kept / lambda: K_DX eps ||H|| |x| (1 / lambda_min,kept + 2 / gap kept-dropped)"""
            lk = [abs(lam[e]) for e in range(6) if kept_e[e]]
            gap = [abs(lam[e] - lam[d]) for e in range(6) if kept_e[e] for d in range(6) if not kept_e[d]]
            if min(lk) == 0 or (gap and min(gap) == 0):
                return math.inf
            t = 1 / min(lk) + (2 / min(gap) if gap else 0)
            return float(K_DX * EPS * nH * x_norm * t)

        if hand == HAND_STD_REG:
            Hr = H.copy()
            if a.is_degenerate:
                for i in range(6):
                    Hr[i, i] += mpmath.mpf(float(prm.std_reg_gamma))
            a.branch = "treg"
            x, b = qr_branch(Hr)
        elif hand == HAND_SR:
            a.branch = "sr"
            x0, b0 = qr_branch(H)
            if not a.is_degenerate or x0 is None:
                x, b = x0, b0
            else:
                kept = [not mask[e] for e in range(6)]
                if not any(kept):
                    x, b = mpmath.matrix(6, 1), 0.0
                else:
                    x = mpmath.matrix(6, 1)
                    for e in range(6):
                        if kept[e]:
                            d = sum(V[i, e] * x0[i] for i in range(6))
                            for i in range(6):
                                x[i] += V[i, e] * d
                    xn = mpmath.sqrt(sum(x0[i] ** 2 for i in range(6)))
                    b = b0 + kept_bound(kept, xn)
        elif hand == HAND_TSVD:
            a.branch = "tsvd"
            kept_pos = [not mask[i] and sv[i] > 1e-9 for i in range(6)]
            tm = []
            for i in range(6):
                if not mask[i]:
                    tm.append(float(abs(sv[i] - mpmath.mpf(1e-9)) / dH) if dH > 0 else math.inf)
            for i in range(5):                                     # a tie that swaps a kept and a dropped position
                if kept_pos[i] != kept_pos[i + 1]:
                    tm.append(float(abs(sv[i] - sv[i + 1]) / dH) if dH > 0 else math.inf)
            for i in range(6):
                if kept_pos[i]:
                    tm.append(float(abs(lam[order[i]]) / dH) if dH > 0 else math.inf)
            a.margins["tsvd"] = tm
            a.clear = a.clear and all(m > 1 for m in tm)
            x = mpmath.matrix(6, 1)
            kept_e = [False] * 6
            for i in range(6):
                if kept_pos[i]:
                    e = order[i]
                    kept_e[e] = True
                    d = sum(V[r, e] * g[r] for r in range(6))
                    sc = (1 if lam[e] >= 0 else -1) * d / sv[i]
                    for r in range(6):
                        x[r] += V[r, e] * sc
            # |f(H + E) g - f(H) g| <= |E| |g| max(1 / lambda_min,kept^2, 1 / (lambda_kept gap)): kept_bound of |g| / lambda_min
            b = kept_bound(kept_e, gnorm / min(sv[i] for i in range(6) if kept_pos[i])) if any(kept_e) else 0.0
        else:                                                      # NONE, ADAPTIVE, PCG when not degenerate, default
            a.branch = "qr"
            x, b = qr_branch(H)
        if x is None:
            a.clear = False
        a.dx = None if x is None else to_float(x)
        a.dx_bound = b if a.clear else math.inf
        return a


def compare_analysis(ref: AnalysisRef, got: dict):
    """got: field -> values as the device writes them.  Returns ({field: worst error / bound}, [failures])."""
    worst, bad = {}, []
    for name in ANALYSIS_FIELDS:
        r = ref.vals[name]
        b = ref.bound[name]
        x = [float(v) for v in got[name]]
        w = 0.0
        for k, (rv, bv) in enumerate(zip(r, b)):
            if not math.isfinite(bv):
                continue
            xv = x[k]
            if math.isnan(rv) or math.isinf(rv):
                ok = (math.isnan(rv) and math.isnan(xv)) or rv == xv
                if not ok:
                    bad.append((name, k, xv, rv))
                continue
            if name in SIGNFREE:
                c = k % 3
                col_r = [r[3 * i + c] for i in range(3)]
                col_x = [x[3 * i + c] for i in range(3)]
                e = min(max(abs(p - q) for p, q in zip(col_x, col_r)), max(abs(p + q) for p, q in zip(col_x, col_r)))
            else:
                e = abs(xv - rv)
            if not e <= bv:
                bad.append((name, k, xv, rv, bv))
            w = max(w, e / bv if bv > 0 else (0.0 if e == 0 else math.inf))
        worst[name] = w
    for name, v in ref.ints.items():
        if [int(t) for t in got[name]] != list(v):
            bad.append((name, list(got[name]), v))
    return worst, bad


@dataclass
class PoseRef:
    R: list = field(default_factory=list)     # 9, row-major
    t: list = field(default_factory=list)
    bound_R: float = 0.0
    bound_t: float = 0.0
    theta: float = 0.0                        # |omega|
    vnorm: float = 0.0                        # |v|
    converged: bool = False                   # |omega| < conv_rot and |v| < conv_trans
    conv_margin: list = field(default_factory=list)   # the two comparisons, in units of their rounding
    clear: bool = True


def boxplus_reference(T, dx, conv_rot=0.0, conv_trans=0.0, dps=DPS) -> PoseRef:
    """R <- R Exp(omega), t <- t + R_old v, exactly, from the pose T (4x4 or 16, taken as exact doubles) and dx.  The
    bound covers the device's FP64 evaluation: K_POSE eps on R's entries (|R| <= 1), K_POSE eps (|t| + |v|) on t."""
    with mpmath.workdps(dps):
        Tf = [float(v) for v in (T.ravel() if hasattr(T, "ravel") else T)]
        R = _mat([[Tf[4 * i + j] for j in range(3)] for i in range(3)])
        t = [mpmath.mpf(Tf[4 * i + 3]) for i in range(3)]
        w = [mpmath.mpf(float(dx[i])) for i in range(3)]
        v = [mpmath.mpf(float(dx[3 + i])) for i in range(3)]
        th = mpmath.sqrt(sum(x * x for x in w))
        E = mpmath.eye(3)
        if th > 0:
            K = _mat([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
            E = E + (mpmath.sin(th) / th) * K + ((1 - mpmath.cos(th)) / th ** 2) * (K * K)
        Rn = R * E
        tn = [t[i] + sum(R[i, j] * v[j] for j in range(3)) for i in range(3)]
        p = PoseRef(R=_flat(Rn), t=[float(x) for x in tn])
        vn = mpmath.sqrt(sum(x * x for x in v))
        p.theta, p.vnorm = float(th), float(vn)
        p.bound_R = K_POSE * EPS * float(max(1, max(abs(R[i, j]) for i in range(3) for j in range(3))))
        p.bound_t = K_POSE * EPS * float(max(abs(x) for x in t) + vn + max(abs(x) for x in tn))
        p.converged = bool(th < conv_rot and vn < conv_trans)
        for val, thr in ((th, conv_rot), (vn, conv_trans)):
            p.conv_margin.append(float(abs(val - thr) / (K_POSE * EPS * val)) if val > 0 else math.inf)
        # the flag is the AND of two comparisons: a band comparison matters only where the other one holds
        rot_ok, tr_ok = th < conv_rot, vn < conv_trans
        p.clear = ((p.conv_margin[0] > 1 or not tr_ok and p.conv_margin[1] > 1) and
                   (p.conv_margin[1] > 1 or not rot_ok and p.conv_margin[0] > 1))
        return p


@dataclass
class CovRef:
    cov: list = field(default_factory=list)   # 36
    bound: float = 0.0                        # absolute, per entry
    invertible: bool = True
    pivot_ratio: float = 0.0                  # exact min |pivot| / max |pivot| of FullPivLU 6x6
    floored: bool = False                     # lambda_min(H^-1) <= 1e-12
    floor_margin: float = math.inf            # |lambda_min(H^-1) - 1e-12| / its bound
    cond_H: float = math.inf
    clear: bool = True


def covariance_reference(H_last, converged, dps=DPS) -> CovRef:
    """covariance_kernel: 1e6 I unless the run converged and H_last (6x6, exact doubles) is invertible by FullPivLU's
    rule (every pivot > 6 eps of the largest); else H^-1, rebuilt with eigenvalues floored at 1e-9 when its smallest
    eigenvalue is <= 1e-12.  Bounds: the FP64 inverse is within K_COV cond(H) eps ||H^-1|| (entries; the floor is
    1-Lipschitz, so the rebuild too, plus its own rounding at the floor's scale); lambda_min(H^-1) = 1 / lambda_max(H) moves by K_COV ||H^-1|| (eps + (eps cond)^2)
    (the inverse's residual seen along H's top eigenvector, plus the second-order term), which decides the floor."""
    c = CovRef()
    eye6 = [1e6 if i % 7 == 0 else 0.0 for i in range(36)]
    if not converged:
        c.cov = eye6
        return c
    with mpmath.workdps(dps):
        H = _mat([[float(H_last[6 * i + j]) for j in range(6)] for i in range(6)])
        piv = fullpiv_pivots(H)
        mx = max(abs(p) for p in piv)
        c.pivot_ratio = float(min(abs(p) for p in piv) / mx) if mx > 0 else 0.0
        c.invertible = bool(mx > 0 and c.pivot_ratio > 6 * EPS)
        zero_row = any(all(H[i, j] == 0 for j in range(6)) for i in range(6))
        c.clear = bool(c.pivot_ratio > COV_PIVOT_CLEAR or zero_row)
        if not c.invertible:
            c.cov = eye6
            return c
        Inv = mpmath.inverse(H)
        li, Vi = _eigsy_sorted(Inv)
        lh = _eigsy_sorted(H)[0]
        c.cond_H = float(max(abs(x) for x in lh) / min(abs(x) for x in lh))
        nI = max(abs(x) for x in li)
        dl = K_COV * float(nI) * (EPS + (EPS * c.cond_H) ** 2)
        c.floored = bool(li[0] <= mpmath.mpf(1e-12))
        c.floor_margin = float(abs(li[0] - mpmath.mpf(1e-12))) / dl
        c.clear = c.clear and c.floor_margin > 1
        c.bound = 4 * K_COV * c.cond_H * EPS * float(nI)
        if c.floored:
            lf = [max(x, mpmath.mpf(1e-9)) for x in li]
            M = Vi * mpmath.diag(lf) * Vi.T
            c.bound += 4 * K_COV * EPS * float(max(lf))             # the rebuild's own rounding, at the floor's scale
        else:
            M = Inv
        c.cov = _flat(M)
        return c
