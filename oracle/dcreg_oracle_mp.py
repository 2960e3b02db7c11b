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
