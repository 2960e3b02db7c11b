"""Slot-level reference of one ICP iteration's normal equations.  TEST INFRASTRUCTURE ONLY (NumPy + SciPy).

Given the pose an iteration ran at (exact FP64), the source as the loop sees it, the target, the radius and the weight
settings, `iteration_reference` returns the reference's H27, sum b^2, sum r^2, N_pt and N_eff
(icp_test_runner.cpp:1714-1919, DESIGN.md §1), a per-entry allowance, and per slot a band flag with its reason.
`k1_reference` does the same for the streaming kernel's seam (points and planes given).

Per slot, following the reference's operations:
  q = fl32(R p + t)   FP64 without FMA, float32 store.  The kernel forms R p + t with an FMA chain, so a coordinate
                      whose FP64 value lies within 2^-50 |v| of a float32 rounding boundary is in band ("q"); any other
                      q is the kernel's q exactly.
  5-NN                float32 corr::dist2 (FLANN L2_Simple), ties broken by target index, then d2[4] < radius^2.
                      Exact given q.
  plane               `qr53`, a vectorised FP64 restatement of dla::colpiv_qr_solve<5,3> (same operations, same order,
                      no FMA; bit-identical to the host build, tests/test_gpu_normal_equations.py), then n = x/|x|,
                      d = 1/|x| and the gates |x| >= min_normal_norm, max_j (n.nb_j + d)^2 < thickness^2.  The device
                      fit contracts to FMAs, so its plane differs from this one by rounding.  How far one FP64
                      evaluation lies from the exact fit is measured per system by running the same algorithm in
                      extended precision (np.longdouble); 64 times that distance bounds the device's difference.  A
                      decision is in band when its margin is below that bound: the rank cut bign^2 < thr (M - k)
                      ("rank": relative margin below 64 cond(A) eps; a column that is exactly zero from the start is
                      clear, a non-zero column of a rank-deficient system is in band), the norm gate ("norm") and the
                      thickness gate ("thick").
  weight              s = 1 - slope |r|, gate s > gate: in band ("gate") when |s - gate| < max(1e-12, slope dr), with
                      dr the bound on the kernel's r minus this r: 64 (|r - r_exact plane| + 4 eps (|n| |q| + |d|))
                      plus the FMA chain's 8 eps (|n| |q| + |d|) for a fitted plane, the latter alone for a given one.
                      fl32(s n_i) and fl32(s r) are in band ("store") when their FP64 argument lies within its own
                      uncertainty of a float32 rounding boundary; a clear store is therefore the kernel's float32 value
                      exactly.  Row scale k = 1, or 2 - 1/s with the weight derivative.
  non-finite          a point, plane component or q that is NaN or +-Inf gives a NaN or infinite r in the reference,
                      so s = max(0, .) = 0: the slot is dropped.

Sums: rows in the reference's frame, (s + r ds/dr) [p x R^T nu, R^T nu] with nu = fl32(s n) / s and b = -fl32(s r)
(oracle/dcreg_oracle.py: build_rows), summed per entry with math.fsum (exact to one rounding).

Allowance of entry (i, j) of the packed sums (27 + sum b^2 + sum r^2):
    sum over band slots of m_i m_j                      (the slot's whole contribution, on either side of its decision)
  + sum over clear slots of e_i m_j + m_i e_j + e_i e_j (the row's own uncertainty)
  + c eps sum over all slots of m_i m_j                 (Gram, congruence and row-sum order)
with, per slot, m the magnitude bound of the row's components (world frame: |k| |p| |u'| for the three rotation
components, |k| |u'| for the translation ones, |b|, |r|; R is orthogonal, so the reference frame's components obey the
same bounds) and e the bound on the kernel's difference from it (from dr and from the eight roundings of R p, the cross
product and the k multiplication: 16 eps relative).  For a band slot without a valid reference row the bound is the
largest row a valid slot can have: |u'| <= 1, |k| <= max over the gate's range, |b|, |r| <= 1 / slope.

Derivation of c.  Every sum the kernels form is a chain of FP64 additions whose terms are slot products c_i c_j, each
added to a partial sum whose magnitude is at most the sum of |terms| so far; a chain of L additions therefore errs by at
most L eps sum |terms| (to first order).  The longest chain:
  * per warp: the loop kernel's DMMA adds 4 slots per instruction into one of two accumulator pairs (k1_reduce.cuh:
    gram_accumulate_dmma), K1 adds one slot per lane per chunk of 32 (k1_stream.cuh: accumulate); either way a
    warp's accumulator sees at most ceil(n / 8) additions of at most 4 products, i.e. <= n / 2 + 4 chained roundings
    for n slots in that warp, and no warp holds more than all n slots;
  * the tail: 5 shuffle rounds, 8 warps of a block, the block rows (at most n / 32 blocks hold a slot) in 8 interleaved
    sequences, 8 sequence totals, the 0.5 (G + G^T) symmetrisation: 5 + 8 + n / 256 + 8 + 1;
  * the congruence R^T H R: 9 FMA terms of two products each: 9 + 18 = 27 roundings, and R's entries are exact inputs.
  Hence c(n) = n / 2 + n / 256 + 64 covers both kernels; c is applied to sum m_i m_j, which bounds every partial sum.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

F = np.float32
EPS = 2.0 ** -52
FLT_MIN_NORMAL = 2.0 ** -126
BAND_FACTOR = 64.0
Q_BAND = 2.0 ** -50
REASONS = ("q", "rank", "norm", "thick", "gate", "store")


# ----------------------------------------------------------------------------------------------------------------------
# dla::colpiv_qr_solve<5,3>(A, b = -1): every system of the batch at once, same operations in the same order
# ----------------------------------------------------------------------------------------------------------------------
def qr53(A, dtype=np.float64):
    """A (K, 5, 3) float64; dtype np.longdouble runs the same algorithm in extended precision.  Returns (x (K, 3),
    rank-cut margins (K,)): the margin is min over the rank-cut tests the QR evaluated of
    |bign^2 - thr (M - k)| / max(bign^2, thr (M - k)) (1.0 where no test was close to a tie)."""
    A = np.array(A, dtype=dtype, copy=True)
    K, M, N = A.shape[0], 5, 3
    rows = np.arange(K)
    b = -np.ones((K, M), dtype)
    with np.errstate(all="ignore"):
        normU = np.zeros((K, N), dtype)
        for j in range(N):
            s = np.zeros(K, dtype)
            for i in range(M):
                s = s + A[:, i, j] * A[:, i, j]
            normU[:, j] = np.sqrt(s)
        normD = normU.copy()
        perm = np.tile(np.arange(N), (K, 1))
        maxn = np.zeros(K, dtype)
        for j in range(N):
            maxn = np.where(normU[:, j] > maxn, normU[:, j], maxn)
        thr = (maxn * EPS) * (maxn * EPS) / float(M)
        dd_thr = 1.4901161193847656e-08
        nz = np.full(K, N)
        margin = np.ones(K)
        for k in range(N):
            big = np.full(K, k)
            bign = normU[:, k].copy()
            for j in range(k + 1, N):
                up = normU[:, j] > bign
                bign = np.where(up, normU[:, j], bign)
                big = np.where(up, j, big)
            lhs, rhs = bign * bign, thr * float(M - k)
            live = nz == N
            m = np.abs(lhs - rhs) / np.maximum(np.maximum(lhs, rhs), 1e-300)
            margin = np.where(live, np.minimum(margin, m), margin)
            nz = np.where(live & (lhs < rhs), k, nz)
            sw = big != k
            if sw.any():
                r = rows[sw]
                bk = big[sw]
                colk = A[r, :, k].copy()
                A[r, :, k] = A[r, :, bk]
                A[r, :, bk] = colk
                for arr in (normU, normD, perm):
                    t = arr[r, k].copy()
                    arr[r, k] = arr[r, bk]
                    arr[r, bk] = t
            tail = np.zeros(K, dtype)
            for i in range(k + 1, M):
                tail = tail + A[:, i, k] * A[:, i, k]
            c0 = A[:, k, k].copy()
            small = tail <= 2.2250738585072014e-308
            beta = np.sqrt(c0 * c0 + tail)
            beta = np.where(c0 >= 0.0, -beta, beta)
            inv = 1.0 / (c0 - beta)
            for i in range(k + 1, M):
                A[:, i, k] = np.where(small, 0.0, A[:, i, k] * inv)
            tau = np.where(small, 0.0, (beta - c0) / beta)
            A[:, k, k] = np.where(small, c0, beta)
            for j in range(k + 1, N):
                tmp = A[:, k, j].copy()
                for i in range(k + 1, M):
                    tmp = tmp + A[:, i, k] * A[:, i, j]
                A[:, k, j] = A[:, k, j] - tau * tmp
                for i in range(k + 1, M):
                    A[:, i, j] = A[:, i, j] - tau * A[:, i, k] * tmp
            act = k < nz
            tmp = b[:, k].copy()
            for i in range(k + 1, M):
                tmp = tmp + A[:, i, k] * b[:, i]
            b[:, k] = np.where(act, b[:, k] - tau * tmp, b[:, k])
            for i in range(k + 1, M):
                b[:, i] = np.where(act, b[:, i] - tau * A[:, i, k] * tmp, b[:, i])
            for j in range(k + 1, N):
                nzc = normU[:, j] != 0.0
                t = np.abs(A[:, k, j]) / normU[:, j]
                t = (1.0 + t) * (1.0 - t)
                t = np.where(t < 0.0, 0.0, t)
                r_ = normU[:, j] / normD[:, j]
                t2 = t * r_ * r_
                s = np.zeros(K, dtype)
                for i in range(k + 1, M):
                    s = s + A[:, i, j] * A[:, i, j]
                fresh = np.sqrt(s)
                redo = nzc & (t2 <= dd_thr)
                keep = nzc & ~(t2 <= dd_thr)
                normD[:, j] = np.where(redo, fresh, normD[:, j])
                normU[:, j] = np.where(redo, fresh, np.where(keep, normU[:, j] * np.sqrt(t), normU[:, j]))
        c = np.zeros((K, N), dtype)
        for i in range(N - 1, -1, -1):
            s = b[:, i].copy()
            for j in range(i + 1, N):
                s = np.where(j < nz, s - A[:, i, j] * c[:, j], s)
            c[:, i] = np.where(i < nz, s / A[:, i, i], 0.0)
        x = np.zeros((K, N), dtype)
        for i in range(N):
            x[rows, perm[:, i]] = np.where(i < nz, c[:, i], 0.0)
    return x, margin


def _plane_of(x, nb, min_norm, thickness):
    """n = x / |x|, d = 1 / |x|, |x| and the worst squared distance of the five (fit_plane_reg's operations)"""
    ps = np.sqrt(x[:, 0] * x[:, 0] + x[:, 1] * x[:, 1] + x[:, 2] * x[:, 2])
    n = x / ps[:, None]
    d = 1.0 / ps
    worst = np.zeros(len(x), x.dtype)
    for j in range(5):
        e = n[:, 0] * nb[:, j, 0] + n[:, 1] * nb[:, j, 1] + n[:, 2] * nb[:, j, 2] + d
        worst = np.maximum(worst, e * e)
    return n, d, ps, worst


def fit_planes_qr(nb, min_norm=1e-6, thickness=0.2):
    """icp_test_runner.cpp:1727-1773 with qr53.  nb (K, 5, 3) float64.  Returns n (K, 3), d (K,), ok (K,), the same
    plane from the extended-precision QR (n_x (K, 3), d_x (K,)), and the band reason per system ("" = clear).

    The device's fit differs from this FP64 one by rounding only (FMA contraction); how far one FP64 evaluation of the
    fit lies from the exact one is measured per system against the extended-precision run of the same algorithm, and
    64 times that (with a floor of 64 kappa eps for a decision margin) is the uncertainty of the device's value."""
    K = nb.shape[0]
    x, rank_margin = qr53(nb)
    xl, _ = qr53(nb, np.longdouble)
    with np.errstate(all="ignore"):
        n, d, ps, worst = _plane_of(x, nb, min_norm, thickness)
        nl, dl, psl, worstl = _plane_of(xl, nb.astype(np.longdouble), min_norm, thickness)
        ok = (ps >= min_norm) & (worst < thickness * thickness)
        # condition of the system without its exactly-zero columns (the rank decision)
        zero_col = np.all(nb == 0.0, axis=1)                                 # (K, 3)
        sv = np.linalg.svd(np.where(zero_col[:, None, :], 0.0, nb), compute_uv=False)   # (K, 3) descending
        rank = 3 - zero_col.sum(axis=1)
        smax = sv[:, 0]
        smin = sv[np.arange(K), np.maximum(rank - 1, 0)]
        kappa = np.where(rank > 0, smax / np.maximum(smin, 1e-300), 1.0)
        deficient = (rank > 0) & (smin <= BAND_FACTOR * EPS * smax)
        reason = np.full(K, "", dtype=object)
        reason[(rank_margin < BAND_FACTOR * kappa * EPS) | deficient] = "rank"
        dps = BAND_FACTOR * (np.abs(ps - psl).astype(np.float64) + 4 * EPS * ps)
        dth = BAND_FACTOR * (np.abs(np.sqrt(worst) - np.sqrt(worstl)).astype(np.float64) + 4 * EPS * thickness)
        norm_band = ~(np.abs(ps - min_norm) > dps)
        thick_band = ~(np.abs(np.sqrt(worst) - thickness) > dth)
        reason[(reason == "") & norm_band] = "norm"
        reason[(reason == "") & thick_band & (ps >= min_norm)] = "thick"
    n = np.where(ok[:, None], n, 0.0)
    d = np.where(ok, d, 0.0)
    nl = np.where(ok[:, None], nl.astype(np.float64), 0.0)
    dl = np.where(ok, dl.astype(np.float64), 0.0)
    return n, d, ok, nl, dl, reason


# ----------------------------------------------------------------------------------------------------------------------
# float32 helpers
# ----------------------------------------------------------------------------------------------------------------------
def f32_boundary_distance(v):
    """|v - the nearest float32 rounding boundary| (a midpoint between adjacent float32 values), for FP64 v; inf for
    non-finite v"""
    v = np.asarray(v, np.float64)
    with np.errstate(all="ignore"):
        f = v.astype(F)
        fin = np.isfinite(f) & np.isfinite(v)
        up = np.nextafter(f, F(np.inf)).astype(np.float64)
        dn = np.nextafter(f, F(-np.inf)).astype(np.float64)
        f64 = f.astype(np.float64)
        dist = np.minimum(np.abs(v - 0.5 * (f64 + up)), np.abs(v - 0.5 * (f64 + dn)))
        # below the normal range the float32 spacing is fixed: the formula above still holds (gradual underflow)
    return np.where(fin, dist, np.inf)


def fl32(v):
    with np.errstate(all="ignore"):
        return np.asarray(v, np.float64).astype(F).astype(np.float64)


def transform_f32(p64, R, t):
    """pointBodyToGlobal: FP64, no FMA (x + y + z then + t, as numpy evaluates it term by term), float32 store"""
    with np.errstate(all="ignore"):
        w = p64[:, 0:1] * R[:, 0][None] + p64[:, 1:2] * R[:, 1][None]
        w = w + p64[:, 2:3] * R[:, 2][None]
        v = w + t[None]
    return v, fl32(v)


# ----------------------------------------------------------------------------------------------------------------------
# 5-NN: float32 distances, (d2, index) order
# ----------------------------------------------------------------------------------------------------------------------
def dist2_f32(q, pts):
    """corr::dist2 (pairwise): float32 differences, products and sums, x then y then z, no fused operations"""
    with np.errstate(all="ignore"):
        ex = (q[:, 0] - pts[:, 0]).astype(F)
        ey = (q[:, 1] - pts[:, 1]).astype(F)
        ez = (q[:, 2] - pts[:, 2]).astype(F)
        return ((ex * ex).astype(F) + (ey * ey).astype(F)).astype(F) + (ez * ez).astype(F)


def knn5(tree, tgt32, q32, radius):
    """The 5 nearest target points of every query by float32 d2, ties by index, among the points that can lie within
    the radius (a float64 ball of sqrt(r2_up) (1 + 1e-5) holds every point whose float32 d2 can be below r2_up).
    Returns idx (n, 5) (-1 padding), d5 (n,) float32 (inf when fewer than 5), near (n,) = d5 < radius^2."""
    n = len(q32)
    idx = np.full((n, 5), -1, np.int64)
    d5 = np.full(n, np.inf, F)
    fin = np.isfinite(q32).all(axis=1)
    sel = np.nonzero(fin)[0]
    if sel.size:
        r2 = radius * radius
        r2_up = F(r2)
        if float(r2_up) < r2:
            r2_up = np.nextafter(r2_up, F(np.inf))
        lists = tree.query_ball_point(q32[sel].astype(np.float64), float(np.sqrt(np.float64(r2_up))) * (1 + 1e-5),
                                      return_sorted=False)
        ln = np.array([len(x) for x in lists], np.int64)
        qi = np.repeat(sel, ln)
        ti = np.concatenate([np.asarray(x, np.int64) for x in lists]) if ln.sum() else np.zeros(0, np.int64)
        d2 = dist2_f32(q32[qi], tgt32[ti])
        key = (d2.view(np.uint32).astype(np.uint64) << np.uint64(32)) | ti.astype(np.uint64)
        order = np.lexsort((key, qi))
        qi, ti, d2 = qi[order], ti[order], d2[order]
        start = np.searchsorted(qi, np.arange(n))
        rank = np.arange(len(qi)) - start[qi]
        keep = rank < 5
        idx[qi[keep], rank[keep]] = ti[keep]
        five = keep & (rank == 4)
        d5[qi[five]] = d2[five]
    near = (idx[:, 4] >= 0) & (d5.astype(np.float64) < radius * radius)
    return idx, d5, near


# ----------------------------------------------------------------------------------------------------------------------
# the slot reference
# ----------------------------------------------------------------------------------------------------------------------
@dataclass
class SlotReference:
    H27: np.ndarray                 # (27,) reference frame (body frame), packed as the records
    sum_b2: float
    sum_r2: float
    n_pt: int
    n_eff: int
    n_eff_clear: int                # valid slots that are not in band
    n_band: int                     # slots in band
    n_pt_band: int                  # slots whose q is in band (N_pt may move by that many)
    allow: np.ndarray               # (29,) allowance of H27, sum b^2, sum r^2
    band: np.ndarray                # (n,) reason per slot, "" = clear
    valid: np.ndarray               # (n,) the reference's gate decision
    n_slots: int
    extras: dict = field(default_factory=dict)

    def band_counts(self):
        return {r: int(np.sum(self.band == r)) for r in REASONS if np.any(self.band == r)}

    def check(self, H27, sum_b2, sum_r2):
        """|error| / allowance per entry (29,)"""
        got = np.concatenate([np.asarray(H27, np.float64), [sum_b2, sum_r2]])
        ref = np.concatenate([self.H27, [self.sum_b2, self.sum_r2]])
        with np.errstate(all="ignore"):
            err = np.abs(got - ref)
            return np.where(err == 0.0, 0.0, err / self.allow)


def c_sum(n):
    return n / 2.0 + n / 256.0 + 64.0


def _pack_outer(a, b):
    """(K, 8) x (K, 8) -> (K, 29): the 21 upper-triangular H entries, the 6 rhs (a_i b_6), b_6 b_6, b_7 b_7"""
    out = []
    for i in range(6):
        for j in range(i, 6):
            out.append(a[:, i] * b[:, j])
    for i in range(6):
        out.append(a[:, i] * b[:, 6])
    out.append(a[:, 6] * b[:, 6])
    out.append(a[:, 7] * b[:, 7])
    return np.stack(out, axis=1) if out else np.zeros((len(a), 29))


def _slot_rows(p64, R, n, r, s, use_wd, slope):
    """The reference's rows (body frame) of slots with s > 0: (K, 8) = [J (6), b, r], plus u' = fl32(s n), k."""
    with np.errstate(all="ignore"):
        u = fl32(s[:, None] * n)
        nu = u / s[:, None]
        nR = nu @ R
        Jrot = np.cross(p64, nR)
        ds_dr = np.where((s > 0) & (s < 1), np.where(r > 0, -slope, slope), 0.0) if use_wd else np.zeros_like(s)
        w = s + r * ds_dr                                    # icp_test_runner.cpp:1780-1783, 1898
        k = w / s
        rows = np.empty((len(s), 8))
        rows[:, :3] = w[:, None] * Jrot
        rows[:, 3:6] = w[:, None] * nR
        rows[:, 6] = -fl32(s * r)
        rows[:, 7] = r
    return rows, u, k


def slot_sums(p64, R, q64, n, d, has, use_wd, slope, gate, dr, exact_r=None):
    """Weight, gate, rows and allowance of slots whose plane (n, d) is known.  dr: per-slot bound on the kernel's r
    minus this r.  exact_r: optional bool mask of slots whose r is computed identically by every evaluation order
    (designed inputs): their stores and gate need no uncertainty.  Returns a dict of per-slot arrays."""
    K = len(p64)
    with np.errstate(all="ignore"):
        r = n[:, 0] * q64[:, 0] + n[:, 1] * q64[:, 1] + n[:, 2] * q64[:, 2] + d
        s = 1.0 - slope * np.abs(r)
        finite = np.isfinite(r)                 # NaN / Inf r: s = max(0, NaN or -Inf) = 0 in the reference
        s = np.where(finite, np.maximum(0.0, s), 0.0)
        valid = has & finite & (s > gate)
        ds = slope * dr
        band = np.full(K, "", dtype=object)
        near_gate = np.abs(s - gate) <= np.maximum(1e-12, ds)
        band[has & finite & near_gate & ~exact_mask(exact_r, K)] = "gate"
        live = has & finite & (s > gate - np.maximum(1e-12, ds))   # rows of every slot that may be valid
        s_row = np.where(live, np.maximum(s, gate), 1.0)
        r_row = np.where(live, r, 0.0)
        n_row = np.where(live[:, None], n, 0.0)
        rows, u, k = _slot_rows(np.where(live[:, None], p64, 0.0), R, n_row, r_row, s_row, use_wd, slope)
        # stores: fl32(s n_i), fl32(s r) with the argument's own uncertainty
        sn = s_row[:, None] * n_row
        srr = s_row * r_row
        # d(s n_i) = n_i slope dr;  d(s r) = (s + slope |r|) dr = dr
        tol_n = np.abs(n_row) * ds[:, None] + 4 * EPS * np.abs(sn)
        tol_r = dr + 4 * EPS * np.abs(srr)
        em = exact_mask(exact_r, K)
        tol_n = np.where(em[:, None], 0.0, tol_n)
        tol_r = np.where(em, 0.0, tol_r)
        # (an exact slot's stores carry no uncertainty: one exactly on a tie rounds to even in both, so it is clear)
        near_n = (f32_boundary_distance(sn) <= tol_n) & (tol_n > 0)
        near_r = (f32_boundary_distance(srr) <= tol_r) & (tol_r > 0)
        store_band = live & (near_n.any(axis=1) | near_r)
        band[(band == "") & store_band] = "store"
        # magnitudes (world frame) and uncertainties of the row components
        pn = np.linalg.norm(np.where(live[:, None], p64, 0.0), axis=1)
        un = np.linalg.norm(u, axis=1)
        ka = np.abs(k)
        m = np.empty((K, 8))
        m[:, :3] = (ka * pn * un)[:, None]
        m[:, 3:6] = (ka * un)[:, None]
        m[:, 6] = np.abs(rows[:, 6])
        m[:, 7] = np.abs(r_row)
        dk = np.where(use_wd, ds / np.maximum(s_row, gate) ** 2, 0.0) + 4 * EPS * ka
        e = np.empty((K, 8))
        e[:, :3] = (dk * pn * un + 16 * EPS * ka * pn * un)[:, None]
        e[:, 3:6] = (dk * un + 4 * EPS * ka * un)[:, None]
        e[:, 6] = 0.0
        e[:, 7] = dr
        # documented deviation: the kernels' float32 round trip (k1::round_f32, k1s::rnd_f32) keeps a result below the
        # float32 normal range as a 24-bit FP64 value instead of a float32 denormal or zero
        sub_n = np.abs(sn) + tol_n
        sub_r = np.abs(srr) + tol_r
        un_sub = np.linalg.norm(np.where(sub_n < FLT_MIN_NORMAL, sub_n, 0.0), axis=1)
        e[:, :3] += (ka * pn * un_sub)[:, None]
        e[:, 3:6] += (ka * un_sub)[:, None]
        e[:, 6] += np.where(sub_r < FLT_MIN_NORMAL, sub_r, 0.0)
        # a store in band rounds to one of two adjacent floats: one float32 spacing (2^-23 relative) on the components
        # built from it, while the slot's validity does not depend on it
        sb = band == "store"
        e[sb, :6] += 2.0 ** -23 * m[sb, :6]
        e[sb, 6] += 2.0 ** -23 * m[sb, 6] + dr[sb] + FLT_MIN_NORMAL * 2.0 ** -23   # (|d(s r)| <= dr)
        m = np.where(live[:, None], m, 0.0)
        e = np.where(live[:, None], e, 0.0)
    return dict(r=r, s=s, valid=valid, band=band, rows=rows, m=m, e=e, live=live)


def exact_mask(exact_r, K):
    return np.zeros(K, bool) if exact_r is None else np.asarray(exact_r, bool)


def _assemble(valid, band, rows, m, e, extra_band_m, n_slots):
    """sums and allowance from per-slot arrays (a "store" band slot is accounted for through its e)"""
    clear = (band == "") | (band == "store")
    P = _pack_outer(rows[valid], rows[valid])
    sums = np.array([math.fsum(P[:, i]) for i in range(P.shape[1])]) if valid.any() else np.zeros(29)
    Mm = _pack_outer(m, m)
    Em = _pack_outer(e, m) + _pack_outer(m, e) + _pack_outer(e, e)
    allow = Mm[~clear].sum(axis=0) + Em[clear].sum(axis=0) + c_sum(max(n_slots, 1)) * EPS * Mm.sum(axis=0)
    if extra_band_m is not None and len(extra_band_m):
        allow += _pack_outer(extra_band_m, extra_band_m).sum(axis=0)
    return sums[:27], sums[27], sums[28], _block_spread(np.maximum(allow, 1e-300))


def _block_spread(allow):
    """The congruence R^T H R mixes the entries of each 3x3 block (and each 3-vector): spread every block's allowance to
    its largest value (a conservative bound for the body-frame entries)."""
    out = allow.copy()
    idx = {}
    q = 0
    for i in range(6):
        for j in range(i, 6):
            idx[(i, j)] = q
            q += 1
    for bi in (0, 3):
        for bj in (0, 3):
            if bj < bi:
                continue
            ent = [idx[(min(i, j), max(i, j))] for i in range(bi, bi + 3) for j in range(bj, bj + 3)]
            out[ent] = allow[ent].max() * 3.0
    for bi in (0, 3):
        ent = [21 + i for i in range(bi, bi + 3)]
        out[ent] = allow[ent].max() * 3.0
    return out


def q_band_mask(v):
    """a coordinate whose FP64 value lies within 2^-50 |v| of a float32 rounding boundary"""
    with np.errstate(all="ignore"):
        return (f32_boundary_distance(v) <= Q_BAND * np.abs(v)).any(axis=1)


def generic_m(p64, use_wd, slope, gate):
    """magnitude bound of any valid row of a slot: |u'| <= 1, |k| <= max over (gate, 1], |b|, |r| <= 1 / slope"""
    kmax = max(1.0, abs(2.0 - 1.0 / gate)) if use_wd else 1.0
    pn = np.linalg.norm(np.where(np.isfinite(p64), p64, 0.0), axis=1)
    m = np.empty((len(p64), 8))
    m[:, :3] = (kmax * pn)[:, None]
    m[:, 3:6] = kmax
    m[:, 6:] = 1.0 / slope
    return m


def iteration_reference(src32, tgt32, tree, T, radius, use_wd, slope=0.9, gate=0.1, min_norm=1e-6, thickness=0.2):
    """One iteration of the loop from pose T (4x4 FP64): the reference's sums over the source slots src32 (n, 3)
    float32 against tgt32 (m, 3) float32 (tree: cKDTree of tgt32 in float64)."""
    R, t = np.asarray(T, np.float64)[:3, :3], np.asarray(T, np.float64)[:3, 3]
    src32 = np.asarray(src32, F)[:, :3]
    N = len(src32)
    p64 = src32.astype(np.float64)
    qv, q32 = transform_f32(p64, R, t)
    qband = q_band_mask(qv) & np.isfinite(q32).all(axis=1)
    idx, d5, near = knn5(tree, np.asarray(tgt32, F), q32.astype(F), radius)
    n = np.zeros((N, 3)); d = np.zeros(N); has = np.zeros(N, bool)
    nx_ = np.zeros((N, 3)); dx_ = np.zeros(N)
    band = np.full(N, "", dtype=object)
    sel = np.nonzero(near)[0]
    if sel.size:
        nb = np.asarray(tgt32, F)[idx[sel]].astype(np.float64)
        nn, dd, ok, nl, dl, reason = fit_planes_qr(nb, min_norm, thickness)
        n[sel], d[sel], has[sel], nx_[sel], dx_[sel] = nn, dd, ok, nl, dl
        band[sel] = reason
    with np.errstate(all="ignore"):
        qf = np.where(np.isfinite(q32), q32, 0.0)
        # the device's r: its plane's rounding (64 x this FP64 fit's measured distance from the exact one at q) and the
        # FMA chain of r itself
        r64 = (n * qf).sum(axis=1) + d
        rx = (nx_ * qf).sum(axis=1) + dx_
        scale = np.linalg.norm(n, axis=1) * np.linalg.norm(qf, axis=1) + np.abs(d)
        dr = BAND_FACTOR * (np.abs(r64 - rx) + 4 * EPS * scale)
        dr += 8 * EPS * ((np.abs(n) * np.abs(qf)).sum(axis=1) + np.abs(d))
    # a plane-stage band only matters for a slot that is near (it decides whether a valid plane exists)
    out = slot_sums(p64, R, q32, n, d, has & near, use_wd, slope, gate, dr)
    fb = out["band"]
    band[(band == "") & (fb != "")] = fb[(band == "") & (fb != "")]
    band[qband] = "q"
    valid = out["valid"]
    # band slots without a reference row: the largest row they could have
    norow = (band != "") & ~out["live"]
    extra = generic_m(p64[norow], use_wd, slope, gate) if norow.any() else None
    m = out["m"].copy()
    qb_live = (band == "q") & out["live"]
    if qb_live.any():
        m[qb_live] = np.maximum(m[qb_live], generic_m(p64[qb_live], use_wd, slope, gate))
    H27, sb2, sr2, allow = _assemble(valid, band, out["rows"], m, out["e"], extra, N)
    clear = (band == "") | (band == "store")
    return SlotReference(H27=H27, sum_b2=sb2, sum_r2=sr2, n_pt=int(near.sum()), n_eff=int(valid.sum()),
                         n_eff_clear=int((valid & clear).sum()), n_band=int((~clear).sum()),
                         n_pt_band=int(qband.sum()), allow=allow, band=band, valid=valid, n_slots=N,
                         extras=dict(n=n, d=d, has=has, near=near, r=out["r"], s=out["s"], idx=idx, q32=q32))


# ----------------------------------------------------------------------------------------------------------------------
# the streaming kernel's seam: points and planes given (dcreg_reduce_normal_equations)
# ----------------------------------------------------------------------------------------------------------------------
def _exact_fma(a, b, c):
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _r_is_exact(q, n, d):
    """r = n.q + d is the same double under the reference's order and the kernel's FMA chain"""
    if not (np.isfinite(q).all() and np.isfinite(n).all() and math.isfinite(d)):
        return False
    plain = float(n[0] * q[0] + n[1] * q[1] + n[2] * q[2] + d)
    chain = _exact_fma(n[0], q[0], _exact_fma(n[1], q[1], _exact_fma(n[2], q[2], d)))
    return plain == chain


def k1_reference(src4, plane4, T, use_wd, slope=0.9, gate=0.1, designed=None):
    """The reference's sums over the (point, plane) slots of the K1 seam: src4 (n, 4) float32, plane4 (n, 4) float32 or
    float64 (nx, ny, nz, d); a slot whose normal is all zero has no plane.  designed: indices of hand-made slots whose
    r is checked for exactness (their gate and stores carry no uncertainty when every evaluation order agrees)."""
    R, t = np.asarray(T, np.float64)[:3, :3], np.asarray(T, np.float64)[:3, 3]
    N = len(src4)
    p64 = np.asarray(src4, F)[:, :3].astype(np.float64)
    pl = np.asarray(plane4)
    n = pl[:, :3].astype(np.float64)
    d = pl[:, 3].astype(np.float64)
    qv, q64 = transform_f32(p64, R, t)
    with np.errstate(all="ignore"):
        has = (n != 0.0).any(axis=1) & np.isfinite(n).all(axis=1) & np.isfinite(d)   # a (non-zero, finite) plane
        fin = np.isfinite(q64).all(axis=1) & np.isfinite(n).all(axis=1) & np.isfinite(d) & np.isfinite(p64).all(axis=1)
        qs = np.where(np.isfinite(q64), q64, 0.0)
        dr = 8 * EPS * ((np.abs(n) * np.abs(qs)).sum(axis=1) + np.abs(d))
        dr = np.where(fin, dr, 0.0)
    qband = q_band_mask(qv) & fin
    exact = np.zeros(N, bool)
    if designed is not None:
        for i in designed:
            if fin[i] and not qband[i] and _r_is_exact(q64[i], n[i], d[i]):
                exact[i] = True
                dr[i] = 0.0
    if pl.dtype == np.float32:
        # documented deviation: K1's float -> double conversion of a plane maps +-0 and float32 denormals to
        # +-2^-127-sized values (k1_stream.cuh: f32_f64), which moves r by up to 2^-126 (|q_i| of each such component,
        # + 1 for d): negligible at ordinary coordinates, a gate decision near 1e38 m
        small = np.abs(pl.astype(np.float64)) < 2.0 ** -126
        with np.errstate(all="ignore"):
            dz = 2.0 ** -126 * ((small[:, :3] * np.abs(np.where(np.isfinite(q64), q64, 0.0))).sum(axis=1) + small[:, 3])
        dz = np.where(fin, dz, 0.0)
        dr = dr + dz
        exact &= dz == 0.0
    pz = np.where(np.isfinite(p64), p64, 0.0)
    out = slot_sums(pz, R, np.where(fin[:, None], q64, 0.0), np.where(fin[:, None], n, 0.0), np.where(fin, d, 0.0),
                    has & fin, use_wd, slope, gate, dr, exact_r=exact)
    band = out["band"]
    band[qband] = "q"
    valid = out["valid"]
    if designed is not None:
        # a designed slot exactly at the gate: s under the kernel's fma(|r|, -slope, 1) must agree too
        for i in designed:
            if exact[i] and has[i]:
                r = float(out["r"][i])
                s_fma = _exact_fma(abs(r), -slope, 1.0)
                if (s_fma > gate) != bool(valid[i]):
                    band[i] = "gate"
    norow = (band != "") & ~out["live"]
    extra = generic_m(pz[norow], use_wd, slope, gate) if norow.any() else None
    m = out["m"].copy()
    qb_live = (band == "q") & out["live"]
    if qb_live.any():
        m[qb_live] = np.maximum(m[qb_live], generic_m(pz[qb_live], use_wd, slope, gate))
    H27, sb2, sr2, allow = _assemble(valid, band, out["rows"], m, out["e"], extra, N)
    clear = (band == "") | (band == "store")
    return SlotReference(H27=H27, sum_b2=sb2, sum_r2=sr2, n_pt=int(has.sum()), n_eff=int(valid.sum()),
                         n_eff_clear=int((valid & clear).sum()), n_band=int((~clear).sum()), n_pt_band=0, allow=allow,
                         band=band, valid=valid, n_slots=N, extras=dict(r=out["r"], s=out["s"], exact=exact))
