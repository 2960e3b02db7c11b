"""CPU property test of the loop kernel's gap certificate (DESIGN.md §3, icp_iter2_kernel), independent of CUDA.

The kernel skips a slot's neighbour search when   (sqrt(d5') + delta) * 1.00002 + 1e-7 < sqrt(lb) * 0.99998   where d5' is
the 5th smallest of the new float32 squared distances to the slot's seven stored neighbours, delta = |q - q_scan| and lb a
lower bound on the squared distance from q_scan to every target point outside the seven.  This test restates that rule
in NumPy float32 arithmetic (same operation order as corr::dist2) with the TIGHTEST valid lb (the 8th smallest
distance) and checks against brute force, on random clouds, exact lattices (ties -> index rule) and clouds with
duplicated points, that whenever the rule says "skip" the re-ranked first five of the seven ARE the five nearest
(ascending (d2, index)) of the moved query.
"""
import numpy as np
import pytest

F = np.float32


def dist2(q, pts, pairwise=False):
    """corr::dist2: float32 differences, products and sums, x then y then z, no fused operations.  Every query against
    every point ((m, n) result), or with pairwise=True query i against point i."""
    if not pairwise:
        q, pts = q[:, None, :], pts[None, :, :]
    ex = (q[..., 0] - pts[..., 0]).astype(F)
    ey = (q[..., 1] - pts[..., 1]).astype(F)
    ez = (q[..., 2] - pts[..., 2]).astype(F)
    return ((ex * ex).astype(F) + (ey * ey).astype(F)).astype(F) + (ez * ez).astype(F)


def order(d2):
    """ascending (d2, index): stable argsort on d2 realises the index rule"""
    return np.argsort(d2, axis=1, kind="stable")


def clouds():
    rng = np.random.default_rng(11)
    yield "random", rng.uniform(-3, 3, (1500, 3)).astype(F)
    g = np.arange(-3, 3, 0.25, dtype=F)
    X, Y = np.meshgrid(g, g)
    lat = np.stack([X.ravel(), Y.ravel(), np.zeros(X.size, F)], axis=1).astype(F)
    yield "lattice", lat
    yield "lattice+duplicates", np.concatenate([lat, lat[::3], lat[::7]]).astype(F)
    surf = rng.uniform(-3, 3, (1500, 3)).astype(F)
    surf[:, 2] = (0.05 * np.sin(surf[:, 0])).astype(F)
    yield "surface", surf


@pytest.mark.parametrize("name,pts", list(clouds()), ids=[n for n, _ in clouds()])
def test_certificate_never_skips_a_changed_neighbour_set(name, pts):
    rng = np.random.default_rng(5)
    q0 = (pts[rng.integers(0, len(pts), 400)] + rng.normal(0, 0.05, (400, 3))).astype(F)
    d0 = dist2(q0, pts)
    o0 = order(d0)
    seven = o0[:, :7]
    lb = np.take_along_axis(d0, o0[:, 7:8], axis=1)[:, 0]            # tightest valid bound: the 8th smallest distance
    skipped = 0
    for scale in (1e-6, 1e-4, 1e-3, 1e-2, 3e-2, 0.1, 0.3):
        for _rep in range(3):
            q1 = (q0 + rng.normal(0, scale, q0.shape)).astype(F)
            e = (q1 - q0).astype(F)
            delta = np.sqrt(((e[:, 0] * e[:, 0]).astype(F) + (e[:, 1] * e[:, 1]).astype(F)).astype(F) + (e[:, 2] * e[:, 2]).astype(F)).astype(F)
            d1 = dist2(q1, pts)
            d7 = np.take_along_axis(d1, seven, axis=1)
            idx7 = seven                                               # original index = position here
            # re-rank the seven by (d2, index)
            key = np.lexsort((idx7, d7), axis=1)
            ranked = np.take_along_axis(idx7, key, axis=1)
            d5 = np.take_along_axis(d7, key, axis=1)[:, 4]
            skip = (np.sqrt(d5).astype(F) + delta).astype(F) * F(1.00002) + F(1e-7) < np.sqrt(lb).astype(F) * F(0.99998)
            truth = order(d1)[:, :5]
            bad = skip & (ranked[:, :5] != truth).any(axis=1)
            assert not bad.any(), (name, scale, int(bad.sum()))
            skipped += int(skip.sum())
    if name in ("random", "surface"):
        assert skipped > 1000          # the rule is not vacuous: most small motions are certified
