"""The neighbour searches of corr.cuh, query by query, against a float32 brute force.

tools/test_corr_search.cu runs the production device functions (knn_search on the dense grid and on the sparse row
index of the same points, knn_search_lb, knn_warp_search with and without the loop kernel's row table, knn_row_range,
nn1_search) and corr.cuh's grid build kernels on a grid and queries written by this file; the reference here is NumPy:

  * the layout twin (grid_layout): cell coordinates floor(float64(v) * (1 / cell)), the points' min / max cell as the
    box, x-fastest cells, ascending original index inside a cell, .w = the index bit-cast to float32, cell_start the
    exclusive scan of the cell counts and pos_of its inverse;
  * distances: corr::dist2 (FLANN L2_Simple in float32, harness.dist2), ordered by the key
    (bits(d2) << 32) | index: the (distance, then index) rule of the kd-tree the searches replace;
  * the cube of a query: the points whose cell differs from the query's cell by at most K = rings on each axis.

Contracts, bit for bit on keys and positions:
  knn_search (dense)  the 5 smallest keys of the cube, padded with knn_key(3e38, 0x7fffffff)
  knn_search (sparse) the dense result
  knn_search_lb       the 7 smallest keys of the cube below knn_key(B, 0x7fffffff) (d2 == B with a real index is kept),
                      padded with that sentinel at position -1; positions are pos_of[index]
  knn_warp_search     got == (cube points with d2 <= B) <= 64; when got, knn_search_lb's list; with the row table
                      (rings == 1) bit-identical to without it, lb included
  knn_row_range       every cube point of the row outside [s, e) has d2 > B, and lb <= its d2
  nn1_search          the smallest float32 d2 over all points
  grid build          the layout twin, byte for byte
and for the lb of both bounded searches: sound (lb <= the d2 of every target point not in the list, all points, so it
also checks that nothing beyond the rings is nearer than the starting bound r2_up * 0.9999) and not vacuous
(lb >= min(r2_up * 0.9999, d2 of the 7th entry): every contribution to lb comes from a candidate, cell or row rejected
against the current 7th entry, which only decreases).
"""
import subprocess

import numpy as np
import pytest

from harness import dist2, tool_program
from search_harness import (CELLS, CLOUDS, RADIUS, SENT, WARP_CAP, F, Layout, Reference, bounds_for, cloud, expand,
                            first_bad, key_d2, key_idx, make_queries, on_face, r2_up, rings_of, write_input)


class Ball:
    """Every target point that can have a float32 d2 below r2_up, per query.  Prefilter: a float64 kd-tree ball of
    radius sqrt(r2_up) (1 + 1e-5).  A float32 d2 is the exact squared distance of the float inputs times (1 +- 5 u),
    u = 2^-24 (one rounding per difference, product and sum), so a point outside that ball has a float32 d2 above
    r2_up (1 + 2e-5) (1 - 3e-7) > r2_up: none is lost."""

    def __init__(self, tree, pts, q, r2):
        lists = tree.query_ball_point(q.astype(np.float64), float(np.sqrt(np.float64(r2))) * (1 + 1e-5), return_sorted=False)
        ln = np.array([len(x) for x in lists])
        self.qi = np.repeat(np.arange(len(q)), ln)
        self.idx = np.concatenate([np.asarray(x, np.int64) for x in lists]) if ln.sum() else np.zeros(0, np.int64)
        self.d2 = dist2(q[self.qi], pts[self.idx], pairwise=True)

    def min_outside(self, list_keys, n):
        """per query the smallest float32 d2 of a point within the ball that is not in its list (inf: none)"""
        nq, k = list_keys.shape
        idx = key_idx(list_keys)
        member = (np.arange(nq)[:, None] * (n + 1) + np.where(idx == SENT, n, idx)).ravel()
        out_pt = ~np.isin(self.qi * (n + 1) + self.idx, member)
        m = np.full(nq, np.inf)
        np.minimum.at(m, self.qi[out_pt], self.d2[out_pt].astype(np.float64))
        return m


def nn1_reference(tree, pts, q):
    """smallest float32 d2 over all points: the float64 nearest distance d, then every point within d (1 + 1e-5) in
    float32 (the float32 minimum lies within d (1 + 3e-7) by the error bound in Ball)"""
    d, _ = tree.query(q.astype(np.float64), k=1)
    lists = tree.query_ball_point(q.astype(np.float64), d * (1 + 1e-5) + 1e-30, return_sorted=False)
    return np.array([dist2(q[i:i + 1], pts[np.asarray(x, np.int64)]).min() for i, x in enumerate(lists)], F)


# ---- the harness --------------------------------------------------------------------------------------------------
def read_output(path, nq, nrr):
    buf = open(path, "rb").read()
    at = 0

    def take(dtype, count, shape=None):
        nonlocal at
        a = np.frombuffer(buf, dtype=dtype, count=count, offset=at)
        at += a.nbytes
        return a.reshape(shape) if shape else a

    out = {"knn5": take(np.uint64, nq * 5, (nq, 5)), "knn5s": take(np.uint64, nq * 5, (nq, 5)),
           "lb_keys": take(np.uint64, nq * 7, (nq, 7)), "lb_pos": take(np.int32, nq * 7, (nq, 7)), "lb": take(F, nq)}
    for w in ("warp", "pre"):
        out[w] = {"got": take(np.int32, nq), "keys": take(np.uint64, nq * 7, (nq, 7)),
                  "pos": take(np.int32, nq * 7, (nq, 7)), "lb": take(F, nq)}
    out["nn1"] = take(F, nq)
    rro = take(np.int32, nrr * 3, (nrr, 3))
    out["rr_s"], out["rr_e"], out["rr_lb"] = rro[:, 0], rro[:, 1], rro[:, 2].copy().view(F)
    out["bounds"] = take(np.int32, 6)
    out["same"] = take(np.int32, 3)
    assert at == len(buf)
    return out


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return tool_program(tmp_path_factory.mktemp("corr_search"), "test_corr_search.cu", compiler="device",
                        skip_missing=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
@pytest.mark.parametrize("name", CLOUDS)
def test_searches_match_brute_force(harness, tmp_path, name, cell):
    from scipy.spatial import cKDTree
    pts = cloud(name)
    n = len(pts)
    L = Layout(pts, cell)
    K = rings_of(RADIUS, cell)
    r2 = r2_up(RADIUS)
    lb0 = F(r2 * F(0.9999))
    kind0, q0 = make_queries(name, pts, L, K, cell, seed=CLOUDS.index(name) * 10 + CELLS.index(cell))
    tree = cKDTree(pts.astype(np.float64))
    Bs = bounds_for(tree, pts, q0, r2)
    rng = np.random.default_rng(99)
    perm = rng.permutation(4 * len(q0))                          # one warp of the per-thread searches mixes kinds
    q = np.tile(q0, (4, 1))[perm]
    kind = np.tile(kind0, 4)[perm]
    B = np.concatenate(Bs)[perm]
    variant = np.repeat(np.arange(4), len(q0))[perm]
    nq = len(q)
    W2 = (2 * K + 1) ** 2
    rq = np.flatnonzero(np.arange(nq) % 3 == 0)                   # every row of a third of the queries
    rr = np.stack([np.repeat(rq, W2), np.tile(np.arange(W2), len(rq))], axis=1)

    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    write_input(inp, pts, L, K, r2, q, B, rr)
    res = subprocess.run([str(harness), str(inp), str(outp)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    o = read_output(outp, nq, len(rr))
    ref = Reference(pts, L, K, q, B)
    ball = Ball(tree, pts, q, r2)
    where = lambda m: f"query {first_bad(m)} ({kind[first_bad(m)]}, q={q[first_bad(m)].tolist()}, B={B[first_bad(m)]!r})"

    # the grid build kernels reproduce the layout the searches ran on
    assert o["bounds"].tolist() == [*L.o, *(L.o + L.n3 - 1)]
    assert o["same"].tolist() == [1, 1, 1], "grid build: pts / pos_of / cell_start differ from the layout twin"

    # knn_search: the cube's five smallest keys, on the dense grid and on the sparse row index
    bad = (o["knn5"] != ref.knn5).any(axis=1)
    assert not bad.any(), f"knn_search: {int(bad.sum())} lists differ, first {where(bad)}: {o['knn5'][first_bad(bad)]} " \
                          f"!= {ref.knn5[first_bad(bad)]}"
    bad = (o["knn5s"] != o["knn5"]).any(axis=1)
    assert not bad.any(), f"knn_search on the sparse row index: {int(bad.sum())} lists differ, first {where(bad)}"

    # knn_search_lb: the cube's seven smallest keys inside the bound, positions, and lb
    bad = (o["lb_keys"] != ref.lb_keys).any(axis=1) | (o["lb_pos"] != ref.lb_pos).any(axis=1)
    assert not bad.any(), f"knn_search_lb: {int(bad.sum())} lists differ, first {where(bad)}: " \
                          f"{o['lb_keys'][first_bad(bad)]} != {ref.lb_keys[first_bad(bad)]}"

    def check_lb(lb, keys, sel, what):
        outside = ball.min_outside(keys, n)
        bad = sel & ~(lb.astype(np.float64) <= outside)
        assert not bad.any(), f"{what}: lb above the d2 of a point outside the list, {int(bad.sum())} queries, first " \
                              f"{where(bad)}: lb {lb[first_bad(bad)]!r} > {outside[first_bad(bad)]!r}"
        bad = sel & ~(lb <= lb0)
        assert not bad.any(), f"{what}: lb above the starting bound, first {where(bad)}"
        floor_ = np.minimum(lb0, key_d2(keys[:, 6]))
        bad = sel & ~(lb >= floor_)
        assert not bad.any(), f"{what}: lb below min(r2_up * 0.9999, 7th d2), first {where(bad)}: " \
                              f"{lb[first_bad(bad)]!r} < {floor_[first_bad(bad)]!r}"

    check_lb(o["lb"], o["lb_keys"], np.ones(nq, bool), "knn_search_lb")

    # knn_warp_search: gives up exactly when more than 64 cube points lie inside the bound; otherwise knn_search_lb's list
    w = o["warp"]
    got = w["got"].astype(bool)
    bad = got != (ref.n_in <= WARP_CAP)
    assert not bad.any(), f"knn_warp_search: got != (inside <= 64), first {where(bad)}: got {got[first_bad(bad)]}, " \
                          f"{ref.n_in[first_bad(bad)]} inside"
    bad = got & ((w["keys"] != ref.lb_keys).any(axis=1) | (w["pos"] != ref.lb_pos).any(axis=1))
    assert not bad.any(), f"knn_warp_search: {int(bad.sum())} lists differ, first {where(bad)}"
    check_lb(w["lb"], w["keys"], got, "knn_warp_search")
    if K == 1:
        p = o["pre"]
        for f in ("got", "keys", "pos"):
            assert np.array_equal(p[f], w[f]), f"knn_warp_search with the row table: {f} differs"
        assert p["lb"].tobytes() == w["lb"].tobytes(), "knn_warp_search with the row table: lb differs"

    # knn_row_range: [s, e) inside the row's cube range; everything of the row it drops is beyond B and not below lb
    qi, r = rr[:, 0], rr[:, 1]
    rs, re_ = ref.rs[qi, r], ref.re[qi, r]
    s, e, rlb = o["rr_s"].astype(np.int64), o["rr_e"].astype(np.int64), o["rr_lb"]
    empty = s >= e
    bad = ~empty & ((s < rs) | (e > re_))
    assert not bad.any(), f"knn_row_range: [s, e) leaves the row's cube range, pair {first_bad(bad)}"
    own, pos = expand(np.concatenate([rs, np.where(empty, rs, e)]), np.concatenate([np.where(empty, re_, s), re_]))
    pair = own % len(rr)
    d2 = dist2(q[qi[pair]], L.pts4[pos, :3], pairwise=True)
    bad_pt = (d2 <= B[qi[pair]]) | (d2 < rlb[pair])
    assert not bad_pt.any(), f"knn_row_range: dropped a point with d2 <= B or d2 < lb: pair {pair[first_bad(bad_pt)]} " \
                             f"(query {qi[pair[first_bad(bad_pt)]]}, row {r[pair[first_bad(bad_pt)]]}), d2 " \
                             f"{d2[first_bad(bad_pt)]!r}, B {B[qi[pair[first_bad(bad_pt)]]]!r}, lb {rlb[pair[first_bad(bad_pt)]]!r}"

    # nn1_search: the smallest d2 over all points
    nn1 = nn1_reference(tree, pts, q)
    bad = o["nn1"] != nn1
    assert not bad.any(), f"nn1_search: {int(bad.sum())} differ, first {where(bad)}: {o['nn1'][first_bad(bad)]!r} " \
                          f"!= {nn1[first_bad(bad)]!r}"

    # the inputs reach the cases they are meant for
    c = L.local_cell(q)
    outside_box = ((c < 0) | (c >= L.n3)).any(axis=1)
    on_face_ = (L.local_cell(np.nextafter(q, F(-np.inf))) != c).any(axis=1)   # the first float of its cell on an axis
    stats = {
        "overflow": int((~got).sum()),
        "sentinels": int((key_idx(o["lb_keys"][:, 6]) == SENT).sum()),
        "short5": int((key_idx(o["knn5"][:, 4]) == SENT).sum()),
        "d2==B": int((key_d2(o["lb_keys"]) == B[:, None]).any(axis=1).sum()),
        "face": int((kind == "face").sum()),
        "out-of-box found": int((outside_box & (key_idx(o["knn5"][:, 0]) != SENT)).sum()),
        "far": int((kind == "far").sum()),
    }
    print(f"\n{name} cell {cell} rings {K}: {n} points, {nq} queries, {len(rr)} row pairs; " +
          ", ".join(f"{k} {v}" for k, v in stats.items()))
    assert stats["sentinels"] > 0 and stats["face"] > 0 and on_face_[kind == "face"].all() and stats["far"] > 0
    assert stats["d2==B"] > 0
    assert (variant == 3).any() and (key_idx(o["lb_keys"][variant == 3, 6]) == SENT).all()
    if name == "lattice":
        assert stats["overflow"] > 0
    if name == "sparse":
        assert stats["short5"] > 0
    if K > 1:
        assert stats["out-of-box found"] > 0


# ---- CPU checks of the reference itself ----------------------------------------------------------------------------
def test_harness_compiles_for_sm90a(tmp_path):
    """tools/test_corr_search.cu builds with the library's flags (no GPU needed to compile)."""
    tool_program(tmp_path, "test_corr_search.cu", compiler="device")


@pytest.mark.parametrize("cell", CELLS)
@pytest.mark.parametrize("name", ["lattice", "surface+30000"])
def test_layout_twin_invariants(name, cell):
    pts = cloud(name)
    n = len(pts)
    L = Layout(pts, cell)
    cs = L.cell_start.astype(np.int64)
    assert cs[0] == 0 and cs[-1] == n and (np.diff(cs) >= 0).all()
    c = L.local_cell(pts)
    assert (c.min(axis=0) == 0).all() and (c.max(axis=0) == L.n3 - 1).all()
    # every point sits in its cell's range, the ranges in x-fastest order, ascending index inside a cell
    cell_at = np.searchsorted(cs, np.arange(n), side="right") - 1
    lin = (c[:, 2] * L.n3[1] + c[:, 1]) * L.n3[0] + c[:, 0]
    assert np.array_equal(cell_at, lin[L.order])
    same_cell = cell_at[1:] == cell_at[:-1]
    assert (np.diff(L.order)[same_cell] > 0).all()
    assert np.array_equal(L.pts4[:, 3].view(np.int32), L.order)
    assert np.array_equal(L.pts4[:, :3], pts[L.order])
    assert np.array_equal(L.pos_of[L.order], np.arange(n))


def test_face_queries_start_their_cells():
    for cell in CELLS:
        inv = 1.0 / cell
        v = np.random.default_rng(3).uniform(-50, 50, 2000).astype(F)
        x = on_face(v, inv)
        k = np.floor(v.astype(np.float64) * inv)
        assert np.array_equal(np.floor(x.astype(np.float64) * inv), k)
        assert (np.floor(np.nextafter(x, F(-np.inf)).astype(np.float64) * inv) == k - 1).all()


@pytest.mark.parametrize("cell", CELLS)
def test_reference_lists_match_kdtree(cell):
    """On tie-free random points the reference's lists are the kd-tree's nearest neighbours wherever the cube holds
    them: the cube contains the ball of radius K cell around the query, and the bounded list the ball of radius
    sqrt(B) = the search radius."""
    from scipy.spatial import cKDTree
    rng = np.random.default_rng(41)
    pts = rng.uniform(-2.0, 2.0, (800, 3)).astype(F)                   # ~6.5 points within the radius of a point
    q = (pts[rng.integers(0, len(pts), 1_500)] + rng.normal(0, 0.2, (1_500, 3))).astype(F)
    L = Layout(pts, cell)
    K = rings_of(RADIUS, cell)
    r2 = r2_up(RADIUS)
    B = np.full(len(q), r2, F)
    ref = Reference(pts, L, K, q, B)
    d, nb = cKDTree(pts.astype(np.float64)).query(q.astype(np.float64), k=8)
    clear = lambda x, t: np.abs(x / t - 1.0) > 1e-5                    # no float32 / float64 ambiguity at the edge
    ok5 = (d[:, 4] < K * cell * (1 - 1e-5))
    assert ok5.sum() > 300
    assert np.array_equal(key_idx(ref.knn5[ok5]), nb[ok5, :5])
    assert np.array_equal(key_d2(ref.knn5[ok5]), np.stack([dist2(q[i:i + 1], pts[nb[i, :5]])[0] for i in np.flatnonzero(ok5)]))
    sel = clear(d[:, :8], RADIUS).all(axis=1)
    inside = d < RADIUS
    assert sel.sum() > 1000 and inside[sel, 6].any()
    for i in np.flatnonzero(sel):
        want = nb[i, :7][inside[i, :7]]
        got = key_idx(ref.lb_keys[i])
        assert np.array_equal(got[:len(want)], want) and (got[len(want):] == SENT).all()
        assert np.array_equal(ref.lb_pos[i, :len(want)], L.pos_of[want]) and (ref.lb_pos[i, len(want):] == -1).all()
    few = sel & ~inside[:, 7]                                          # all points inside the radius are among the eight
    assert few.sum() > 100 and np.array_equal(ref.n_in[few], inside[few].sum(axis=1))
