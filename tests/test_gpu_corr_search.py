"""The neighbour searches of corr.cuh, query by query, against a float32 brute force.

tools/test_corr_search.cu runs the production device functions (knn_search on the dense grid and on the sparse row
index of the same points, knn_search_lb, knn_warp_search with and without the loop kernel's row table, knn_row_range,
nn1_search) and corr.cuh's grid build kernels on a grid and queries written by this file; the reference here is NumPy:

  * the layout twin (grid_layout): cell coordinates floor(float64(v) * (1 / cell)), the points' min / max cell as the
    box, x-fastest cells, ascending original index inside a cell, .w = the index bit-cast to float32, cell_start the
    exclusive scan of the cell counts and pos_of its inverse;
  * distances: corr::dist2 (FLANN L2_Simple in float32, test_certificate_logic.dist2), ordered by the key
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
import functools
import os
import subprocess

import numpy as np
import pytest

from test_certificate_logic import dist2

F = np.float32
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tools", "test_corr_search.cu")
MAGIC = 0x43525331
RADIUS = 0.5
CELLS = [0.5, 0.3, 0.25, 0.2, 0.125]                 # rings 1, 2, 2, 3, 4
SENT = 0x7FFFFFFF
LOOK = F(1.21)                                       # kNnLook: the seeded bound is 1.21 x the 7th squared distance
WARP_CAP = 64                                        # kWarpKnnCap


def rings_of(radius, cell):
    """search_rings in dcreg_b200.cu"""
    return int(np.ceil(radius / cell - 1e-9))


def r2_up(radius):
    r2 = radius * radius
    f = F(r2)
    return np.nextafter(f, F(np.inf)) if float(f) < r2 else f


def keys_of(d2, idx):
    d2 = np.asarray(d2, F)
    return (d2.view(np.uint32).astype(np.uint64) << np.uint64(32)) | np.asarray(idx, np.int64).astype(np.uint64)


def key_d2(keys):
    return (np.asarray(keys, np.uint64) >> np.uint64(32)).astype(np.uint32).view(F)


def key_idx(keys):
    return (np.asarray(keys, np.uint64) & np.uint64(0xFFFFFFFF)).astype(np.int64)


# ---- the layout twin ----------------------------------------------------------------------------------------------
class Layout:
    def __init__(self, pts, cell):
        self.inv = 1.0 / cell
        c = np.floor(pts.astype(np.float64) * self.inv).astype(np.int64)
        self.o = c.min(axis=0)
        self.n3 = c.max(axis=0) - self.o + 1
        nx, ny, _ = self.n3
        lin = ((c[:, 2] - self.o[2]) * ny + (c[:, 1] - self.o[1])) * nx + (c[:, 0] - self.o[0])
        self.ncells = int(np.prod(self.n3))
        self.lin = lin
        self.order = np.argsort(lin, kind="stable")          # by cell, then by index
        self.cell_start = np.zeros(self.ncells + 1, np.int32)
        self.cell_start[1:] = np.cumsum(np.bincount(lin, minlength=self.ncells))
        self.pts4 = np.empty((len(pts), 4), F)
        self.pts4[:, :3] = pts[self.order]
        self.pts4[:, 3] = self.order.astype(np.int32).view(F)
        self.pos_of = np.empty(len(pts), np.int32)
        self.pos_of[self.order] = np.arange(len(pts), dtype=np.int32)

    def local_cell(self, q):
        return np.floor(np.asarray(q, F).astype(np.float64) * self.inv).astype(np.int64) - self.o

    def row_ranges(self, q, K):
        """position range [s, e) in pts4 of the cube cells of every (query, row), rows r = (dz + K) W + (dy + K),
        W = 2K + 1, as knn_row_range numbers them; (nq, W^2) each, s == e where the row holds nothing"""
        c = self.local_cell(q)
        W = 2 * K + 1
        r = np.arange(W * W)
        dz, dy = r // W - K, r % W - K
        nx, ny, nz = self.n3
        yy, zz = c[:, 1:2] + dy[None], c[:, 2:3] + dz[None]
        valid = (yy >= 0) & (yy < ny) & (zz >= 0) & (zz < nz)
        base = np.where(valid, (zz * ny + yy) * nx, 0)
        xa = np.clip(c[:, 0:1] - K, 0, nx)
        xb = np.clip(c[:, 0:1] + K + 1, 0, nx)
        s = np.where(valid, self.cell_start[base + xa], 0)
        e = np.where(valid, self.cell_start[base + xb], 0)
        return s, np.maximum(e, s)


def expand(s, e):
    """the ranges [s, e) as flat (range number, position) pairs"""
    s, e = s.ravel().astype(np.int64), e.ravel().astype(np.int64)
    ln = e - s
    owner = np.repeat(np.arange(len(s)), ln)
    pos = np.arange(int(ln.sum())) - np.repeat(np.cumsum(ln) - ln, ln) + np.repeat(s, ln)
    return owner, pos


def smallest(group, keys, ngroups, k, fill_keys, payload=None, fill_payload=-1):
    """per group the k smallest keys, ascending, padded with fill_keys[group] (and the payload of each key)"""
    order = np.lexsort((keys, group))
    g, ks = group[order], keys[order]
    rank = np.arange(len(g)) - np.searchsorted(g, np.arange(ngroups))[g]
    keep = rank < k
    out = np.repeat(np.asarray(fill_keys, np.uint64).reshape(-1, 1), k, axis=1) if np.ndim(fill_keys) else \
        np.full((ngroups, k), fill_keys, np.uint64)
    out[g[keep], rank[keep]] = ks[keep]
    if payload is None:
        return out
    pay = np.full((ngroups, k), fill_payload, np.int64)
    pay[g[keep], rank[keep]] = payload[order][keep]
    return out, pay


class Reference:
    """The brute force over every query's cube (exact: the cube's points are gathered from the layout twin)."""

    def __init__(self, pts, L, K, q, B):
        nq = len(q)
        self.W2 = (2 * K + 1) ** 2
        self.rs, self.re = L.row_ranges(q, K)
        owner, pos = expand(self.rs, self.re)
        qi = owner // self.W2
        d2 = dist2(q[qi], L.pts4[pos, :3], pairwise=True)
        keys = keys_of(d2, L.order[pos])
        self.knn5 = smallest(qi, keys, nq, 5, keys_of(F(3.0e38), SENT))
        inb = keys < keys_of(B, SENT)[qi]
        self.lb_keys, self.lb_pos = smallest(qi[inb], keys[inb], nq, 7, keys_of(B, SENT), pos[inb])
        self.n_in = np.bincount(qi[d2 <= B[qi]], minlength=nq)       # cube points inside the bound


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


# ---- scenes -------------------------------------------------------------------------------------------------------
def surface(seed=21, n=16_000):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-4.0, 4.0, (n, 2))
    z = 0.15 * np.sin(1.3 * xy[:, 0]) * np.cos(0.9 * xy[:, 1]) + rng.normal(0, 0.005, n)
    return np.column_stack([xy, z]).astype(F)


def lattice():
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


@functools.lru_cache(maxsize=None)
def cloud(name):
    if name == "surface":
        return surface()
    if name == "lattice":
        return lattice()
    if name == "sparse":                 # ~2.5 points within 0.5 m of a point: many lists shorter than 5 or 7
        return np.random.default_rng(23).uniform(-4.0, 4.0, (2_500, 3)).astype(F)
    if name == "surface+4096":
        return (surface().astype(np.float64) + [4096.3, -2047.7, 130.1]).astype(F)
    if name == "surface+30000":          # inside arena_plan::kCoordLimit at cell 0.125; eps = 2e-6 |q| ~ 0.08 m
        return (surface().astype(np.float64) + [30000.3, -12000.7, 50.1]).astype(F)
    raise KeyError(name)


CLOUDS = ["surface", "lattice", "sparse", "surface+4096", "surface+30000"]
PATCH = {"lattice": ((-1.0, -1.0, -0.02), (0.95, 0.95, 0.02))}


def on_face(v, inv):
    """the smallest float32 of the cell that contains v, on each coordinate: a point exactly on the cell's lower faces"""
    v = np.asarray(v, F)
    k = np.floor(v.astype(np.float64) * inv)
    x = (k / inv).astype(F)
    for _ in range(8):                   # walk to the first float whose cell is k (float cells need not start at k * cell)
        x = np.where(np.floor(x.astype(np.float64) * inv) < k, np.nextafter(x, F(np.inf)), x)
        x = np.where(np.floor(np.nextafter(x, F(-np.inf)).astype(np.float64) * inv) >= k, np.nextafter(x, F(-np.inf)), x)
    return x


def make_queries(name, pts, L, K, cell, seed):
    rng = np.random.default_rng(seed)
    n = len(pts)
    pick = lambda m: pts[rng.integers(0, n, m)].astype(np.float64)
    kinds = []

    def add(kind, q):
        kinds.append((kind, np.asarray(q, np.float64).astype(F)))

    for s in (0.0, 1e-4, 3e-3, 0.03, 0.15, 0.4):                     # target points plus noise
        add("noise", pick(50) + rng.normal(0, s, (50, 3)))
    for naxes in (1, 2, 3):                                           # on faces, edges, corners
        q = (pick(60) + rng.normal(0, 0.05, (60, 3))).astype(F)
        snapped = on_face(q, L.inv)
        for i in range(len(q)):
            ax = rng.choice(3, naxes, replace=False)
            q[i, ax] = snapped[i, ax]
        add("face", q)
    lo, hi = L.o * cell, (L.o + L.n3) * cell                         # box faces (up to the rounding of the cells)
    for axis in range(3):                                             # outside the box on each side
        srt = np.argsort(pts[:, axis])
        for side, base in ((-1, lo[axis]), (1, hi[axis])):
            near = srt[:max(20, n // 50)] if side < 0 else srt[-max(20, n // 50):]
            for off in (0.5 * cell, K * cell - 0.02 * cell, K * cell + 0.02 * cell):
                q = pts[rng.choice(near, 8)].astype(np.float64)
                q[:, axis] = base + side * off
                add("outside", q)
    ctr = 0.5 * (pts.min(axis=0).astype(np.float64) + pts.max(axis=0))
    d = rng.normal(0, 1, (30, 3))
    add("far", ctr + d / np.linalg.norm(d, axis=1, keepdims=True) * rng.uniform(3.0, 30.0, (30, 1)))
    if name in PATCH:
        a, b = PATCH[name]
        add("patch", rng.uniform(a, b, (80, 3)))
    kind = np.concatenate([[k] * len(q) for k, q in kinds])
    q = np.concatenate([q for _, q in kinds]).astype(F)
    return kind, q


def bounds_for(tree, pts, q, r2):
    """the four bounds B of every query: r2_up (first iteration), min(1.21 d7, r2_up) (seeded), d7 exactly (d2 == B),
    just below d3 (sentinels); d3 / d7 the 3rd / 7th smallest float32 d2 (r2_up where that is farther)"""
    _, nb = tree.query(q.astype(np.float64), k=24)
    d = np.sort(dist2(q[:, None, :], pts[nb], pairwise=True), axis=1)
    d3, d7 = d[:, 2], d[:, 6]
    b_seed = np.minimum(r2, (d7 * LOOK).astype(F))
    b_exact = np.where(d7 <= r2, d7, r2)
    b_below = np.minimum(r2, np.nextafter(d3, F(0)))
    return [np.full(len(q), r2, F), b_seed.astype(F), b_exact.astype(F), b_below.astype(F)]


# ---- the harness --------------------------------------------------------------------------------------------------
def write_input(path, pts, L, K, r2, q, B, rr):
    hdr = np.array([MAGIC, len(pts), len(q), len(rr), K, *L.o, *L.n3, 0], np.int64).astype(np.int32)
    hdr[11] = np.array([r2], F).view(np.int32)[0]
    with open(path, "wb") as f:
        for a in (hdr, np.float64(L.inv), np.ascontiguousarray(pts, F), L.pts4, L.pos_of, L.cell_start,
                  np.ascontiguousarray(q, F), np.ascontiguousarray(B, F), np.ascontiguousarray(rr, np.int32)):
            f.write(np.asarray(a).tobytes())


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
    from dcreg_b200.build import _nvcc
    from test_host_la import device_program_flags
    exe = tmp_path_factory.mktemp("corr_search") / "test_corr_search"
    subprocess.run([_nvcc()] + device_program_flags() + ["-o", str(exe), HARNESS], check=True, capture_output=True, text=True)
    return exe


def first_bad(mask):
    return int(np.flatnonzero(mask)[0]) if mask.any() else -1


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
    from dcreg_b200.build import _nvcc
    from test_host_la import device_program_flags
    try:
        nvcc = _nvcc()
    except RuntimeError:
        pytest.skip("nvcc not available")
    res = subprocess.run([nvcc] + device_program_flags() + ["-o", str(tmp_path / "h"), HARNESS], capture_output=True, text=True)
    assert res.returncode == 0, res.stderr


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
