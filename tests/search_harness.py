"""The neighbour-search reference that tests/test_gpu_corr_search.py and tests/test_gpu_sparse_search.py share: the
layout twin of the dense grid, the float32 brute force over every query's cube of cells, the scenes and queries, and the
input file of tools/test_corr_search.cu (which tools/test_sparse_search.cu reads too)."""
import functools

import numpy as np

from harness import dist2, ties_lattice

F = np.float32
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


# ---- scenes -------------------------------------------------------------------------------------------------------
def surface(seed=21, n=16_000):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(-4.0, 4.0, (n, 2))
    z = 0.15 * np.sin(1.3 * xy[:, 0]) * np.cos(0.9 * xy[:, 1]) + rng.normal(0, 0.005, n)
    return np.column_stack([xy, z]).astype(F)


@functools.lru_cache(maxsize=None)
def cloud(name):
    if name == "surface":
        return surface()
    if name == "lattice":
        return ties_lattice()
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


# ---- the input of tools/test_corr_search.cu -----------------------------------------------------------------------
def write_input(path, pts, L, K, r2, q, B, rr):
    hdr = np.array([MAGIC, len(pts), len(q), len(rr), K, *L.o, *L.n3, 0], np.int64).astype(np.int32)
    hdr[11] = np.array([r2], F).view(np.int32)[0]
    with open(path, "wb") as f:
        for a in (hdr, np.float64(L.inv), np.ascontiguousarray(pts, F), L.pts4, L.pos_of, L.cell_start,
                  np.ascontiguousarray(q, F), np.ascontiguousarray(B, F), np.ascontiguousarray(rr, np.int32)):
            f.write(np.asarray(a).tobytes())


def first_bad(mask):
    return int(np.flatnonzero(mask)[0]) if mask.any() else -1
