"""The neighbour searches on the sparse row index (dcreg_set_target_sparse) against the same searches on the dense grid
of the same points, and against the float32 brute force.

tools/test_sparse_search.cu takes tools/test_corr_search.cu's input (the points, their dense layout and the queries of
tests/test_gpu_corr_search.py, inside and outside the box, at ring counts 1-4), builds the sparse index with the
production build (build_sparse_arena's kernels on a one-cloud arena, the builder of every sparse index) and runs
knn_search, knn_search_lb, knn_warp_search (with and, at one ring, without the loop's row table) and knn_row_range on
both.  Contracts:
  * the sparse build's points and positions are byte-identical to the dense layout;
  * every search returns bit-identical keys, positions and lb on both (row pairs: lb, and [s, e) unless it is empty,
    which the sparse index reports as [0, 0) where the dense grid has [cs, cs));
  * the brute-force contracts of tests/test_gpu_corr_search.py hold on the sparse results: knn_search's five smallest
    keys of the cube, knn_search_lb's seven smallest inside the bound with their positions, knn_warp_search's
    got == (cube points inside the bound <= 64) and, when got, knn_search_lb's list.
"""
import subprocess

import numpy as np
import pytest

from harness import tool_program
from search_harness import (CELLS, CLOUDS, RADIUS, WARP_CAP, Layout, Reference, bounds_for, cloud, first_bad,
                            make_queries, r2_up, rings_of, write_input)


def read_output(path, nq, nrr):
    buf = open(path, "rb").read()
    at = 0

    def take(dtype, count, shape=None):
        nonlocal at
        a = np.frombuffer(buf, dtype=dtype, count=count, offset=at)
        at += a.nbytes
        return a.reshape(shape) if shape else a

    check = take(np.int32, 3)
    sides = []
    for _ in range(2):
        o = {"knn5": take(np.uint64, nq * 5, (nq, 5)), "lb_keys": take(np.uint64, nq * 7, (nq, 7)),
             "lb_pos": take(np.int32, nq * 7, (nq, 7)), "lb": take(np.uint32, nq)}
        for w in ("warp", "pre"):
            o[w + "_got"] = take(np.int32, nq)
            o[w + "_keys"] = take(np.uint64, nq * 7, (nq, 7))
            o[w + "_pos"] = take(np.int32, nq * 7, (nq, 7))
            o[w + "_lb"] = take(np.uint32, nq)
        o["rr"] = take(np.int32, nrr * 3, (nrr, 3))
        sides.append(o)
    assert at == len(buf)
    return check, sides[0], sides[1]


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return tool_program(tmp_path_factory.mktemp("sparse_search"), "test_sparse_search.cu", compiler="device",
                        skip_missing=False)


@pytest.mark.gpu
@pytest.mark.parametrize("cell", CELLS)
@pytest.mark.parametrize("name", CLOUDS)
def test_sparse_searches_equal_dense(harness, tmp_path, name, cell):
    from scipy.spatial import cKDTree
    pts = cloud(name)
    L = Layout(pts, cell)
    K = rings_of(RADIUS, cell)
    r2 = r2_up(RADIUS)
    kind0, q0 = make_queries(name, pts, L, K, cell, seed=100 + CLOUDS.index(name) * 10 + CELLS.index(cell))
    tree = cKDTree(pts.astype(np.float64))
    Bs = bounds_for(tree, pts, q0, r2)
    perm = np.random.default_rng(98).permutation(4 * len(q0))
    q = np.tile(q0, (4, 1))[perm]
    kind = np.tile(kind0, 4)[perm]
    B = np.concatenate(Bs)[perm]
    nq = len(q)
    W2 = (2 * K + 1) ** 2
    rq = np.flatnonzero(np.arange(nq) % 3 == 0)
    rr = np.stack([np.repeat(rq, W2), np.tile(np.arange(W2), len(rq))], axis=1)

    inp, outp = tmp_path / "in.bin", tmp_path / "out.bin"
    write_input(inp, pts, L, K, r2, q, B, rr)
    res = subprocess.run([str(harness), str(inp), str(outp)], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    check, dense, sparse = read_output(outp, nq, len(rr))
    assert check[0] == 1 and check[1] == 1, "sparse build: pts / pos_of differ from the dense layout"
    assert 0 < check[2] <= 18 * len(np.unique(L.lin))

    where = lambda m: f"query {first_bad(m)} ({kind[first_bad(m)]}, q={q[first_bad(m)].tolist()})"
    for f in dense:
        if f == "rr":
            # an empty range has no positions: the dense grid gives [cs, cs), the sparse index [0, 0) where a lookup
            # misses; a non-empty range and every lb must be identical
            d, s = dense[f], sparse[f]
            d_empty, s_empty = d[:, 0] >= d[:, 1], s[:, 0] >= s[:, 1]
            bad = (d[:, 2] != s[:, 2]) | (d_empty != s_empty) | (~d_empty & ((d[:, 0] != s[:, 0]) | (d[:, 1] != s[:, 1])))
            assert not bad.any(), f"knn_row_range: {int(bad.sum())} pairs differ, first pair {first_bad(bad)}"
            assert (~d_empty).any()
            continue
        if f.startswith("pre") and K != 1:
            continue
        a, b = dense[f], sparse[f]
        bad = (a != b).reshape(nq, -1).any(axis=1)
        assert not bad.any(), f"{f}: {int(bad.sum())} queries differ between the dense grid and the sparse index, first {where(bad)}"

    ref = Reference(pts, L, K, q, B)
    assert np.array_equal(sparse["knn5"], ref.knn5)
    assert np.array_equal(sparse["lb_keys"], ref.lb_keys) and np.array_equal(sparse["lb_pos"], ref.lb_pos)
    got = sparse["warp_got"].astype(bool)
    assert np.array_equal(got, ref.n_in <= WARP_CAP)
    assert np.array_equal(sparse["warp_keys"][got], ref.lb_keys[got])
    assert np.array_equal(sparse["warp_pos"][got], ref.lb_pos[got])
    c = L.local_cell(q)
    outside = ((c < 0) | (c >= L.n3)).any(axis=1)
    assert outside.any() and (~outside).any()                  # queries inside and outside the box


def test_sparse_harness_compiles_for_sm90a(tmp_path):
    """tools/test_sparse_search.cu builds with the library's flags (no GPU needed to compile)."""
    tool_program(tmp_path, "test_sparse_search.cu", compiler="device")
