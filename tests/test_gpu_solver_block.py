"""The loop kernel's solver block (single folded runs: block 0 sums the rows as they land and solves) against the ticket
path (DCREG_NO_SOLVER_BLOCK=1): both add the same rows in the same order, so sums, counts and poses must agree bit for
bit in every iteration."""
import os

import numpy as np
import pytest

from dcreg_b200.scenes import g2_initial_pose, make_cylinder
from harness import ctx  # noqa: F401

pytestmark = pytest.mark.gpu


def _run(ctx, prm, T0, **env):
    for k, v in env.items():
        os.environ[k] = v
    try:
        res = ctx.icp_run(prm, T0)
        blocks, solve = ctx.iteration_timeline(prm, T0, 2)
    finally:
        for k in env:
            del os.environ[k]
    return res, len(blocks), int(solve[14])


def _records(res):
    return [(L.n_effective, L.n_corr_pt, np.array(L.H27).tobytes(), np.array(L.dx).tobytes(), np.array(L.T).tobytes())
            for L in res.logs]


@pytest.mark.parametrize("n", [100_000, 12_347])          # C2, and a ragged size cut into 32-slot tiles
def test_solver_block_equals_ticket_path_bit_for_bit(ctx, n):
    from dcreg_b200 import default_params
    pts = make_cylinder(n, seed=42)
    T0 = g2_initial_pose()
    prm = default_params(search_radius=1.0, max_iterations=50, fixed_iterations=1, kappa_target=10.0)
    ctx.set_target(pts, 1.0)
    ctx.set_source(pts)
    new, nb_new, mark_new = _run(ctx, prm, T0)
    old, nb_old, mark_old = _run(ctx, prm, T0, DCREG_NO_SOLVER_BLOCK="1")
    assert (mark_new, mark_old) == (1, 0)                  # the solver block ran (timeline marker), then the ticket path
    assert nb_new == nb_old + 1
    assert new.iterations == old.iterations == 50
    assert new.status == old.status == 0
    assert np.array(new.T).tobytes() == np.array(old.T).tobytes()
    assert _records(new) == _records(old)
