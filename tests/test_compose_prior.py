"""compose_prior: the NumPy twin of the frame advance of dcreg_icp_run_sequences.  Its bits are pinned by the documented
order of operations (((a0 b0 + a1 b1) + a2 b2), then + t, one rounding each), evaluated here with plain Python floats;
the GPU tests check the device against the same function byte for byte."""
import numpy as np

from dcreg_b200.api import compose_prior
from dcreg_b200.scenes import pose6d_to_matrix


def scalar_compose(T, D):
    out = [[0.0] * 4 for _ in range(4)]
    for r in range(3):
        for c in range(4):
            a = float(T[r][0]) * float(D[0][c])
            b = float(T[r][1]) * float(D[1][c])
            e = float(T[r][2]) * float(D[2][c])
            s = (a + b) + e
            if c == 3:
                s = s + float(T[r][3])
            out[r][c] = s
    out[3][3] = 1.0
    return np.array(out)


def poses(n, seed):
    rng = np.random.default_rng(seed)
    return [pose6d_to_matrix(*rng.uniform(-30, 30, 3), *rng.uniform(-np.pi, np.pi, 3)) for _ in range(n)]


def test_bits_follow_the_documented_order():
    for T, D in zip(poses(200, 1), poses(200, 2)):
        assert compose_prior(T, D).tobytes() == scalar_compose(T, D).tobytes()


def test_is_the_product_up_to_rounding():
    for T, D in zip(poses(50, 3), poses(50, 4)):
        assert np.allclose(compose_prior(T, D), T @ D, rtol=0, atol=1e-12)


def test_batched_and_identity():
    Ts, Ds = np.array(poses(8, 5)), np.array(poses(8, 6))
    out = compose_prior(Ts, Ds)
    assert out.shape == (8, 4, 4)
    for k in range(8):
        assert out[k].tobytes() == compose_prior(Ts[k], Ds[k]).tobytes()
    for T in Ts:                                     # a rotation times the identity keeps its entries
        assert np.array_equal(compose_prior(T, np.eye(4)), T)
