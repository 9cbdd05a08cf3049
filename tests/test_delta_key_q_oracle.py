"""The NumPy delta_key_q (oracle/delta_key_q.py) against scipy's rotations: (c^-1 i d i^-1 c)^-1, on random and
near-identity extrinsics and rotations."""
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle.delta_key_q import conjugate, delta_key_q, quat_product


def _same_rotation(q, r):
    q = np.asarray(q) / np.linalg.norm(q)
    r = r.as_quat()
    return min(np.max(np.abs(q - r)), np.max(np.abs(q + r)))


@pytest.mark.parametrize("scale", [np.pi, 1e-3, 1e-8])
def test_delta_key_q_matches_scipy(scale):
    rng = np.random.default_rng(7)
    for _ in range(200):
        c, i, d = (Rotation.from_rotvec(rng.normal(size=3) * s)
                   for s in (scale, scale, np.pi if scale == np.pi else scale))
        want = (c.inv() * i * d * i.inv() * c).inv()
        got = delta_key_q(c.as_quat(), i.as_quat(), d.as_quat())
        assert _same_rotation(got, want) <= 1e-15


def test_identity_extrinsics_give_the_inverse_rotation():
    rng = np.random.default_rng(3)
    e = np.array([0.0, 0.0, 0.0, 1.0])
    for _ in range(50):
        d = Rotation.from_rotvec(rng.normal(size=3)).as_quat()
        assert np.array_equal(delta_key_q(e, e, d), conjugate(d))


def test_quat_product_order():
    """Eigen's quat_product sums w*b + a*w first: a case where that order differs from another in the last bit"""
    a = np.array([0.1, 0.2, 0.3, 0.9])
    b = np.array([0.3, -0.7, 0.2, 0.6])
    p = quat_product(a, b)
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    assert p[1] == aw * by + ay * bw + az * bx - ax * bz
    assert p[3] == aw * bw - ax * bx - ay * by - az * bz
