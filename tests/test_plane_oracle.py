"""CPU tests of the plane RANSAC oracle (oracle/plane_oracle.py): its 3-draw sample schedule against the one libstdc++
draws (tests/golden/lotbox3_golden.npz, written by tests/golden/make_lotbox3_golden.py), Eigen's stableNormalize on
vectors a plain normalisation gets wrong, the recovery of a known plane among outliers, the degenerate-sample quirk of
PlaneSolver, and the budget of Ransac::solve (ransac.h:87-91)."""
import math
import os

import numpy as np

from oracle import plane_oracle as po
from oracle.twoview_oracle import lotbox_schedule

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lotbox3_golden.npz")


def test_schedule_matches_libstdcxx():
    g = np.load(GOLDEN)
    assert int(g["count"]) >= 7
    for i in range(int(g["count"])):
        n, seed, dof = (int(x) for x in g[f"case{i}"])
        assert seed == 0 and dof == 3
        ref = g[f"s{i}"]
        np.testing.assert_array_equal(lotbox_schedule(n, seed, dof, len(ref)), ref, err_msg=f"n={n}")


def _direction(v):
    """v / |v| without overflow or underflow: scaled by an exact power of two first"""
    e = max(math.frexp(float(x))[1] for x in v if x != 0)
    u = np.array([math.ldexp(float(x), -e) for x in v])
    return u / np.linalg.norm(u)


def test_stable_normalize():
    np.testing.assert_array_equal(po.stable_normalize([0.0, 0.0, 0.0]), np.zeros(3))
    for v in ([1e-300, 2e-300, 0.0], [3e-320, -4e-320, 0.0], [1e300, 1e300, -1e300], [1e308, 1e-308, 0.0],
              [0.0, 0.0, -5.0], [3.0, 4.0, 12.0], [-2e-170, 1e-170, 2e-170]):
        got = po.stable_normalize(v)
        np.testing.assert_allclose(got, _direction(v), rtol=0, atol=4e-16, err_msg=str(v))
        with np.errstate(all="ignore"):
            naive = np.asarray(v) / math.sqrt(sum(x * x for x in v)) if sum(x * x for x in v) > 0 else np.zeros(3)
        m = max(abs(x) for x in v)
        if m < 1e-150 or m > 1e150:
            assert not np.allclose(naive, got)        # the crafted cases are the ones the plain formula gets wrong


def _plane_points(rng, n_on, n_off, normal, d, noise):
    normal = normal / np.linalg.norm(normal)
    b1 = np.cross(normal, [1.0, 0.0, 0.0] if abs(normal[0]) < 0.9 else [0.0, 1.0, 0.0])
    b1 /= np.linalg.norm(b1)
    b2 = np.cross(normal, b1)
    uv = rng.uniform(-3, 3, (n_on, 2))
    on = d * normal + uv[:, :1] * b1 + uv[:, 1:] * b2 + rng.normal(0, noise, (n_on, 1)) * normal
    off = rng.uniform(-3, 3, (n_off, 3)) + 2.0 * normal
    pts = np.vstack([on, off])
    perm = rng.permutation(len(pts))
    return pts[perm], perm < n_on, normal


def test_recovers_known_plane_with_outliers():
    rng = np.random.default_rng(5)
    for mode in (po.EXTRACT, po.REFIT):
        pts, truth_on, normal = _plane_points(rng, 180, 120, np.array([0.3, -0.2, 1.0]), 1.7, 0.004)
        r = po.plane_ransac(pts, mode)
        assert r["status"] == po.ACCEPTED
        n, d = r["plane"][:3], r["plane"][3]
        assert np.degrees(np.arccos(min(1.0, abs(n @ normal)))) < 0.5
        assert d >= 0 and abs(d - 1.7) < 0.01
        assert (r["mask"] & truth_on).sum() >= 0.95 * truth_on.sum()
        assert (np.abs(pts[r["mask"]] @ normal - 1.7) < 0.05).all()     # an outlier in the mask lies near the plane
        np.testing.assert_array_equal(r["plane"][4:], po.centroid(pts, r["mask"]))
        w, V = np.linalg.eigh(po.covariance(pts, r["mask"], r["plane"][4:]))
        assert abs(abs(V[:, 0] @ n) - 1) < 1e-12


def test_degenerate_sample_counts_every_point():
    p = np.array([0.4, -1.0, 2.5])
    n, d = po.plane_solve(p, p, p)
    np.testing.assert_array_equal(n, np.zeros(3))
    assert d == 0.0
    rng = np.random.default_rng(1)
    pts = rng.normal(0, 1, (40, 3))
    assert po.inlier_mask(pts, n, d, 0.03).all()
    # a sample with a repeated point (here iteration 1 shares one with iteration 2) wins with every point as an inlier
    sched = lotbox_schedule(40, 0, 3, 1000)
    dup = pts.copy()
    dup[sched[2]] = pts[sched[2][0]]
    r = po.ransac(dup, 0.03)
    b = r["best_it"]
    assert 0 <= b <= 2 and r["inliers"] == 40 and r["counts"][b] == 40 and r["mask"].all()
    assert len({tuple(x) for x in dup[sched[b]]}) < 3
    assert r["iterations"] == b + 1                   # ratio 1: the budget drops to 0 after the winning iteration


def test_budget_shrinks_as_reference():
    rng = np.random.default_rng(9)
    for n_on, n_off in ((60, 40), (100, 20), (40, 200)):
        pts, _, _ = _plane_points(rng, n_on, n_off, np.array([0.0, 0.0, 1.0]), 0.5, 0.002)
        r = po.ransac(pts, 0.03)
        n = len(pts)
        K = math.log(max(1 - po.CONFIDENCE, 1e-5))
        iter_max, best = po.MAX_ITERATION, 0
        for it, c in enumerate(r["counts"]):
            assert it < iter_max
            if c > best:
                best = c
                N = K / math.log(1 - math.pow(c / n, 5)) if c < n else 0.0
                if N < iter_max:
                    iter_max = int(math.ceil(N))
        assert r["iterations"] == len(r["counts"]) == min(iter_max, po.MAX_ITERATION)
        assert r["iterations"] < po.MAX_ITERATION or best / n < 0.3


def test_baseline():
    p = [np.array([0.0, 0, 0]), np.array([0.3, 0, 0]), np.array([0.3, 0.4, 0])]
    assert po.compute_baseline(p) == 0.3 + 0.4
    assert po.enough_baseline(p, 0.1)                  # 0.7 > 0.5
    assert not po.enough_baseline(p[:2], 1.0)          # 0.3, 0.3 * 1.0 < 0.5
    assert po.enough_baseline(p[:2], 2.0)              # 0.3 * 2 > 0.5 with inverse depth below 5
    assert not po.enough_baseline(p[:2], 6.0)
