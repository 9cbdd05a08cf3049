"""The CPU oracle of init_sfm's two-view step (oracle/twoview_oracle.py), checked against known answers: the LotBox
schedule against the one libstdc++ draws (tests/golden/lotbox_golden.npz), the minimal solvers on noise-free
problems, the decompositions against OpenCV's, the serial RANSAC on noisy scenes with outliers, the selection rule on
hand-built counts; and the ctypes record of pvio_b200_batch_two_view against the header (no GPU needed)."""
import ctypes as C
import math
import os

import numpy as np
import pytest

from oracle import twoview_oracle as tv
from pvio_b200 import _lib
from synthetic import synth

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lotbox_golden.npz")


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def _rotation(rng, scale=0.3):
    return synth._rodrigues(rng.normal(0, scale, 3))


def test_schedule_equals_libstdcxx():
    g = np.load(GOLDEN)
    assert int(g["count"]) >= 24
    for i in range(int(g["count"])):
        n, seed, dof = (int(v) for v in g[f"case{i}"])
        ref = g[f"s{i}"]
        got = tv.lotbox_schedule(n, seed, dof, len(ref))
        np.testing.assert_array_equal(got, ref, err_msg=f"n={n} seed={seed} dof={dof}")


def test_schedule_rows_are_distinct_and_in_range():
    s = tv.lotbox_schedule(6, 648, 5, 200)
    assert s.min() >= 0 and s.max() < 6
    assert all(len(set(r)) == 5 for r in s)


def test_five_point_solver_finds_the_true_essential_matrix():
    rng = np.random.default_rng(11)
    found = 0
    trials = 220
    for _ in range(trials):
        R = _rotation(rng)
        t = rng.normal(0, 1, 3)
        X = np.c_[rng.uniform(-2, 2, (5, 2)), rng.uniform(2, 8, 5)]
        Xj = X @ R.T + t
        p1, p2 = X[:, :2] / X[:, 2:], Xj[:, :2] / Xj[:, 2:]
        Et = _skew(t) @ R
        Et /= np.linalg.norm(Et)
        models, _ = tv.essential_5pt(p1, p2)
        assert 1 <= len(models) <= 10
        errs = [min(np.abs(E / np.linalg.norm(E) - Et).max(), np.abs(E / np.linalg.norm(E) + Et).max()) for E in models]
        found += min(errs) < 1e-8
    assert found >= 200, f"true E among the solutions of {found} / {trials} problems"


def test_four_point_solver_reproduces_the_plane_homography():
    rng = np.random.default_rng(12)
    for _ in range(50):
        R, t = _rotation(rng, 0.2), rng.normal(0, 0.5, 3)
        nrm = rng.normal(0, 0.2, 3) + np.array([0, 0, 1.0])
        nrm /= np.linalg.norm(nrm)
        d = rng.uniform(3, 8)
        H = R + np.outer(t, nrm) / d
        xy = rng.uniform(-0.5, 0.5, (4, 2))
        X = np.c_[xy, np.ones(4)]
        X *= (d / (X @ nrm))[:, None]                         # on the plane n . X = d
        Xj = X @ R.T + t
        p1, p2 = X[:, :2] / X[:, 2:], Xj[:, :2] / Xj[:, 2:]
        G = tv.homography_4pt(p1, p2)
        assert np.abs(G / G[2, 2] - H / H[2, 2]).max() < 1e-9


def test_decompose_homography_matches_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(13)
    for _ in range(40):
        R, t = _rotation(rng, 0.2), rng.normal(0, 0.5, 3)
        nrm = rng.normal(0, 0.3, 3) + np.array([0, 0, 1.0])
        nrm /= np.linalg.norm(nrm)
        H = (R + np.outer(t, nrm) / rng.uniform(3, 8)) * rng.uniform(0.5, 2.0)
        ok, R1, R2, T1, T2 = tv.decompose_homography(H)
        assert ok
        _, Rs, Ts, _ = cv2.decomposeHomographyMat(H, np.eye(3))
        for Ri, Ti in ((R1, T1), (R2, T2)):
            # a match in OpenCV's four solutions: the same rotation, the translation up to the sign of (t, n)
            hit = [k for k in range(len(Rs)) if np.abs(Rs[k] - Ri).max() < 1e-9]
            assert hit, "rotation not among OpenCV's"
            tn = tv.normalized(Ti)
            assert any(min(np.abs(tv.normalized(Ts[k].ravel()) - tn).max(),
                           np.abs(tv.normalized(Ts[k].ravel()) + tn).max()) < 1e-9 for k in hit)


def test_decompose_homography_flags_a_pure_rotation():
    R = _rotation(np.random.default_rng(14), 0.2)
    ok, R1, R2, T1, T2 = tv.decompose_homography(2.5 * R)
    assert not ok
    assert np.abs(R1 - R).max() < 1e-12 and np.all(T1 == 0)


def test_decompose_essential_matches_opencv():
    cv2 = pytest.importorskip("cv2")
    rng = np.random.default_rng(15)
    for _ in range(40):
        R, t = _rotation(rng), rng.normal(0, 1, 3)
        E = _skew(t) @ R
        R1, R2, T = tv.decompose_essential(E)
        c1, c2, ct = cv2.decomposeEssentialMat(E)
        assert (np.abs(R1 - c1).max() < 1e-9 and np.abs(R2 - c2).max() < 1e-9) or \
               (np.abs(R1 - c2).max() < 1e-9 and np.abs(R2 - c1).max() < 1e-9)
        assert min(np.abs(T - ct.ravel()).max(), np.abs(T + ct.ravel()).max()) < 1e-9
        assert any(np.abs(Rc - R).max() < 1e-9 for Rc in (R1, R2))


def _rot_angle(A, B):
    return math.acos(max(-1.0, min(1.0, (np.trace(A.T @ B) - 1) / 2)))


@pytest.mark.parametrize("outliers", [0.0, 0.25, 0.5])
def test_serial_ransac_recovers_the_relative_pose(outliers):
    s = synth.make_two_view(seed=20 + int(100 * outliers), n=300, outlier_frac=outliers, noise_px=0.5)
    o = tv.two_view(s["p1"], s["p2"], s["fx"], s["fy"])
    assert o["status"] == tv.STATUS_OK
    assert o["candidate"] >= 4                                  # a general scene: an essential-matrix candidate
    assert _rot_angle(o["R"], s["R"]) < math.radians(0.5)
    t = s["t"] / np.linalg.norm(s["t"])
    assert math.acos(min(1.0, float(o["T"] @ t))) < math.radians(3.0)
    no = int(outliers * 300)
    assert not o["e"]["mask"][:no].any() or o["e"]["mask"][:no].mean() < 0.05
    assert o["e"]["mask"][no:].mean() > 0.75                      # 0.5 px noise against a 0.7 px threshold


def test_early_stop_follows_the_fifth_power():
    """Both RANSACs shrink the budget with pow(ratio, 5): the homography's 4 samples included."""
    s = synth.make_two_view(seed=30, n=200, outlier_frac=0.2, kind="plane")
    thr_h, _ = tv.thresholds(s["fx"])
    r = tv.ransac("H", s["p1"], s["p2"], thr_h)
    K = math.log(1e-3)
    N5 = math.ceil(K / math.log(1 - (r["inliers"] / 200) ** 5))
    N4 = math.ceil(K / math.log(1 - (r["inliers"] / 200) ** 4))
    assert N4 != N5
    assert r["iterations"] == max(min(1000, N5), r["best_it"] + 1)
    # the run is the serial loop: no iteration after the stop was evaluated
    assert len(r["counts"]) == r["iterations"]


def test_ransac_stops_after_the_iteration_that_makes_every_match_an_inlier():
    s = synth.make_two_view(seed=31, n=60, noise_px=0.0, kind="plane")
    thr_h, _ = tv.thresholds(s["fx"])
    r = tv.ransac("H", s["p1"], s["p2"], thr_h)
    assert r["inliers"] == 60 and r["iterations"] == r["best_it"] + 1


def test_selection_rule():
    # a lower mean score wins among candidates above the threshold
    assert tv.select_candidate([15, 25, 24, 0, 0, 0, 0, 0], [0.01, 0.3, 0.2, 0, 0, 0, 0, 0], 20) == 2
    # the score test compares against the current best even while the best's count is below the threshold: a
    # candidate above the threshold with a worse score than a below-threshold best only wins on count
    assert tv.select_candidate([15, 25], [0.01, 0.5], 20) == 1
    assert tv.select_candidate([15, 25, 30], [0.01, 0.5, 0.6], 20) == 2
    # ... and more points still win over an above-threshold best with a better score
    assert tv.select_candidate([25, 30], [0.1, 0.6], 20) == 1
    # below the threshold only the count matters
    assert tv.select_candidate([5, 8, 7], [0.0, 0.9, 0.1], 20) == 1
    # ties keep the earlier candidate
    assert tv.select_candidate([10, 10], [0.2, 0.2], 5) == 0


def test_gates_in_init_sfm_order():
    s = synth.make_two_view(seed=32, n=40)
    assert tv.two_view(s["p1"], s["p2"], s["fx"], s["fy"])["status"] == tv.STATUS_FEW_MATCHES
    s = synth.make_two_view(seed=33, n=100, kind="small")
    o = tv.two_view(s["p1"], s["p2"], s["fx"], s["fy"])
    assert o["parallax"] < 10 and o["status"] == tv.STATUS_LOW_PARALLAX
    s = synth.make_two_view(seed=34, n=100, kind="rotation", noise_px=0.0)
    assert tv.two_view(s["p1"], s["p2"], s["fx"], s["fy"])["status"] == tv.STATUS_PURE_ROTATION


def test_two_view_record_matches_header():
    R = _lib.CTwoView
    assert C.sizeof(R) == 184                                    # include/pvio_b200.h: 184 bytes on LP64
    offsets = {"n_matches": 0, "seed": 4, "p1": 8, "p2": 16, "fx": 24, "fy": 32, "min_matches": 40,
               "min_triangulation": 44, "min_parallax": 48, "confidence": 56, "max_iteration": 64, "info": 72,
               "parallax": 80, "H": 88, "E": 96, "R": 104, "T": 112, "h_mask": 120, "e_mask": 128, "points": 136,
               "point_status": 144, "h_schedule": 152, "e_schedule": 160, "h_counts": 168, "e_counts": 176}
    assert {k: getattr(R, k).offset for k in offsets} == offsets
    assert "pvio_b200_batch_two_view" in _lib.EXPORTS
