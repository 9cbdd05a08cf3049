"""The F-matrix RANSAC oracle (oracle/fm_oracle.py: OpenCV's findFundamentalMat(FM_RANSAC) restated for
opencv_image.cpp:121-129) PINNED against the reference's real dependency, cv2.findFundamentalMat: inlier masks equal
scene by scene (the sample schedule of cv::RNG is restated, so the runs agree iteration for iteration), cv::solveCubic
root for root, and the committed golden vectors (tests/golden/fm_golden.npz, made by make_fm_golden.py)."""
import os

import numpy as np
import pytest

from oracle import fm_oracle as fo
from synthetic import synth

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fm_golden.npz")
SCENES = [(150, 0.1), (300, 0.3), (400, 0.5), (60, 0.2), (15, 0.1), (20, 0.0), (200, 0.7)]


def test_solve_cubic_matches_cv2():
    cv2 = pytest.importorskip("cv2")
    r = np.random.default_rng(0)
    for i in range(600):
        c = r.normal(size=4)
        if i % 10 == 0:
            c[0] = 0
        if i % 50 == 0:
            c[1] = 0
        n, roots = cv2.solveCubic(c.reshape(1, 4))
        mine = fo.solve_cubic(c)
        assert n == len(mine)
        assert np.allclose(roots.ravel()[:n], mine, rtol=1e-12, atol=1e-12)


def test_rng_is_opencv_mwc():
    """cv::RNG(-1): first values of the multiply-with-carry generator, computed independently with Python integers."""
    rng = fo.CvRNG()
    s = 0xFFFFFFFFFFFFFFFF
    for _ in range(5):
        s = ((s & 0xFFFFFFFF) * 4164903690 + (s >> 32)) & 0xFFFFFFFFFFFFFFFF
        assert rng.next() == (s & 0xFFFFFFFF)
    assert fo.CvRNG(0).state == 0xFFFFFFFF
    sch = fo.sample_schedule(*synth.make_fm_matches(n=50), 20)
    assert sch.shape == (20, 7) and all(len(set(row)) == 7 for row in sch) and sch.min() >= 0 and sch.max() < 50


@pytest.mark.parametrize("null_space", [fo.null_space_svd, fo.null_space_householder])
def test_ransac_masks_equal_cv2(null_space):
    cv2 = pytest.importorskip("cv2")
    for seed in range(6):
        for n, of in SCENES:
            p, q = synth.make_fm_matches(seed, n, of, planar=(seed % 7 == 3))
            _, mask = cv2.findFundamentalMat(p, q, cv2.FM_RANSAC, 1.0, 0.99)
            m, F, info = fo.find_fundamental_mask(p, q, null_space=null_space, return_info=True)
            assert np.array_equal(mask.ravel(), m), (seed, n, of, info)
            assert info["method"] == "ransac"


def test_lmeds_branch_below_15_matches():
    """8 <= n < 15: cv::findFundamentalMat(FM_RANSAC) silently runs LMedS.  n == 14 is pinned against cv2; for n <= 13 the
    median element (index n / 2 <= 6) is one of the 7 matches every model fits exactly, i.e. rounding noise decides inside
    OpenCV itself, so only the structure of the answer is checked there."""
    cv2 = pytest.importorskip("cv2")
    for seed in range(12):
        p, q = synth.make_fm_matches(2000 + seed, 14, 0.15 if seed % 2 else 0.3)
        _, mask = cv2.findFundamentalMat(p, q, cv2.FM_RANSAC, 1.0, 0.99)
        _, mask_l = cv2.findFundamentalMat(p, q, cv2.FM_LMEDS, 1.0, 0.99)
        assert np.array_equal(mask, mask_l)
        m, _, info = fo.find_fundamental_mask(p, q, return_info=True)
        assert info["method"] == "lmeds" and info["iterations"] == 300
        assert np.array_equal(mask.ravel(), m)
    p, q = synth.make_fm_matches(5, 10, 0.1)
    m, F, info = fo.find_fundamental_mask(p, q, return_info=True)
    assert info["method"] == "lmeds" and F is not None and m.sum() >= 7


def test_small_inputs():
    p, q = synth.make_fm_matches(1, 7, 0.0)
    m, F = fo.find_fundamental_mask(p, q)
    assert m.tolist() == [1] * 7 and F is not None
    m, F = fo.find_fundamental_mask(p[:5], q[:5])
    assert m.tolist() == [0] * 5 and F is None


def test_injected_schedule_is_followed():
    p, q = synth.make_fm_matches(3, 120, 0.3)
    own = fo.sample_schedule(p, q, 1000)
    a = fo.find_fundamental_mask(p, q, schedule=own, return_info=True)
    b = fo.find_fundamental_mask(p, q, return_info=True)
    assert np.array_equal(a[0], b[0]) and a[2] == b[2]
    r = np.random.default_rng(0)
    sch = np.stack([r.choice(120, 7, replace=False) for _ in range(1000)]).astype(np.int32)
    c = fo.find_fundamental_mask(p, q, schedule=sch, return_info=True)
    assert c[0][36:].mean() > 0.75 and c[0][:36].mean() < 0.1 and c[2]["iterations"] < 1000          # the inliers are found whatever the schedule


def test_golden_vectors():
    g = np.load(GOLD)
    for i in range(int(g["count"])):
        p, q = g[f"p{i}"], g[f"q{i}"]
        m = fo.find_fundamental_mask(p, q)[0]
        assert np.array_equal(m, g[f"cv_mask{i}"])


def test_library_sample_schedule_equals_the_oracle():
    """Host side of pvio_b200_find_fundamental_mask (no GPU): the subsets the library draws are the oracle's, i.e. OpenCV's
    (the oracle's RANSAC masks equal cv2's iteration for iteration only if the schedule does)."""
    from pvio_b200 import _lib
    lib = _lib.load()
    fn = lib.pvio_b200_fm_sample_schedule
    for seed, n in [(1, 15), (2, 60), (3, 400), (4, 9)]:
        p, q = synth.make_fm_matches(seed, n, 0.2)
        out = np.zeros((300, 7), dtype=np.int32)
        got = fn(n, _lib.ptr(p), _lib.ptr(q), 300, _lib.ptr(out))
        assert got == 300
        assert np.array_equal(out, fo.sample_schedule(p, q, 300, 10000 if n >= 15 else 1000))
    assert fn(5, _lib.ptr(p), _lib.ptr(q), 10, _lib.ptr(out)) < 0
