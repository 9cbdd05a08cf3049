"""The feature tracker's host-side pieces without a device: the restated std::sort (pvio_b200/csrc/introsort.cuh)
against libstdc++'s own, the CPU statement of the per-frame step (oracle/feature_oracle.py) on a short synthetic
sequence, and the wrapper's rejections of the header's slot rules."""
import math

import numpy as np
import pytest

from oracle import feature_oracle as fo
from pvio_b200 import feature_track as ft

cv2 = pytest.importorskip("cv2")


def test_restated_sort_equals_std_sort():
    rng = np.random.default_rng(11)
    differs_from_stable = 0
    for t in range(3000):
        n = int(rng.integers(0, 2001)) if t % 3 else int(rng.integers(0, 64))
        length = rng.integers(2, int(rng.integers(3, 61)), n).astype(np.int32)
        idx = np.arange(n, dtype=np.int32)
        want = fo.std_sort_by_length(idx, length)
        assert np.array_equal(fo.restated_sort_by_length(idx, length), want), (t, n)
        differs_from_stable += not np.array_equal(want, idx[np.argsort(-length, kind="stable")])
    assert differs_from_stable > 1000            # the ties really are ordered by the algorithm
    # shapes that drive the introsort into its heap-sort fallback and its degenerate partitions
    for n in (17, 100, 1000, 5000):
        for length in (np.full(n, 5), np.arange(n), np.arange(n)[::-1], np.minimum(np.arange(n), n - np.arange(n))):
            length = np.ascontiguousarray(length, dtype=np.int32)
            idx = np.arange(n, dtype=np.int32)
            assert np.array_equal(fo.restated_sort_by_length(idx, length), fo.std_sort_by_length(idx, length))


def _sequence(n_frames, w=320, h=240, seed=3):
    """frames of a smooth random texture seen by a camera that rotates (and shifts a little), with the rotation
    between frames as predict_q"""
    from scipy.spatial.transform import Rotation
    rng = np.random.default_rng(seed)
    tex = cv2.GaussianBlur(rng.integers(0, 256, (3 * h, 3 * w)).astype(np.float32), (0, 0), 2.0)
    tex = cv2.normalize(tex, None, 0, 255, cv2.NORM_MINMAX).astype(np.uint8)
    K = (300.0, 300.0, w / 2 - 0.5, h / 2 + 0.25)
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    T = np.array([[1, 0, -w], [0, 1, -h], [0, 0, 1.0]])        # texture pixel -> reference camera pixel
    frames, qs, R = [], [], np.eye(3)
    for k in range(n_frames):
        Rk = Rotation.from_rotvec(rng.normal(0, 0.006, 3)).as_matrix()
        R = Rk @ R
        qs.append(Rotation.from_matrix(Rk).as_quat())
        H = Km @ R @ np.linalg.inv(Km) @ T
        H[:2, 2] += rng.normal(0, 0.3, 2)
        frames.append(cv2.warpPerspective(tex, H, (w, h), flags=cv2.INTER_LINEAR))
    return frames, qs, K


def test_oracle_step_on_a_synthetic_sequence():
    frames, qs, K = _sequence(6)
    clahe = cv2.createCLAHE(6.0, (8, 8))
    eq = [clahe.apply(f) for f in frames]
    r = 20.0
    z, prev, birth, counts = fo.step(None, eq[0], np.zeros((0, 2)), [], [], 0, 0, K, K, None, r)
    assert counts[:3] == [0, 0, 0] and counts[3] == len(z) > 20 and np.all(prev == -1) and np.all(birth == 1)
    for k in range(1, 6):
        zp, pp, bp = z, prev, birth
        z, prev, birth, counts = fo.step(eq[k - 1], eq[k], zp, pp, bp, k, k, K, K, qs[k], r)
        assert counts[0] >= counts[1] >= counts[2] > 0.5 * len(zp)
        assert len(z) == counts[2] + counts[3]
        kept = prev[prev >= 0]
        assert np.all(np.diff(kept) > 0)                        # survivors in previous-frame order
        assert np.array_equal(birth[:counts[2]], bp[kept])
        px = fo.apply_k(z, K)
        # survivors that had a track are at least r apart (the filter's skipped cell lies a full r away)
        tracked = px[:counts[2]][pp[kept] != -1]
        if len(tracked) > 1:
            d = np.linalg.norm(tracked[:, None] - tracked[None], axis=2) + np.eye(len(tracked)) * 1e9
            assert d.min() >= r - 1e-9
        # detections: integer pixels inside the 20-px border, after every survivor
        det = px[counts[2]:]
        assert np.allclose(det, np.round(det)) and np.all(det >= 20 - 1e-9)
    # the guesses: cv2's LK from these initial positions equals its LK from the rotated positions
    p0, p1 = fo.guesses(z, K, K, qs[1])
    assert p0.dtype == np.float32 and p1.dtype == np.float32 and np.abs(p1 - p0).max() > 0.1
    assert np.array_equal(fo.guesses(z, K, K, None)[1], p0)


def test_capacity_bound_and_rejections():
    img = np.zeros((480, 752), np.uint8)
    gs = 20 / math.sqrt(2)
    assert ft.min_capacity(752, 480, 20) == (math.floor(752 / gs) + 1) * (math.floor(480 / gs) + 1) + 2000
    ok = {"slot": 0, "frame_id": 1, "image": img, "K": (400, 400, 376, 240), "map_frames": 0}
    ft.check_frames([ok, dict(ok, slot=1)], 20.0)
    with pytest.raises(ValueError, match="twice"):
        ft.check_frames([ok, dict(ok)], 20.0)
    with pytest.raises(ValueError, match="below"):
        ft.check_frames([dict(ok, max_keypoints=ft.min_capacity(752, 480, 20) - 1)], 20.0)
    with pytest.raises(ValueError, match="frame id"):
        ft.check_frames([dict(ok, frame_id=0)], 20.0)
    with pytest.raises(ValueError, match="frame id"):
        ft.check_frames([dict(ok, image=None)], 20.0)
    with pytest.raises(ValueError, match="map_frames"):
        ft.check_frames([dict(ok, map_frames=-1)], 20.0)
    with pytest.raises(ValueError, match="out of range"):
        ft.check_frames([dict(ok, slot=65536)], 20.0)
    with pytest.raises(ValueError, match="keypoint_distance"):
        ft.check_frames([ok], 0.0)
