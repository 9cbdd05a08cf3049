"""Growth paths of the handle's buffers: plane staging that is re-strided while earlier slots are packed, and module
state (KLT, detector, F-matrix RANSAC) rebuilt when the image shape or the point count changes, plus the per-call
buffers of triangulate / preintegrate / CLAHE.  Every result must equal the same call on a fresh handle."""
import numpy as np
import pytest

from oracle import lie, tri_oracle
from pvio_b200 import imu, klt
from pvio_b200 import triangulate as tri
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200.detect import detect_keypoints
from synthetic import synth

pytestmark = pytest.mark.gpu

CAPS = dict(max_frames=9, max_landmarks=320, max_obs=6000)


def test_plane_staging_survives_restride():
    """Slot 1 needs more than the 256 plane tracks the staging starts with: the staging is re-strided while slot 0
    already holds a packed window, and both slots must still solve as their own single-window solves do."""
    small = synth.make_cfg4()[:2]
    big = synth.make_cfg4(seed=651, tracks_per_plane=130)[:2]
    assert small[0].n_ptracks == 80 and big[0].n_ptracks > 256
    ref = BundleAdjustor(max_windows=1, **CAPS)
    singles = [ref.solve(w, st, max_iterations=7) for w, st in (small, big)]
    ref.close()
    b = BundleAdjustor(max_windows=2, **CAPS)
    try:
        b.batch_set(0, *small)
        b.batch_set(1, *big)              # ensure_planes grows Tcap past 256 here
        b.batch_upload(2)
        b.batch_solve(2, max_iterations=7)
        frames, rho, sm = b.batch_download_state(2, CAPS["max_frames"], CAPS["max_landmarks"])
    finally:
        b.close()
    for i, (w, st) in enumerate((small, big)):
        ref_state, ref_sum = singles[i]
        assert sm[i]['iterations'] == ref_sum['iterations'] and sm[i]['termination'] == ref_sum['termination']
        assert sm[i]['accepted_steps'] == ref_sum['accepted_steps']
        assert abs(sm[i]['final_cost'] - ref_sum['final_cost']) <= 1e-9 * ref_sum['final_cost']
        assert np.allclose(frames[i, :w.N, 4:7], ref_state.p, rtol=0, atol=1e-9)
        assert np.allclose(rho[i, :w.M], ref_state.rho, rtol=1e-9, atol=0)


def _tri_inputs(n_tracks, seed):
    rng = np.random.default_rng(seed)
    F = 6
    P = np.array([tri_oracle.projection_matrix(lie.expmap(rng.normal(0, 0.05, 3)), np.array([0.25 * i, 0.02 * i, 0.0]))
                  for i in range(F)])
    begin, fr, zs = [0], [], []
    for _ in range(n_tracks):
        X = np.array([rng.uniform(-1, 1), rng.uniform(-1, 1), rng.uniform(2, 10)])
        frames = np.sort(rng.choice(F, int(rng.integers(2, F + 1)), replace=False))
        for f in frames:
            y = P[f] @ np.r_[X, 1.0]
            fr.append(f)
            zs.append(y[:2] / y[2] + rng.normal(0, 1e-3, 2))
        begin.append(len(fr))
    return P, begin, fr, np.array(zs)


def _imu_inputs(n_factors, seed):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n_factors):
        K = int(rng.integers(5, 40))
        t = np.arange(K) / 200.0
        samples = np.c_[t, rng.normal(0, 0.3, (K, 3)), rng.normal(0, 1.0, (K, 3)) + np.array([0.0, 0.0, 9.81])]
        out.append((samples, t[-1] + 0.004, rng.normal(0, 1e-2, 3), rng.normal(0, 5e-2, 3)))
    return out


IMU_COV = (np.eye(3) * 2.8791e-8, np.eye(3) * 4.0e-6, np.eye(3) * 3.7608e-10, np.eye(3) * 9.0e-6)


def _calls():
    """(name, call(ba)) in the order one handle runs them: every stateful call at one size, a larger size that
    forces a rebuild, then the first size again."""
    pairs = {s: synth.make_klt_pair(size=s, n_points=1200) for s in ((752, 480), (1280, 720))}
    small, large = pairs[(752, 480)], pairs[(1280, 720)]
    assert len(small[2]) < 1024 < len(large[2])          # the large call also outgrows the point capacity
    fm = {n: synth.make_fm_matches(n=n, seed=652 + n) for n in (300, 1500)}
    tri_in = {n: _tri_inputs(n, 700 + n) for n in (50, 400)}
    imu_in = {n: _imu_inputs(n, 800 + n) for n in (3, 40)}
    calls = []
    for pr in (small, large, small):
        calls.append(("klt", lambda ba, pr=pr: klt.track_keypoints(ba, pr[0], pr[1], pr[2], raw=True, clahe_clip=6.0)))
    for pr in (small, large, small):
        calls.append(("detect", lambda ba, pr=pr: detect_keypoints(ba, pr[1], clahe_clip=6.0, want_gftt=True)))
    for n in (300, 1500, 300):
        calls.append(("fm", lambda ba, n=n: klt.find_fundamental_mask(ba, *fm[n], return_info=True)))
    for n in (50, 400, 50):
        calls.append(("triangulate", lambda ba, n=n: tri.triangulate(ba, *tri_in[n])))
    for n in (3, 40, 3):
        calls.append(("preintegrate", lambda ba, n=n: imu.preintegrate(ba, imu_in[n], IMU_COV)))
    for pr in (small, large, small):
        calls.append(("clahe", lambda ba, pr=pr: klt.clahe(ba, pr[0])))
    return calls


def _same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return np.array_equal(np.asarray(a), np.asarray(b))


def _handle():
    return BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)


def test_module_state_rebuilt_on_shape_changes():
    calls = _calls()
    fresh = []
    for _, call in calls:
        b = _handle()
        try:
            fresh.append(call(b))
        finally:
            b.close()
    for _ in range(2):                    # the second pass runs on a handle created after the first was destroyed
        b = _handle()
        try:
            for (name, call), want in zip(calls, fresh):
                assert _same(call(b), want), name
        finally:
            b.close()
