"""cov_oracle.covariance, the reference of pvio_b200_batch_window_covariance, on small windows: H Sigma = I over the free
coordinates, the landmark-elimination formula of the device equal to the diagonal of the dense inverse, the frame blocks
equal to the dense inverse's, and zero rows / columns and NaN variances where a coordinate is not free."""
import numpy as np
import pytest

from oracle import ba_oracle, cov_oracle
from synthetic import synth


def _windows():
    w4, s4 = synth.make_cfg4(seed=981, N=4, M=24)[:2]            # prior, IMU, planes
    w2, s2 = synth.make_cfg2(seed=982, N=4, M=30)[:2]            # visual only, two fixed frames
    return [(w4, s4), (w2, s2)]


@pytest.mark.parametrize("k", [0, 1])
def test_covariance_inverts_h_on_the_free_coordinates(k):
    w, st = _windows()[k]
    free = ba_oracle.free_mask(w)
    H = ba_oracle.normal_equations(w, st)[0][np.ix_(free, free)]
    for refine in (False, True):
        _, _, Sig = cov_oracle.covariance(w, st, [], [], refine=refine)
        d = np.sqrt(np.diag(H))
        # in the diagonal scaling: D^-1/2 H D^-1/2 (D^1/2 Sigma D^1/2) = I
        R = (H / np.outer(d, d)) @ (Sig * np.outer(d, d)) - np.eye(len(d))
        assert np.abs(R).max() < 1e-6, (refine, np.abs(R).max())
        assert np.allclose(Sig, Sig.T, rtol=0, atol=1e-12 * np.abs(Sig).max())


@pytest.mark.parametrize("k", [0, 1])
def test_landmark_formula_is_the_diagonal_of_the_inverse(k):
    w, st = _windows()[k]
    tracks = list(range(w.M)) + [None, -1]
    cov, var, Sig = cov_oracle.covariance(w, st, list(range(w.N)), tracks, refine=True)
    assert np.isnan(var[-2:]).all()
    ref = np.array([cov_oracle.landmark_variance(w, st, l) for l in range(w.M)])
    assert np.all(var[:w.M] > 0)
    assert np.max(np.abs(var[:w.M] - ref) / ref) < 1e-7
    # frames: the joint block of the dense inverse, zero where a coordinate is not free
    free = ba_oracle.free_mask(w)[:15 * w.N]
    assert np.all(cov[~free, :] == 0) and np.all(cov[:, ~free] == 0)
    idx = np.flatnonzero(free)
    assert np.array_equal(cov[np.ix_(idx, idx)], Sig[:len(idx), :len(idx)])
    # a sub-selection in another order is the matching block of the whole
    sel = [w.N - 1, 0]
    c2 = cov_oracle.covariance(w, st, sel, [], refine=True)[0]
    cols = np.concatenate([15 * f + np.arange(15) for f in sel])
    assert np.array_equal(c2, cov[np.ix_(cols, cols)])
    if not w.use_inertial:
        assert w.frame_fixed.sum() == 2
