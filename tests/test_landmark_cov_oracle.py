"""landmark_oracle, the reference of pvio_b200_batch_window_landmarks, on small windows: the elimination form of a world
point's covariance (what the device computes) equal to the dense form (Sigma over the free coordinates through a
central-difference Jacobian), the world point against tri_oracle's camera matrices, and the fixed-anchor case."""
import numpy as np
import pytest

import landmark_oracle as lo
from oracle import ba_oracle, cov_oracle, tri_oracle
from synthetic import synth


def _windows():
    w4, s4 = synth.make_cfg4(seed=981, N=4, M=24)[:2]            # gauge prior, IMU, planes
    w3, s3 = synth.make_cfg3(seed=983, N=5, M=30)[:2]            # IMU, a prior over all but the newest frame (the
    w2, s2 = synth.make_cfg2(seed=982, N=4, M=30)[:2]            #   shape after a marginalisation); visual only, two fixed frames
    return [(w4, s4), (w3, s3), (w2, s2)]


def _rel(C, R):
    d = np.sqrt(np.abs(np.diag(R)))
    return float(np.max(np.abs(C - R) / np.outer(d, d)))


@pytest.mark.parametrize("k", [0, 1, 2])
def test_elimination_form_equals_the_dense_form(k):
    w, st = _windows()[k]
    if k == 1:
        assert 0 < w.n_prior < w.N
    tracks = list(range(w.M)) + [None]
    dense = lo.point_covariance(w, st, tracks)
    elim, var = lo.point_covariance_elim(w, st, tracks)
    assert np.isnan(dense[-1]).all() and np.isnan(elim[-1]).all() and np.isnan(var[-1])
    _, var_ref, _ = cov_oracle.covariance(w, st, [], tracks[:-1], refine=True)
    assert np.max(np.abs(var[:-1] - var_ref) / var_ref) < 1e-8
    worst = max(_rel(elim[l], dense[l]) for l in range(w.M))
    assert worst < 1e-8, worst
    for l in range(w.M):
        assert np.allclose(elim[l], elim[l].T, rtol=0, atol=1e-14 * np.abs(elim[l]).max())
        assert np.linalg.eigvalsh(dense[l]).min() > -1e-12 * np.abs(dense[l]).max()


@pytest.mark.parametrize("k", [0, 2])
def test_point_reprojects_onto_the_anchor_keypoint(k):
    w, st = _windows()[k]
    for l in range(w.M):
        a = int(w.lm_anchor[l])
        P = tri_oracle.projection_matrix(*lo.camera_pose(w, st, a))
        y = P @ np.append(lo.landmark_point(w, st, l), 1.0)
        assert np.allclose(y[:2] / y[2], w.lm_z_ref[l], rtol=0, atol=1e-12)
        assert abs(y[2] * st.rho[l] - 1.0) < 1e-12


def test_fixed_anchor_reduces_to_the_inverse_depth_term():
    w, st = _windows()[2]
    fixed = [l for l in range(w.M) if w.frame_fixed[int(w.lm_anchor[l])]]
    assert fixed
    elim, var = lo.point_covariance_elim(w, st, fixed)
    dense = lo.point_covariance(w, st, fixed)
    for k, l in enumerate(fixed):
        a = int(w.lm_anchor[l])
        x = lo.landmark_point(w, st, l)
        c = -(x - lo.camera_pose(w, st, a)[1]) / st.rho[l]
        ref = np.outer(c, c) * var[k]
        assert _rel(elim[k], ref) < 1e-12
        assert _rel(dense[k], ref) < 1e-8
    assert ba_oracle.free_mask(w)[15 * w.N:].all()
