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


def _mp_spd_inverse(A):
    """the inverse of a symmetric positive definite matrix of mpf entries (lists of rows) by Cholesky, at the working
    mpmath precision: L L^T = A, W = L^-1 row by row, A^-1 = W^T W"""
    import mpmath as mp
    n = len(A)
    L = [[mp.mpf(0)] * n for _ in range(n)]
    for j in range(n):
        Lj = L[j]
        Lj[j] = mp.sqrt(A[j][j] - mp.fdot(Lj[:j], Lj[:j]))
        for i in range(j + 1, n):
            L[i][j] = (A[i][j] - mp.fdot(L[i][:j], Lj[:j])) / Lj[j]
    W = [[mp.mpf(0)] * n for _ in range(n)]
    for i in range(n):
        W[i][i] = 1 / L[i][i]
        for j in range(i):
            W[i][j] = -mp.fdot(L[i][j:i], [W[k][j] for k in range(j, i)]) / L[i][i]
    cols = [[W[k][j] for k in range(n)] for j in range(n)]
    X = [[None] * n for _ in range(n)]
    for i in range(n):
        for j in range(i, n):
            X[i][j] = X[j][i] = mp.fdot(cols[i][j:], cols[j][j:])
    return X


@pytest.mark.parametrize("case", ["inertial N 11", "visual N 16"])
def test_refined_reference_matches_a_50_digit_inverse(case):
    """the largest windows of test_gpu_batch_window_covariance_shapes.py (40 landmarks): the free-coordinate Schur
    complement of the fp64 H formed and inverted in 50 digits, and Var(rho_l) = 1 / H_ll + h_l^T Sigma_ff h_l / H_ll^2
    from it; cov_oracle.covariance(refine=True) agrees to 1e-12 on every frame block (relative to sqrt(C_ii C_jj)) and
    every Var(rho), so that the GPU bars measure the kernels and not the reference"""
    import mpmath as mp
    if case.startswith("inertial"):
        w, st = synth.make_cfg3(seed=1211, N=11, M=40)[:2]
    else:
        w, st = synth.make_cfg2(seed=1016, N=16, M=40)[:2]
    H = ba_oracle.normal_equations(w, st)[0]
    free = ba_oracle.free_mask(w)
    n = 15 * w.N
    ff, fl = np.flatnonzero(free[:n]), n + np.flatnonzero(free[n:])
    with mp.workdps(50):
        S = [[mp.mpf(x) for x in row] for row in H[np.ix_(ff, ff)].tolist()]
        coup = []
        for c in fl:                                     # S = H_ff - sum_l h_l h_l^T / H_ll (H_ll is diagonal)
            nz = np.flatnonzero(H[ff, c])
            h = [mp.mpf(H[ff[i], c]) for i in nz]
            hll = mp.mpf(H[c, c])
            coup.append((nz, h, hll))
            for a, i in enumerate(nz):
                hi = h[a] / hll
                for b, j in enumerate(nz):
                    S[i][j] -= hi * h[b]
        X = _mp_spd_inverse(S)
        var = [1 / hll + mp.fsum(h[a] * h[b] * X[i][j] for a, i in enumerate(nz) for b, j in enumerate(nz)) / hll ** 2
               for nz, h, hll in coup]
        Xf = np.array([[float(x) for x in row] for row in X])
        vf = np.array([float(v) for v in var])
    cov, v_ref, _ = cov_oracle.covariance(w, st, list(range(w.N)), list(range(w.M)), refine=True)
    sub = cov[np.ix_(ff, ff)]
    d = np.sqrt(np.diag(Xf))
    e_cov = float(np.max(np.abs(sub - Xf) / np.outer(d, d)))
    e_var = float(np.max(np.abs(v_ref[fl - n] - vf) / vf))
    print(f"{case}: {len(ff)} frame coordinates, {len(fl)} landmarks, frames {e_cov:.3g}, Var(rho) {e_var:.3g}")
    assert np.all(cov[~free[:n]] == 0)
    assert e_cov < 1e-12 and e_var < 1e-12, (e_cov, e_var)
