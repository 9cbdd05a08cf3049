"""Reference of the resident windows' covariance (pvio_b200_batch_window_covariance): the dense inverse of the
bundle-adjustment normal equations of ba_oracle over its free coordinates, and the landmark-elimination form of an
inverse-depth variance that the device computes."""
import numpy as np

from . import ba_oracle, chol_oracle


def covariance(win, st, frames, tracks, refine=False):
    """The covariance the resident slots return (pvio_b200_batch_window_covariance): the inverse of H = J^T J
    (ba_oracle.normal_equations, no regulariser) over ba_oracle.free_mask, taken densely.  frames: window indices,
    their joint block [15 k, 15 k] with zero rows / columns for the coordinates that are not free; tracks: landmark
    indices of `win` (None or < 0: not a landmark), their inverse-depth variances (NaN for None or a landmark without free coordinate).
    refine: the inverse by residual refinement (chol_oracle.refined_inverse), for ill-conditioned windows, instead of
    one factorisation.  Returns (cov, var, Sigma) with Sigma over the free coordinates in local-coordinate order."""
    H, _, _ = ba_oracle.normal_equations(win, st)
    free = ba_oracle.free_mask(win)
    idx = np.flatnonzero(free)
    Hf = H[np.ix_(idx, idx)]
    if refine:
        Sig = chol_oracle.refined_inverse(Hf)
        Sig = 0.5 * (Sig + Sig.T)
    else:
        Sig = np.linalg.inv(Hf)
    pos = -np.ones(ba_oracle.local_dim(win), dtype=int)
    pos[idx] = np.arange(len(idx))
    cols = np.concatenate([15 * int(f) + np.arange(15) for f in frames]) if len(frames) else np.zeros(0, dtype=int)
    cov = np.zeros((len(cols), len(cols)))
    pc = pos[cols]
    ok = pc >= 0
    cov[np.ix_(ok, ok)] = Sig[np.ix_(pc[ok], pc[ok])]
    var = np.full(len(tracks), np.nan)
    for k, l in enumerate(tracks):
        if l is not None and l >= 0 and pos[15 * win.N + l] >= 0:
            var[k] = Sig[pos[15 * win.N + l], pos[15 * win.N + l]]
    return cov, var, Sig


def landmark_variance(win, st, l, Sig_ff=None):
    """Var(rho_l) by the elimination: 1 / H_ll + h_l^T Sigma_ff h_l / H_ll^2, h_l the landmark's coupling to the free
    frame coordinates and Sigma_ff the frame block of the inverse of H over free_mask (the Schur complement's inverse)."""
    H, _, _ = ba_oracle.normal_equations(win, st)
    free = ba_oracle.free_mask(win)
    ff = np.flatnonzero(free[:15 * win.N])
    fl = 15 * win.N + np.flatnonzero(free[15 * win.N:])
    if Sig_ff is None:
        Hff, Hfl, Hll = H[np.ix_(ff, ff)], H[np.ix_(ff, fl)], H[np.ix_(fl, fl)]
        Sig_ff = np.linalg.inv(Hff - Hfl @ np.diag(1.0 / np.diag(Hll)) @ Hfl.T)
    c = 15 * win.N + l
    h = H[ff, c]
    return 1.0 / H[c, c] + h @ Sig_ff @ h / H[c, c] ** 2
