"""TEST INFRASTRUCTURE (CPU oracle) -- the state of a resident inertial window at any time inside it, as
pvio_b200_batch_window_trajectory defines it (include/pvio_b200.h), composed from the existing restatements:
imu_oracle.integrate over the sample prefix, imu_stream_cov_oracle.predict for the state, imu_stream_cov_oracle.factor
for Phi and Psi, and Sigma_k from cov_oracle.covariance (the caller passes it).  No algebra of its own.

A window's factors are given as a list, factor k (frames k, k + 1) as (samples [m][7] or None, t_end)."""
import numpy as np

from . import imu_oracle
from . import imu_stream_cov_oracle as sco


def _holds(f):
    return f[0] is not None and len(f[0]) > 0


def noise_of(noise, k):
    """factor k's noise (cov_w, cov_a, cov_bg, cov_ba): noise is one such tuple for every factor, or a list of one per
    factor (None for a factor without samples)"""
    per_factor = len(noise) > 0 and (noise[0] is None or np.ndim(noise[0]) == 3)
    return noise[k] if per_factor else noise


def factor_of(t, factors):
    """the factor k that takes time t: the largest k holding samples with s_0.t <= t, when t <= its t_end or factor
    k + 1 holds samples too; -1 when none does"""
    ks = [k for k, f in enumerate(factors) if _holds(f) and f[0][0, 0] <= t]
    if not ks:
        return -1
    k = ks[-1]
    if t <= factors[k][1] or (k + 1 < len(factors) and _holds(factors[k + 1])):
        return k
    return -1


class _NoSqrtInv:
    """numpy as imu_oracle.integrate sees it, with the final LLT(cov^-1) left NaN: a prefix of one increment, or of
    zero length, has a singular covariance, and the trajectory does not use sqrt_inv_cov"""
    class linalg:
        @staticmethod
        def inv(a):
            return np.full_like(a, np.nan)

        @staticmethod
        def cholesky(a):
            return a

    def __getattr__(self, k):
        return getattr(np, k)


def delta(samples, t, bg, ba, noise):
    """PreIntegrator::integrate(t, bg, ba) over the samples at or before t, the last one up to t (imu_oracle.integrate's
    dict; at t = s_0.t the increment has length 0)"""
    s = np.asarray(samples, dtype=np.float64).reshape(-1, 7)
    pre = s[s[:, 0] <= t]
    try:
        return imu_oracle.integrate(pre, t, bg, ba, *noise)
    except np.linalg.LinAlgError:
        imu_oracle.np = _NoSqrtInv()
        try:
            return imu_oracle.integrate(pre, t, bg, ba, *noise)
        finally:
            imu_oracle.np = np


def propagate(x_k, d, Sig_k):
    """Phi Sigma_k Phi^T + Psi Sigma_delta Psi^T, symmetrised, with Phi and Psi those of the FACTOR seed
    (imu_stream_cov_oracle.factor; neither depends on the factor's sqrt_inv_cov, so the record carries the identity
    there) and Sigma_delta = d['cov'] taken directly"""
    rec = imu_oracle.record(dict(d, sqrt_inv_cov=np.eye(15)), x_k[10:13], x_k[13:16])      # U unused: the identity
    Phi, Psi, _, _ = sco.factor(sco.predict(x_k, d)[0:4], rec, Sig_k)
    P = 0.5 * (Sig_k + Sig_k.T)
    S = Phi @ P @ Phi.T + Psi @ d["cov"] @ Psi.T
    return 0.5 * (S + S.T)


def trajectory(times, frames, factors, noise, Sig=None):
    """frames [N][16] the window's states; factors as above; noise (cov_w, cov_a, cov_bg, cov_ba), or one such tuple per
    factor (noise_of); Sig: per frame its
    15 x 15 marginal covariance (None: no covariances).  Returns (frame [n], states [n][16], covs [n][15][15] or None):
    frame -1 with a zero state and a NaN covariance for a time no factor takes."""
    n = len(times)
    fr, st = np.full(n, -1, dtype=np.int32), np.zeros((n, 16))
    cov = None if Sig is None else np.full((n, 15, 15), np.nan)
    for i, t in enumerate(times):
        k = factor_of(t, factors)
        if k < 0:
            continue
        x = np.asarray(frames[k], dtype=np.float64)
        d = delta(factors[k][0], t, x[10:13], x[13:16], noise_of(noise, k))
        fr[i], st[i] = k, sco.predict(x, d)
        if Sig is not None:
            cov[i] = propagate(x, d, Sig[k])
    return fr, st, cov
