"""TEST INFRASTRUCTURE (CPU oracle) -- the state of a resident inertial window at any time inside it conditioned on both
solved frames around it, as pvio_b200_batch_window_smoothed_trajectory defines it (include/pvio_b200.h), composed from
the existing restatements as oracle/trajectory_oracle.trajectory is: imu_oracle.integrate over the sample prefix
(trajectory_oracle.delta), imu_stream_cov_oracle.predict for the state and imu_stream_cov_oracle.factor for Phi and Psi,
with the joint frame covariance from cov_oracle.covariance (the caller passes it).

Cov(e(t), e(T)) is taken by a route of its own, not the device's adjoint: an augmented 30-dimensional covariance
[frozen copy of e(t); running e] propagated along the split chain (imu_stream_cov_oracle.step's 9 x 9 block per
step), whose cross block is read off.  Factors are given as trajectory_oracle takes them: factor k (frames k, k + 1) as
(samples [m][7] or None, t_end)."""
import numpy as np

from oracle import imu_oracle
from oracle import imu_stream_cov_oracle as sco
from oracle import lie
from oracle.trajectory_oracle import delta, factor_of, noise_of

_G = sco.GRAVITY


def chol_pd(S):
    """Sigma(T) positive definite as the device decides it: sqrt_inv_block's factor S = R R^T, R upper triangular, run
    from the last row up, with every pivot R_jj^2 above 1e-10 times S_jj (a one-sample factor's C(T) has rank 6, and
    its missing pivots are rounding)"""
    S = np.asarray(S, dtype=np.float64)
    n = len(S)
    R = np.zeros((n, n))
    for j in range(n - 1, -1, -1):
        d = S[j, j] - R[j, j + 1:] @ R[j, j + 1:]
        if not d > 1e-10 * S[j, j]:
            return False
        R[j, j] = np.sqrt(d)
        for i in range(j):
            R[i, j] = (S[i, j] - R[i, j + 1:] @ R[j, j + 1:]) / R[j, j]
    return True


def target(x_k, x_k1, T):
    """Delta*: the increment (dq, dp, dv, bias step) that imu_stream_cov_oracle.predict maps from x_k onto x_k1 exactly
    over T"""
    q = x_k[0:4]
    Rt = lie.qmat(q).T
    return (lie.qmul(lie.qconj(q), x_k1[0:4]),
            Rt @ (x_k1[4:7] - x_k[4:7] - x_k[7:10] * T - 0.5 * _G * T * T),
            Rt @ (x_k1[7:10] - x_k[7:10] - _G * T),
            x_k1[10:16] - x_k[10:16])


def residual(x_k, x_k1, dT):
    """r = Delta* (-) Delta(T), [r_theta r_p r_v r_bg r_ba]"""
    dq, dp, dv, db = target(x_k, x_k1, dT["dt"])
    return np.concatenate([lie.logmap(lie.qmul(lie.qconj(dT["dq"]), dq)), dp - dT["dp"], dv - dT["dv"], db])


def _aug_step(P, q, smp, dt, bg, ba, noise):
    """one step of the augmented covariance [frozen e(t); running e]: the running half moves as imu_oracle.integrate
    moves the increment's covariance over dt of sample smp from rotation q (sco.step's 9 x 9 block, bias walks)"""
    F, Q = sco.step((0.0, q, None, None, bg, ba), dt, smp[1:4], smp[4:7], noise)
    Fi = np.eye(15)
    Fi[0:9, 0:9] = F[0:9, 0:9]
    Qi = np.zeros((15, 15))
    Qi[0:9, 0:9] = Q[0:9, 0:9]
    Qi[9:15, 9:15] = Q[9:15, 9:15]
    Fa = np.eye(30)
    Fa[15:30, 15:30] = Fi
    Qa = np.zeros((30, 30))
    Qa[15:30, 15:30] = Qi
    return Fa @ P @ Fa.T + Qa


def cross_cov(samples, t, t_end, bg, ba, noise):
    """Cov(e(t), e(T)) by the augmented 30-dimensional covariance along the split chain: from t, the rest of the sample
    t lies in, then the whole later samples up to t_end (past t_end: from t_end on to t over the last sample, then read
    transposed).  The chain's rotations are the prefix integrations' own."""
    s = np.asarray(samples, dtype=np.float64).reshape(-1, 7)
    nz = np.concatenate([np.asarray(c, dtype=np.float64).reshape(9) for c in noise])
    if t > t_end:
        dT = delta(s, t_end, bg, ba, noise)
        S = dT["cov"]
        P = _aug_step(np.block([[S, S], [S, S]]), dT["dq"], s[-1], t - t_end, bg, ba, nz)
        return P[15:30, 0:15]
    d = delta(s, t, bg, ba, noise)
    S = d["cov"]
    P = np.block([[S, S], [S, S]])
    j = int(np.flatnonzero(s[:, 0] <= t)[-1])
    knots = list(s[:, 0]) + [float(t_end)]
    kq = _knot_rotations(s, bg) if np.all(np.diff(s[:, 0]) > 0) else None
    q, t0 = d["dq"], t
    for i in range(j, len(s)):
        P = _aug_step(P, q, s[i], knots[i + 1] - t0, bg, ba, nz)
        if i + 1 < len(s):
            q = delta(s, knots[i + 1], bg, ba, noise)["dq"] if kq is None else kq[i + 1]
            t0 = knots[i + 1]
    return P[0:15, 15:30]


def _knot_rotations(s, bg):
    """delta(s, s_i.t, bg, ...)["dq"] for every sample i of strictly increasing times, in one pass instead of one
    prefix integration per knot: imu_oracle.integrate's rotation chain over samples 0 .. i - 1, then the zero-length
    step of sample i that closes a prefix ending at s_i.t -- the same operations in the same order, so the same bits"""
    bg = np.asarray(bg, dtype=np.float64)
    dq, out = np.array([0.0, 0.0, 0.0, 1.0]), []
    for i in range(len(s)):
        w = s[i, 1:4] - bg
        out.append(lie.qnormalized(lie.qmul(dq, lie.expmap(w * (s[i, 0] - s[i, 0])))))
        if i + 1 < len(s):
            dq = lie.qnormalized(lie.qmul(dq, lie.expmap(w * (s[i + 1, 0] - s[i, 0]))))
    return out


def gain(samples, t, t_end, bg, ba, noise):
    """(K(t), Sigma_c(t), Delta(t), Delta(T)): K = Cov(e(t), e(T)) Sigma(T)^-1, Sigma_c = Sigma(t) - K Cov(e(T), e(t));
    None when Sigma(T) is not positive definite"""
    d = delta(samples, t, bg, ba, noise)
    dT = delta(samples, t_end, bg, ba, noise)
    ST = dT["cov"]
    if not (chol_pd(ST[0:9, 0:9]) and chol_pd(ST[9:12, 9:12]) and chol_pd(ST[12:15, 12:15])):
        return None
    X = cross_cov(samples, t, t_end, bg, ba, noise)
    K = np.linalg.solve(ST, X.T).T
    return K, d["cov"] - K @ X.T, d, dT


def _boxplus(d, u):
    """Delta (+) u: the rotation on the right, the rest added"""
    return dict(d, dq=lie.qmul(d["dq"], lie.expmap(u[0:3])), dp=d["dp"] + u[3:6], dv=d["dv"] + u[6:9])


def smoothed_state(x_k, x_k1, d, dT, K):
    """x_s(t) = predict(x_k, Delta(t) (+) K r), the bias part of K r added to x_k's biases"""
    x_k, x_k1 = np.asarray(x_k, dtype=np.float64), np.asarray(x_k1, dtype=np.float64)
    u = K @ residual(x_k, x_k1, dT)
    x = sco.predict(x_k, _boxplus(d, u))
    x[10:16] = x_k[10:16] + u[9:15]
    return x


def jacobians(x_k, x_k1, d, dT, K):
    """(J_k, J_k1) = d x_s / d x_k, d x_s / d x_k1 in the covariance call's coordinates with K held fixed, Delta(t) and
    Delta(T) moving with x_k's biases through their bias Jacobians: J_k = Phi + Psi G K dr/dx_k, J_k1 = Psi G K dr/dx_k1,
    Phi and Psi the FACTOR seed's at Delta_s(t) (its dq_dbg carried through exp(u_theta)), G the box-plus Jacobian
    diag(Jr(u_theta), I)"""
    x_k, x_k1 = np.asarray(x_k, dtype=np.float64), np.asarray(x_k1, dtype=np.float64)
    r = residual(x_k, x_k1, dT)
    u = K @ r
    ds = _boxplus(d, u)
    Eu = lie.qmat(lie.expmap(u[0:3]))
    rec = imu_oracle.record(dict(ds, dq_dbg=Eu.T @ d["dq_dbg"], sqrt_inv_cov=np.eye(15)), x_k[10:13], x_k[13:16])
    Phi, Psi, _, _ = sco.factor(sco.predict(x_k, ds)[0:4], rec, np.eye(15))
    T = dT["dt"]
    dq_s, dp_s, dv_s, _ = target(x_k, x_k1, T)
    Rk = lie.qmat(x_k[0:4])
    Jri = np.linalg.inv(lie.right_jacobian(r[0:3]))
    Er = lie.qmat(lie.expmap(r[0:3]))
    Dk, Dk1 = np.zeros((15, 15)), np.zeros((15, 15))
    Dk[0:3, 0:3] = -Jri @ lie.qmat(dq_s).T
    Dk[0:3, 9:12] = -Jri @ Er.T @ dT["dq_dbg"]
    Dk[3:6, 0:3] = lie.hat(dp_s)
    Dk[3:6, 3:6] = -Rk.T
    Dk[3:6, 6:9] = -T * Rk.T
    Dk[3:6, 9:12], Dk[3:6, 12:15] = -dT["dp_dbg"], -dT["dp_dba"]
    Dk[6:9, 0:3] = lie.hat(dv_s)
    Dk[6:9, 6:9] = -Rk.T
    Dk[6:9, 9:12], Dk[6:9, 12:15] = -dT["dv_dbg"], -dT["dv_dba"]
    Dk[9:15, 9:15] = -np.eye(6)
    Dk1[0:3, 0:3] = Jri
    Dk1[3:6, 3:6] = Rk.T
    Dk1[6:9, 6:9] = Rk.T
    Dk1[9:15, 9:15] = np.eye(6)
    G = np.eye(15)
    G[0:3, 0:3] = lie.right_jacobian(u[0:3])
    return Phi + Psi @ G @ K @ Dk, Psi @ G @ K @ Dk1, Psi


def smoothed(times, frames, factors, noise, Sig_joint=None):
    """frames, factors, noise as trajectory() (one tuple, or one per factor); Sig_joint: the 15 N x 15 N joint covariance of the window's frames (None:
    no covariances).  Returns (frame [n], states [n][16], covs [n][15][15] or None): frame as trajectory() gives it, or
    -2 with a zero state and a NaN covariance when the factor's Sigma(T) is not positive definite."""
    n = len(times)
    fr, st = np.full(n, -1, dtype=np.int32), np.zeros((n, 16))
    cov = None if Sig_joint is None else np.full((n, 15, 15), np.nan)
    for i, t in enumerate(times):
        k = factor_of(t, factors)
        if k < 0:
            continue
        x, x1 = np.asarray(frames[k], dtype=np.float64), np.asarray(frames[k + 1], dtype=np.float64)
        g = gain(factors[k][0], t, factors[k][1], x[10:13], x[13:16], noise_of(noise, k))
        if g is None:
            fr[i] = -2
            continue
        K, Sc, d, dT = g
        fr[i], st[i] = k, smoothed_state(x, x1, d, dT, K)
        if Sig_joint is not None:
            Jk, Jk1, Psi = jacobians(x, x1, d, dT, K)
            J = np.concatenate([Jk, Jk1], axis=1)
            Sj = np.asarray(Sig_joint, dtype=np.float64)[15 * k:15 * k + 30, 15 * k:15 * k + 30]
            S = J @ (0.5 * (Sj + Sj.T)) @ J.T + Psi @ (0.5 * (Sc + Sc.T)) @ Psi.T
            cov[i] = 0.5 * (S + S.T)
    return fr, st, cov
