"""TEST INFRASTRUCTURE (CPU oracle) -- the covariance of the IMU-rate pose of a stream slot
(pvio_b200_batch_imu_stream_set_covariance / pvio_b200_batch_imu_stream_predict), in fp64 NumPy.

Coordinates are [dtheta dp dv dbg dba] with q perturbed on the right, q (x) exp(dtheta) (lie.quat_plus), as
pvio_b200_batch_window_covariance gives them.  The nonlinear side is imu_stream_oracle's: propagate (propagate_state,
core.cpp:32-39) and the output pose of predict_pose (:158-159).  Here:
  - step: the Jacobian F of one propagate step and its discretised noise (PreIntegrator::increment's, preintegrator.cpp:
    59-67: cov_w / max(dt, 1e-7) through dt Jr into dtheta, cov_a / max(dt, 1e-7) through dt R and dt^2 R / 2 into dv and
    dp, cov_bg dt and cov_ba dt into the biases);
  - chain: P propagated over a slot's kept samples, as predict_pose propagates the state;
  - pose_jacobian: the map to [dtheta_out dp_out] of the OutputPose;
  - factor: the seed of a state predicted through an IMU factor (PreIntegrator::predict, preintegrator.cpp:102-109) from
    a source frame with a known covariance, built on imu_oracle's integration and record layout."""
import numpy as np

from . import imu_stream_oracle as so
from . import lie

GRAVITY = np.array([0.0, 0.0, -so.GRAVITY])


def noise_blocks(noise_cov):
    """noise_cov [4][9] (cov_w, cov_a, cov_bg, cov_ba) -> four 3 x 3 matrices"""
    n = np.asarray(noise_cov, dtype=np.float64).reshape(4, 3, 3)
    return n[0], n[1], n[2], n[3]


def step(st, t, w, a, noise_cov):
    """(F, Q) of so.propagate(st, t, w, a): P <- F P F^T + Q.  p and v move with the old rotation, as propagate moves
    them."""
    ct, q, _, _, bg, ba = st
    cov_w, cov_a, cov_bg, cov_ba = noise_blocks(noise_cov)
    dt = t - ct
    R = lie.qmat(q)
    acc = np.asarray(a, dtype=np.float64) - np.asarray(ba)
    u = (np.asarray(w, dtype=np.float64) - np.asarray(bg)) * dt
    Jr = lie.right_jacobian(u)
    M = R @ lie.hat(acc)
    F = np.eye(15)
    F[0:3, 0:3] = lie.qmat(lie.expmap(u)).T
    F[0:3, 9:12] = -dt * Jr
    F[3:6, 0:3] = -0.5 * dt * dt * M
    F[3:6, 6:9] = dt * np.eye(3)
    F[3:6, 12:15] = -0.5 * dt * dt * R
    F[6:9, 0:3] = -dt * M
    F[6:9, 12:15] = -dt * R
    G = np.zeros((15, 6))
    G[0:3, 0:3] = dt * Jr
    G[3:6, 3:6] = 0.5 * dt * dt * R
    G[6:9, 3:6] = dt * R
    inv_dt = 1.0 / max(dt, 1.0e-7)
    W = np.zeros((6, 6))
    W[0:3, 0:3], W[3:6, 3:6] = cov_w * inv_dt, cov_a * inv_dt
    Q = G @ W @ G.T
    Q[9:12, 9:12] += cov_bg * dt
    Q[12:15, 12:15] += cov_ba * dt
    return F, Q


def chain(state_t, state16, P, samples, t, noise_cov, sincos=so._sincos):
    """The slot's latest state (state_t, state16) with covariance P propagated over the kept samples (t_k, w, a) with
    state_t < t_k <= t, as predict_pose propagates it.  Returns (st, P, Phi): st as so.propagate returns it, Phi the
    product of the steps' F."""
    x = [float(c) for c in state16]
    st = [float(state_t), tuple(x[0:4]), tuple(x[4:7]), tuple(x[7:10]), tuple(x[10:13]), tuple(x[13:16])]
    P = np.array(P, dtype=np.float64)
    Phi = np.eye(15)
    for (tk, w, a) in samples:
        if tk <= state_t or tk > t:
            continue
        F, Q = step(st, tk, w, a, noise_cov)
        P = F @ P @ F.T + Q
        Phi = F @ Phi
        st = so.propagate(st, tk, w, a, sincos)
    return st, P, Phi


def pose_jacobian(q, q_ob, p_ob):
    """[dtheta_out dp_out] of q_out = q q_ob, p_out = p + q p_ob (perturbed as q) over [dtheta dp dv dbg dba]"""
    J = np.zeros((6, 15))
    J[0:3, 0:3] = lie.qmat(q_ob).T
    J[3:6, 0:3] = -lie.qmat(q) @ lie.hat(p_ob)
    J[3:6, 3:6] = np.eye(3)
    return J


def pose_cov(q, P, q_ob, p_ob):
    J = pose_jacobian(q, q_ob, p_ob)
    return J @ P @ J.T


def predict(src16, d):
    """PreIntegrator::predict (preintegrator.cpp:102-109) from the source state [16] through the factor dict d
    (imu_oracle.integrate's keys dt, dq, dp, dv)"""
    q, p, v = np.asarray(src16[0:4]), np.asarray(src16[4:7]), np.asarray(src16[7:10])
    T = d["dt"]
    v_n = v + GRAVITY * T + lie.qrot(q, d["dv"])
    p_n = p + 0.5 * GRAVITY * T * T + v * T + lie.qrot(q, d["dp"])
    return np.concatenate([lie.qmul(q, d["dq"]), p_n, v_n, src16[10:16]])


def factor(q_state, rec, P_src):
    """FACTOR's seed: (Phi, Psi, Sigma_d, Sigma) with Sigma = Phi P_src Phi^T + Psi Sigma_d Psi^T.  rec: the [288] factor
    record (imu_oracle.record layout) returned with the predicted state, q_state the predicted state's q; the source
    rotation is that of q_state (x) dq^-1."""
    rec = np.asarray(rec, dtype=np.float64)
    T, dq, dp, dv = rec[0], rec[1:5], rec[5:8], rec[8:11]
    U = np.triu(rec[11:236].reshape(15, 15))
    J = {k: rec[o:o + 9].reshape(3, 3) for k, o in (("dq_dbg", 236), ("dp_dbg", 245), ("dp_dba", 254),
                                                    ("dv_dbg", 263), ("dv_dba", 272))}
    Rs = lie.qmat(lie.qmul(q_state, lie.qconj(dq)))
    Phi = np.zeros((15, 15))
    Phi[0:3, 0:3] = lie.qmat(dq).T
    Phi[0:3, 9:12] = J["dq_dbg"]
    Phi[3:6, 0:3] = -Rs @ lie.hat(dp)
    Phi[3:6, 3:6] = np.eye(3)
    Phi[3:6, 6:9] = T * np.eye(3)
    Phi[3:6, 9:12] = Rs @ J["dp_dbg"]
    Phi[3:6, 12:15] = Rs @ J["dp_dba"]
    Phi[6:9, 0:3] = -Rs @ lie.hat(dv)
    Phi[6:9, 6:9] = np.eye(3)
    Phi[6:9, 9:12] = Rs @ J["dv_dbg"]
    Phi[6:9, 12:15] = Rs @ J["dv_dba"]
    Phi[9:15, 9:15] = np.eye(6)
    Psi = np.eye(15)
    Psi[3:6, 3:6] = Rs
    Psi[6:9, 6:9] = Rs
    Ui = np.linalg.inv(U)
    Sig_d = Ui @ Ui.T
    P = 0.5 * (P_src + P_src.T)
    return Phi, Psi, Sig_d, Phi @ P @ Phi.T + Psi @ Sig_d @ Psi.T
