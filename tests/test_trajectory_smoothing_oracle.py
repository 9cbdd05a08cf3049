"""tests/trajectory_smoothing_oracle.smoothed, the reference of pvio_b200_batch_window_smoothed_trajectory, on synthetic cfg3
factors: its endpoints are the two frames, it is the forward trajectory when the frames agree with the factor, its
cross-covariance is the chain's transition, its Jacobians are the derivatives of its state, its covariance reaches both
frames' and shrinks between them, and a one-sample factor has no smoother."""
import numpy as np
import pytest

from oracle import imu_stream_cov_oracle as sco
from oracle import lie
from oracle import imu_oracle
from oracle import trajectory_oracle as to
from synthetic import synth

import trajectory_smoothing_oracle as tso


def _window(seed=880, N=6):
    w, st, truth = synth.make_cfg3(N=N, M=60, seed=seed)
    frames = np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)
    factors = [(s.copy(), t) for s, t, _, _ in truth.imu_factors]
    return frames, factors, truth.imu_noise


def _times(s, t_end):
    """the factor's first sample, interior points of its first, a middle and its last sample, and t_end"""
    m = len(s)
    knots = list(s[:, 0]) + [t_end]
    ts = [s[0, 0]]
    for j in (0, m // 2, m - 1):
        ts += [knots[j] + f * (knots[j + 1] - knots[j]) for f in (0.25, 0.5)]
    return ts + [knots[m // 2], t_end]


def _consistent(frames, factors, noise):
    """frames k + 1 = predict(frame k, Delta(T)) with equal biases: every residual is 0"""
    out = frames.copy()
    for k, (s, t_end) in enumerate(factors):
        x = out[k]
        out[k + 1] = sco.predict(x, to.delta(s, t_end, x[10:13], x[13:16], noise))
    return out


def _joint(frames, factors, noise, k, seed=5):
    """a joint covariance of frames k, k + 1 as a window's would be: frame k with a covariance, frame k + 1 reached
    through the factor, then both conditioned on a measurement of frame k + 1; the other frames' blocks the identity"""
    rng = np.random.default_rng(seed)
    x = frames[k]
    dT = to.delta(factors[k][0], factors[k][1], x[10:13], x[13:16], noise)
    rec = imu_oracle.record(dict(dT, sqrt_inv_cov=np.eye(15)), x[10:13], x[13:16])
    Phi, Psi, _, _ = sco.factor(sco.predict(x, dT)[0:4], rec, np.eye(15))
    A = rng.normal(size=(15, 15))
    P = A @ A.T * 1e-5 + np.eye(15) * 1e-6
    prior = np.block([[P, P @ Phi.T], [Phi @ P, Phi @ P @ Phi.T + Psi @ dT["cov"] @ Psi.T]])
    H = np.concatenate([np.zeros((15, 15)), np.eye(15)], axis=1)
    Rm = np.eye(15) * 1e-5
    post = prior - prior @ H.T @ np.linalg.solve(H @ prior @ H.T + Rm, H @ prior)
    N = len(frames)
    S = np.eye(15 * N)
    S[15 * k:15 * k + 30, 15 * k:15 * k + 30] = 0.5 * (post + post.T)
    return S


def test_endpoints_are_the_two_frames():
    frames, factors, noise = _window()
    for k, (s, t_end) in enumerate(factors):
        x, x1 = frames[k], frames[k + 1]
        K, _, d, dT = tso.gain(s, s[0, 0], t_end, x[10:13], x[13:16], noise)
        assert np.array_equal(tso.smoothed_state(x, x1, d, dT, K), x), k
        K, _, d, dT = tso.gain(s, t_end, t_end, x[10:13], x[13:16], noise)
        assert np.abs(tso.smoothed_state(x, x1, d, dT, K) - x1).max() < 1e-12, k
        assert np.abs(tso.residual(x, x1, dT)).max() > 1e-6        # the synthetic frames do not agree with the factor


def test_zero_residual_gives_the_forward_trajectory():
    frames, factors, noise = _window(seed=881)
    frames = _consistent(frames, factors, noise)
    ts = [t for s, t_end in factors for t in _times(s, t_end)[:-1]]
    fr, st, _ = to.trajectory(ts, frames, factors, noise)
    frs, sts, _ = tso.smoothed(ts, frames, factors, noise)
    assert np.array_equal(fr, frs)
    assert np.abs(st - sts).max() < 1e-12


def _A(q, smp, dt, bg, ba):
    """imu_oracle.integrate's 9 x 9 A of one step, written out"""
    w, a = smp[1:4] - bg, smp[4:7] - ba
    Rd = lie.qmat(q)
    A = np.eye(9)
    A[0:3, 0:3] = lie.qmat(lie.qconj(lie.expmap(w * dt)))
    A[6:9, 0:3] = -dt * Rd @ lie.hat(a)
    A[3:6, 0:3] = -0.5 * dt * dt * Rd @ lie.hat(a)
    A[3:6, 6:9] = dt * np.eye(3)
    return A


def test_augmented_cross_covariance_is_the_transition_product():
    frames, factors, noise = _window(seed=882)
    s, t_end = factors[1]
    bg, ba = frames[1][10:13], frames[1][13:16]
    knots = list(s[:, 0]) + [t_end]
    for t in _times(s, t_end) + [t_end + 4e-6]:
        X = tso.cross_cov(s, t, t_end, bg, ba, noise)
        Phi = np.eye(15)
        if t > t_end:
            dT = to.delta(s, t_end, bg, ba, noise)
            Phi[0:9, 0:9] = _A(dT["dq"], s[-1], t - t_end, bg, ba)
            ref = Phi @ dT["cov"]
        else:
            d = to.delta(s, t, bg, ba, noise)
            j = int(np.flatnonzero(s[:, 0] <= t)[-1])
            P9 = _A(d["dq"], s[j], knots[j + 1] - t, bg, ba)
            for i in range(j + 1, len(s)):
                P9 = _A(to.delta(s, knots[i], bg, ba, noise)["dq"], s[i], knots[i + 1] - knots[i], bg, ba) @ P9
            Phi[0:9, 0:9] = P9
            ref = d["cov"] @ Phi.T
        assert np.abs(X - ref).max() <= 1e-12 * max(np.abs(ref).max(), 1e-300), t


def _corrected(d, dbg, dba):
    """Delta at biases moved by (dbg, dba), to first order through its bias Jacobians"""
    return dict(d, dq=lie.qmul(d["dq"], lie.expmap(d["dq_dbg"] @ dbg)),
                dp=d["dp"] + d["dp_dbg"] @ dbg + d["dp_dba"] @ dba,
                dv=d["dv"] + d["dv_dbg"] @ dbg + d["dv_dba"] @ dba)


def _plus(x, e):
    y = np.array(x, dtype=np.float64)
    y[0:4] = lie.qmul(x[0:4], lie.expmap(e[0:3]))
    y[4:16] = x[4:16] + e[3:15]
    return y


def _minus(y, x):
    return np.concatenate([lie.logmap(lie.qmul(lie.qconj(x[0:4]), y[0:4])), y[4:16] - x[4:16]])


def test_jacobians_match_finite_differences():
    frames, factors, noise = _window(seed=883)
    k = 2
    s, t_end = factors[k]
    x, x1 = frames[k], frames[k + 1]
    for t in _times(s, t_end)[1:] + [t_end + 4e-6]:
        K, _, d, dT = tso.gain(s, t, t_end, x[10:13], x[13:16], noise)
        Jk, Jk1, _ = tso.jacobians(x, x1, d, dT, K)

        def f(xa, xb):
            db = xa[10:16] - x[10:16]
            return tso.smoothed_state(xa, xb, _corrected(d, db[0:3], db[3:6]), _corrected(dT, db[0:3], db[3:6]), K)

        y0 = f(x, x1)
        scale = max(np.abs(Jk).max(), np.abs(Jk1).max())     # at t_end J_k is 0 up to rounding
        for which, J in ((0, Jk), (1, Jk1)):
            num = np.zeros((15, 15))
            for c in range(15):
                h = 1e-6
                e = np.zeros(15)
                e[c] = h
                if which == 0:
                    yp, ym = f(_plus(x, e), x1), f(_plus(x, -e), x1)
                else:
                    yp, ym = f(x, _plus(x1, e)), f(x, _plus(x1, -e))
                num[:, c] = (_minus(yp, y0) - _minus(ym, y0)) / (2 * h)
            assert np.abs(num - J).max() <= 1e-6 * scale, (t, which, np.abs(num - J).max() / scale)


@pytest.mark.parametrize("k", [0, 3])
def test_covariance_reaches_both_frames_and_shrinks_between(k):
    frames, factors, noise = _window(seed=884)
    Sj = _joint(frames, factors, noise, k)
    s, t_end = factors[k]
    ts = _times(s, t_end)
    # factor k's own arithmetic at t_end, which factor_of gives to factor k + 1
    fac = [(None, f[1]) if i != k else f for i, f in enumerate(factors)]
    fr, st, cov = tso.smoothed(ts, frames, fac, noise, Sj)
    assert np.all(fr == k)
    Sk, Sk1 = Sj[15 * k:15 * k + 15, 15 * k:15 * k + 15], Sj[15 * k + 15:15 * k + 30, 15 * k + 15:15 * k + 30]
    assert np.abs(cov[0] - Sk).max() <= 1e-9 * np.abs(Sk).max()
    assert np.abs(cov[-1] - Sk1).max() <= 1e-9 * np.abs(Sk1).max()
    Sig = np.zeros((len(frames), 15, 15))
    Sig[k] = Sk
    _, _, fwd = to.trajectory(ts, frames, fac, noise, Sig)
    for i in range(1, len(ts) - 1):
        assert np.all(np.isfinite(cov[i]))
        assert np.trace(cov[i]) <= np.trace(fwd[i]), (i, np.trace(cov[i]), np.trace(fwd[i]))


def test_one_sample_factor_has_no_smoother():
    frames, factors, noise = _window(seed=885)
    s, t_end = factors[1]
    factors[1] = (s[:1].copy(), t_end)
    ts = [s[0, 0], 0.5 * (s[0, 0] + t_end), factors[2][0][0, 0]]
    fr, st, cov = tso.smoothed(ts, frames, factors, noise, np.eye(15 * len(frames)))
    assert list(fr) == [-2, -2, 2]
    assert np.all(st[:2] == 0.0) and np.isnan(cov[:2]).all() and np.isfinite(cov[2]).all()
