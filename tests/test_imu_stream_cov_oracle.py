"""oracle/imu_stream_cov_oracle.py against the nonlinear oracles it linearises: each step's Jacobian and chains of 1-40
samples against central differences of imu_stream_oracle.propagate, FACTOR's Phi against central differences of
imu_oracle.integrate + predict, the output-pose map against differences of predict_pose's output, and the whole
propagation against a Monte Carlo run of the nonlinear oracle with the discretised reading and bias noise."""
import numpy as np

from oracle import imu_oracle, lie
from oracle import imu_stream_cov_oracle as co
from oracle import imu_stream_oracle as so

NOISE = np.stack([np.diag([1e-4, 2e-4, 1.5e-4]), np.diag([3e-3, 2e-3, 4e-3]), np.diag([1e-7, 2e-7, 1e-7]),
                  np.diag([2e-5, 1e-5, 3e-5])]).reshape(4, 9)


def _state(rng):
    q = rng.normal(size=4)
    q /= np.linalg.norm(q)
    return np.concatenate([q, rng.normal(size=3), rng.normal(size=3) * 0.5, rng.normal(size=3) * 0.02,
                           rng.normal(size=3) * 0.1])


def _st(t, x):
    return [float(t), tuple(x[0:4]), tuple(x[4:7]), tuple(x[7:10]), tuple(x[10:13]), tuple(x[13:16])]


def _plus(st, d):
    """st (so.propagate's layout) moved by d [15] in [dtheta dp dv dbg dba]"""
    t, q, p, v, bg, ba = st
    return [t, tuple(lie.quat_plus(np.array(q), d[0:3])), tuple(np.add(p, d[3:6])), tuple(np.add(v, d[6:9])),
            tuple(np.add(bg, d[9:12])), tuple(np.add(ba, d[12:15]))]


def _minus(a, b):
    """a - b in [dtheta dp dv dbg dba]"""
    dth = lie.logmap(lie.qmul(lie.qconj(np.array(b[1])), np.array(a[1])))
    return np.concatenate([dth] + [np.subtract(a[k], b[k]) for k in range(2, 6)])


def _numeric(f, st0, h=1e-6):
    """central differences of f (st -> st) at st0"""
    y0 = f(st0)
    J = np.zeros((15, 15))
    for k in range(15):
        e = np.zeros(15)
        e[k] = h
        J[:, k] = (_minus(f(_plus(st0, e)), y0) - _minus(f(_plus(st0, -e)), y0)) / (2 * h)
    return J


def _samples(rng, t0, n, equal=False):
    ts = t0 + np.cumsum(rng.uniform(0.003, 0.007, n))
    ts[0] = t0 + 1e-6                                   # right after state_time
    if equal and n > 3:
        ts[2] = ts[1]
        ts[n - 1] = ts[n - 2]
    return [(float(t), tuple(rng.normal(size=3) * 0.8), tuple(np.array([0, 0, 9.8]) + rng.normal(size=3)))
            for t in ts]


def _blockdiag(*blocks):
    out = np.zeros((3 * len(blocks), 3 * len(blocks)))
    for k, b in enumerate(blocks):
        out[3 * k:3 * k + 3, 3 * k:3 * k + 3] = b
    return out


def _close(A, B, rel):
    assert np.max(np.abs(A - B)) <= rel * max(np.max(np.abs(B)), 1.0), np.max(np.abs(A - B))


def test_step_jacobian_matches_central_differences():
    rng = np.random.default_rng(1)
    for _ in range(20):
        st = _st(0.1, _state(rng))
        t, w, a = 0.1 + rng.uniform(0.0, 0.02), rng.normal(size=3), np.array([0, 0, 9.8]) + rng.normal(size=3)
        F, _ = co.step(st, t, w, a, NOISE)
        _close(F, _numeric(lambda s: so.propagate(s, t, w, a), st), 1e-6)


def test_chains_of_1_to_40_samples_match_central_differences():
    rng = np.random.default_rng(2)
    for n in (1, 2, 5, 13, 40):
        x, t0 = _state(rng), 0.5
        smp = _samples(rng, t0, n, equal=True)
        t = smp[-1][0]

        def run(s):
            for (tk, w, a) in smp:
                s = so.propagate(s, tk, w, a)
            return s
        _, _, Phi = co.chain(t0, x, np.zeros((15, 15)), smp, t, NOISE)
        _close(Phi, _numeric(run, _st(t0, x)), 1e-6)


def test_factor_phi_matches_integrate_and_predict():
    rng = np.random.default_rng(3)
    nz = co.noise_blocks(NOISE)
    for _ in range(6):
        src = _state(rng)
        smp = np.array([[t, *w, *a] for t, w, a in _samples(rng, 0.0, 12)])
        t_end = smp[-1, 0] + 0.004

        def f(s):
            x = np.concatenate([s[1], s[2], s[3], s[4], s[5]])
            d = imu_oracle.integrate(smp, t_end, x[10:13], x[13:16], *nz)
            y = co.predict(x, d)
            return _st(0.0, y)
        d = imu_oracle.integrate(smp, t_end, src[10:13], src[13:16], *nz)
        rec = imu_oracle.record(d, src[10:13], src[13:16])
        q_state = co.predict(src, d)[0:4]
        Phi, Psi, Sig_d, _ = co.factor(q_state, rec, np.eye(15))
        _close(Phi, _numeric(f, _st(0.0, src)), 1e-6)
        _close(Sig_d, d["cov"], 1e-8)
        Rs = lie.qmat(src[0:4])
        assert np.allclose(Psi[3:6, 3:6], Rs, atol=1e-12) and np.allclose(Psi[6:9, 6:9], Rs, atol=1e-12)


def test_output_pose_map_matches_differences():
    rng = np.random.default_rng(4)
    for _ in range(10):
        x = _state(rng)
        q_ob = lie.qnormalized(rng.normal(size=4))
        p_ob = rng.normal(size=3)

        def out(s):
            rp = so.qrot(s[1], p_ob)
            return so.qmul(s[1], q_ob), np.add(s[2], rp)
        st0 = _st(0.0, x)
        q0, p0 = out(st0)
        J = np.zeros((6, 15))
        h = 1e-6
        for k in range(15):
            e = np.zeros(15)
            e[k] = h
            (qa, pa), (qb, pb) = out(_plus(st0, e)), out(_plus(st0, -e))
            da = np.concatenate([lie.logmap(lie.qmul(lie.qconj(np.array(q0)), np.array(qa))), pa - p0])
            db = np.concatenate([lie.logmap(lie.qmul(lie.qconj(np.array(q0)), np.array(qb))), pb - p0])
            J[:, k] = (da - db) / (2 * h)
        _close(co.pose_jacobian(x[0:4], q_ob, p_ob), J, 1e-6)


def test_monte_carlo_matches_the_propagated_covariance():
    """20 000 draws of the seed state and of every step's reading and bias noise, through the nonlinear oracle: the
    sample covariance is within 6 % of the oracle's, entry by entry in the oracle's correlation scale"""
    rng = np.random.default_rng(5)
    x, t0 = _state(rng), 0.0
    smp = _samples(rng, t0, 8)
    A = rng.normal(size=(15, 15)) * 1e-3
    P0 = A @ A.T + np.eye(15) * 1e-6
    st_n, P, _ = co.chain(t0, x, P0, smp, smp[-1][0], NOISE)
    cov_w, cov_a, cov_bg, cov_ba = co.noise_blocks(NOISE)
    n = 20000
    x0 = rng.normal(size=(n, 15)) @ np.linalg.cholesky(P0).T
    dts = np.diff([t0] + [tk for tk, _, _ in smp])
    # per step: reading noise (w, a) with the discretised covariance, then the bias walk (bg, ba)
    draws = [rng.normal(size=(n, 12)) @ np.linalg.cholesky(np.kron(np.diag([1 / max(dt, 1e-7)] * 2 + [dt] * 2),
                                                                    np.eye(3)) * _blockdiag(cov_w, cov_a, cov_bg, cov_ba)).T
             for dt in dts]
    err = np.zeros((n, 15))
    for i in range(n):
        s = _plus(_st(t0, x), x0[i])
        for k, (tk, w, a) in enumerate(smp):
            e = draws[k][i]
            s = so.propagate(s, tk, np.add(w, e[0:3]), np.add(a, e[3:6]))
            s[4], s[5] = tuple(np.add(s[4], e[6:9])), tuple(np.add(s[5], e[9:12]))
        err[i] = _minus(s, st_n)
    C = np.cov(err.T)
    d = np.sqrt(np.diag(P))
    assert np.max(np.abs(C - P) / np.outer(d, d)) < 0.06
    assert np.max(np.abs(np.diag(C) / np.diag(P) - 1)) < 0.06


def test_zero_noise_and_no_samples_leave_p_and_outputs_are_symmetric_psd():
    rng = np.random.default_rng(6)
    x = _state(rng)
    A = rng.normal(size=(15, 15))
    P0 = A @ A.T
    _, P, Phi = co.chain(1.0, x, P0, [], 2.0, np.zeros((4, 9)))
    assert np.array_equal(P, P0) and np.array_equal(Phi, np.eye(15))
    smp = _samples(rng, 0.0, 20) + [(0.0, (0, 0, 0), (0, 0, 0))]  # a sample at state_time is not propagated over
    _, P, _ = co.chain(0.0, x, P0, smp, 10.0, NOISE)
    sym = 0.5 * (P + P.T)
    assert np.allclose(P, sym, rtol=0, atol=1e-12 * np.abs(P).max())
    assert np.linalg.eigvalsh(sym).min() > -1e-12 * np.abs(P).max()
    pc = co.pose_cov(x[0:4], sym, lie.qnormalized(rng.normal(size=4)), rng.normal(size=3))
    assert np.linalg.eigvalsh(0.5 * (pc + pc.T)).min() > -1e-12 * np.abs(pc).max()
