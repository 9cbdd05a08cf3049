"""TEST INFRASTRUCTURE (50-digit judge) -- the forward state of pvio_b200_batch_window_trajectory restated in mpmath:
PreIntegrator's prefix integration of q, p and v over the samples at or before t, the last one up to t
(imu_oracle.integrate's recurrence), then PreIntegrator::predict (imu_stream_cov_oracle.predict).  No numpy on the
arithmetic path: the inputs are fp64 numbers read as exact binary fractions and every operation runs at 50 digits, so
the result is the exact value of the definition to far below fp64 rounding.  The inv_dt clamp (1 / max(dt, 1e-7))
scales only the covariance, which this judge does not compute: q, p and v of a step over dt < 1e-7 are those of the
step over dt itself.  When the device and trajectory_oracle disagree, this says which one is wrong."""
import mpmath as mp

mp.mp.dps = 50
_G = (mp.mpf(0), mp.mpf(0), -mp.mpf("9.80665"))


def _f(x):
    return mp.mpf(float(x))


def qmul(a, b):
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    return (aw * bx + ax * bw + ay * bz - az * by, aw * by + ay * bw + az * bx - ax * bz,
            aw * bz + az * bw + ax * by - ay * bx, aw * bw - ax * bx - ay * by - az * bz)


def qrot(q, v):
    """q v q^-1"""
    x, y, z, w = qmul(qmul(q, (v[0], v[1], v[2], mp.mpf(0))), (-q[0], -q[1], -q[2], q[3]))
    return (x, y, z)


def expmap(u):
    a = mp.sqrt(u[0] ** 2 + u[1] ** 2 + u[2] ** 2)
    if a == 0:
        return (mp.mpf(0), mp.mpf(0), mp.mpf(0), mp.mpf(1))
    s = mp.sin(a / 2) / a
    return (s * u[0], s * u[1], s * u[2], mp.cos(a / 2))


def normalized(q):
    n = mp.sqrt(sum(c * c for c in q))
    return tuple(c / n for c in q)


def delta(samples, t, bg, ba):
    """(T, dq, dp, dv) of the samples s with s.t <= t, the last one integrated up to t"""
    t = _f(t)
    pre = [[_f(c) for c in row] for row in samples if float(row[0]) <= float(t)]
    bg, ba = [_f(c) for c in bg], [_f(c) for c in ba]
    dq, dp, dv, T = (mp.mpf(0), mp.mpf(0), mp.mpf(0), mp.mpf(1)), [mp.mpf(0)] * 3, [mp.mpf(0)] * 3, mp.mpf(0)
    for i, s in enumerate(pre):
        dt = (pre[i + 1][0] if i + 1 < len(pre) else t) - s[0]
        w = [s[1 + c] - bg[c] for c in range(3)]
        a = qrot(dq, [s[4 + c] - ba[c] for c in range(3)])
        dp = [dp[c] + dt * dv[c] + dt * dt / 2 * a[c] for c in range(3)]
        dv = [dv[c] + dt * a[c] for c in range(3)]
        dq = normalized(qmul(dq, expmap([w[c] * dt for c in range(3)])))
        T += dt
    return T, dq, dp, dv


def predict(x, d):
    """PreIntegrator::predict from the state x [16] through d = (T, dq, dp, dv): [q p v bg ba]"""
    T, dq, dp, dv = d
    q, p, v = [_f(c) for c in x[0:4]], [_f(c) for c in x[4:7]], [_f(c) for c in x[7:10]]
    rp, rv = qrot(q, dp), qrot(q, dv)
    vn = [v[c] + _G[c] * T + rv[c] for c in range(3)]
    pn = [p[c] + _G[c] * T * T / 2 + v[c] * T + rp[c] for c in range(3)]
    return list(qmul(q, dq)) + pn + vn + [_f(c) for c in x[10:16]]


def state(x, samples, t):
    """the forward state at t from frame state x through its factor's samples, as a list of 16 floats"""
    return [float(c) for c in predict(x, delta(samples, t, x[10:13], x[13:16]))]
