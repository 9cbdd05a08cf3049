"""TEST INFRASTRUCTURE (CPU oracle) -- the IMU side of PVIO::Core in Python fp64, with the reference's deques kept
unbounded: Core::track_gyroscope / track_accelerometer (core.cpp:59-107), the frame enqueue of Core::track_camera
(:109-127), Core::track_imu (:129-141), Core::predict_pose (:143-164) recomputed from the latest state for every
reading as the reference does, propagate_state (:32-39), and the prepend rule of FeatureTracker::work
(feature_tracker.cpp:78-84) applied to each released frame against the previously released one.

Arithmetic is scalar, in Eigen's scalar evaluation order without contraction, as csrc/imu_stream.cu computes it:
interpolation w0 + lambda (w - w0) per coefficient, q * v as Eigen's _transformVector, quaternion products in the order
of Eigen's scalar quat_product, normalized() as division by the root of ((x^2 + y^2) + z^2) + w^2, and expmap as the
device's (ba_math.cuh: the stable normalisation by a reciprocal).  sin and cos come from `sincos` (default: the math
library's), so a test can give the device's values.

The lockstep rule of pvio_b200_batch_imu_stream: push() consumes events up to and including the first that releases
a frame."""
import collections
import math

GYROSCOPE, ACCELEROMETER, CAMERA = 0, 1, 2
GRAVITY = 9.80665                                       # PVIO_GRAVITY_NOMINAL, common.h:62


def _sincos(x):
    return math.sin(x), math.cos(x)


def qmul(a, b):
    """Eigen's scalar quat_product, (x, y, z, w)"""
    ax, ay, az, aw = a
    bx, by, bz, bw = b
    w = aw * bw - ax * bx - ay * by - az * bz
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    return (x, y, z, w)


def qrot(q, v):
    """Eigen's _transformVector: uv = 2 (q.vec x v); v + w uv + q.vec x uv"""
    x, y, z, w = q
    tx, ty, tz = 2.0 * (y * v[2] - z * v[1]), 2.0 * (z * v[0] - x * v[2]), 2.0 * (x * v[1] - y * v[0])
    return (v[0] + w * tx + (y * tz - z * ty), v[1] + w * ty + (z * tx - x * tz), v[2] + w * tz + (x * ty - y * tx))


def expmap(u, sincos=_sincos):
    m = max(abs(u[0]), abs(u[1]), abs(u[2]))
    ax, ay, az = u
    if m > 0:
        a0, a1, a2 = u[0] / m, u[1] / m, u[2] / m
        k = 1.0 / (math.sqrt(a0 * a0 + a1 * a1 + a2 * a2) * m)
        ax, ay, az = u[0] * k, u[1] * k, u[2] * k
    angle = math.sqrt(u[0] * u[0] + u[1] * u[1] + u[2] * u[2])
    s, c = sincos(0.5 * angle)
    return (s * ax, s * ay, s * az, c)


def propagate(st, t, w, a, sincos=_sincos):
    """propagate_state: st = [time, q(4), p(3), v(3), bg(3), ba(3)] as tuples; returns the new st"""
    ct, q, p, v, bg, ba = st
    dt = t - ct
    ra = qrot(q, (a[0] - ba[0], a[1] - ba[1], a[2] - ba[2]))
    acc = (0.0 + ra[0], 0.0 + ra[1], -GRAVITY + ra[2])
    hdt = 0.5 * dt * dt
    p = tuple(p[j] + dt * v[j] + hdt * acc[j] for j in range(3))
    v = tuple(v[j] + dt * acc[j] for j in range(3))
    qn = qmul(q, expmap(((w[0] - bg[0]) * dt, (w[1] - bg[1]) * dt, (w[2] - bg[2]) * dt), sincos))
    nrm = math.sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3])
    return [t, tuple(c / nrm for c in qn), p, v, bg, ba]


class Stream:
    """One sequence's Core, IMU side.  Poses are 7-tuples (q xyzw, p); released frames (t, [[t, w xyz, a xyz], ...])."""

    def __init__(self, output_q=(0.0, 0.0, 0.0, 1.0), output_p=(0.0, 0.0, 0.0), sincos=_sincos):
        self.q_ob, self.p_ob = tuple(float(c) for c in output_q), tuple(float(c) for c in output_p)
        self.sincos = sincos
        self.gyroscopes = collections.deque()      # (t, w)
        self.accelerometers = collections.deque()  # (t, a)
        self.frontal_imus = collections.deque()    # (t, w, a)
        self.imus = collections.deque()
        self.frames = collections.deque()          # [t, samples]
        self.latest_state = None                   # (t, state16)
        self.last_frame = None                     # the previously released frame: (t, samples)
        self.released = []

    # ---- the latest state (FeatureTracker::latest_state) -------------------------------------------------------
    def set_state(self, t, state16):
        self.latest_state = (float(t), tuple(float(c) for c in state16))

    def clear_state(self):
        self.latest_state = None

    # ---- Core ---------------------------------------------------------------------------------------------------
    def gyroscope(self, t, x, y, z):
        g = self.gyroscopes
        if self.accelerometers:
            if t < self.accelerometers[0][0]:
                g.clear()
            else:
                while self.accelerometers and t >= self.accelerometers[0][0]:
                    at, a = self.accelerometers[0]
                    t0, w0 = g[0]
                    lam = (at - t0) / (t - t0)
                    w = (w0[0] + lam * (x - w0[0]), w0[1] + lam * (y - w0[1]), w0[2] + lam * (z - w0[2]))
                    self.track_imu(at, w, a)
                    self.accelerometers.popleft()
                if self.accelerometers:
                    while g and g[0][0] < t:
                        g.popleft()
        g.append((t, (x, y, z)))
        return self.predict_pose(t)

    def accelerometer(self, t, x, y, z):
        g = self.gyroscopes
        if g and t >= g[0][0]:
            if t > g[-1][0]:
                while len(g) > 1:
                    g.popleft()
                self.accelerometers.append((t, (x, y, z)))
            elif t == g[-1][0]:
                while len(g) > 1:
                    g.popleft()
                self.track_imu(t, g[0][1], (x, y, z))
            else:
                while t >= g[1][0]:
                    g.popleft()
                (t0, w0), (t1, w1) = g[0], g[1]
                lam = (t - t0) / (t1 - t0)
                w = tuple(w0[j] + lam * (w1[j] - w0[j]) for j in range(3))
                self.track_imu(t, w, (x, y, z))
        return self.predict_pose(t)

    def camera(self, t):
        self.frames.append([t, []])
        return self.predict_pose(t)

    def track_imu(self, t, w, a):
        s = (t, tuple(w), tuple(a))
        self.frontal_imus.append(s)
        self.imus.append(s)
        while self.imus and self.frames:
            if self.imus[0][0] <= self.frames[0][0]:
                self.frames[0][1].append(self.imus.popleft())
            else:
                self.release(*self.frames.popleft())

    def release(self, t, samples):
        """FeatureTracker::work's prepend rule (feature_tracker.cpp:78-84) against the previously released frame"""
        rows = [[s[0], *s[1], *s[2]] for s in samples]
        if self.last_frame is not None and self.last_frame[1]:
            lt, lrows = self.last_frame
            if not rows or rows[0][0] - lt > 1.0e-5:
                rows.insert(0, [lt] + lrows[-1][1:])
        self.last_frame = (t, rows)
        self.released.append((t, rows))

    def predict_pose(self, t):
        if self.latest_state is None:
            return (0.0,) * 7
        ts, x = self.latest_state
        while self.frontal_imus and self.frontal_imus[0][0] <= ts:
            self.frontal_imus.popleft()
        st = [ts, x[0:4], x[4:7], x[7:10], x[10:13], x[13:16]]
        for (it, w, a) in self.frontal_imus:
            if it <= t:
                st = propagate(st, it, w, a, self.sincos)
        q, p = st[1], st[2]
        rp = qrot(q, self.p_ob)
        return (*qmul(q, self.q_ob), p[0] + rp[0], p[1] + rp[1], p[2] + rp[2])

    # ---- lockstep ----------------------------------------------------------------------------------------------
    def push(self, events, state=None, clear=False):
        """pvio_b200_batch_imu_stream for one record: state (t, state16) set or clear before the events; returns
        (poses, n_consumed, released frames)"""
        if clear:
            self.clear_state()
        if state is not None:
            self.set_state(*state)
        poses = []
        self.released = []
        for ev in events:
            kind, t, x, y, z = (float(c) for c in ev)
            if kind == GYROSCOPE:
                poses.append(self.gyroscope(t, x, y, z))
            elif kind == ACCELEROMETER:
                poses.append(self.accelerometer(t, x, y, z))
            elif kind == CAMERA:
                poses.append(self.camera(t))
            else:
                raise ValueError(f"unknown event kind {kind}")
            if self.released:
                break
        return poses, len(poses), self.released
