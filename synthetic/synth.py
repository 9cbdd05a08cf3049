"""Synthetic sliding windows for the BASELINE.json configs (SURVEY.md 8d).

No datasets exist on the box, so each config reproduces the calibration and factor mix
of the named dataset (config/euroc.yaml, config/tum-vi.yaml in the reference), not its
images.  Everything is seeded; seed 648 is the reference's own RNG seed (config.cpp:91-93).
Returns (Window, State initial_guess, State truth).
"""
import numpy as np
from pvio_b200.window import Window, State
from . import so3

EUROC = dict(
    K=(458.654, 457.296, 367.215, 248.375), size=(752, 480),
    q_bc=np.array([-7.7071797555374275e-03, 1.0499323370587278e-02, 7.0175280029197162e-01, 7.1230146066895372e-01]),
    p_bc=np.array([-0.0216401454975, -0.064676986768, 0.00981073058949]),
    noise_px2=0.5, cov_g=2.8791302399999997e-08, cov_a=4.0e-6, cov_bg=3.7608844899999997e-10, cov_ba=9.0e-6)
TUMVI = dict(
    K=(190.97847715128717, 190.9733070521226, 254.93170605935475, 256.8974428996504), size=(512, 512),
    q_bc=np.array([-0.013272, -0.694726, 0.719112, 0.007648]),
    p_bc=np.array([0.04536566, -0.071996, -0.04478181]),
    noise_px2=0.5, cov_g=2.56e-08, cov_a=7.84e-6, cov_bg=4.84e-10, cov_ba=7.396e-07)

GRAVITY = np.array([0.0, 0.0, -9.80665])
# camera x(right) y(down) z(forward) -> world -y, -z, +x
R_WC0 = np.array([[0., 0., 1.], [-1., 0., 0.], [0., -1., 0.]])


def _base_window(cal, N, use_inertial):
    w = Window(N=N, use_inertial=use_inertial)
    w.cam_q_cs = so3.qnormalize(cal['q_bc'].copy())
    w.cam_p_cs = cal['p_bc'].copy()
    fx, fy = cal['K'][0], cal['K'][1]
    s = np.sqrt(cal['noise_px2'])
    w.sqrt_inv_cov = np.array([[fx / s, 0.0], [0.0, fy / s]])   # core/core.cpp:112-116
    w.K_fx, w.K_fy = fx, fy
    w.frame_fixed = np.zeros(N, dtype=np.uint8)
    return w


def _cam_pose(qb, pb, w):
    return so3.qmul(qb, w.cam_q_cs), pb + so3.qrot(qb, w.cam_p_cs)


def _project(qb, pb, w, x):
    qc, pc = _cam_pose(qb, pb, w)
    y = so3.qrot(so3.qconj(qc), x - pc)
    return y[..., :2] / y[..., 2:3], y[..., 2]


def _in_view(z, depth, cal, margin=20.0):
    fx, fy, cx, cy = cal['K']
    W, H = cal['size']
    u, v = z[..., 0] * fx + cx, z[..., 1] * fy + cy
    return (depth > 0.5) & (u > margin) & (u < W - margin) & (v > margin) & (v < H - margin)


def _sample_landmark(rng, cal, w, q_t, p_t, frames, dmin=2.0, dmax=10.0):
    """A world point uniform in depth inside the anchor's field of view and visible in
    all `frames` (anchor first)."""
    fx, fy, cx, cy = cal['K']
    W, H = cal['size']
    a = frames[0]
    qc, pc = _cam_pose(q_t[a], p_t[a], w)
    for _ in range(1000):
        u, v = rng.uniform(25, W - 25), rng.uniform(25, H - 25)
        d = rng.uniform(dmin, dmax)
        zr = np.array([(u - cx) / fx, (v - cy) / fy])
        x = so3.qrot(qc, np.array([zr[0], zr[1], 1.0]) * d) + pc
        ok = True
        for f in frames[1:]:
            z, dep = _project(q_t[f], p_t[f], w, x)
            if not _in_view(z, dep, cal):
                ok = False
                break
        if ok:
            return x, zr, d
    raise RuntimeError("could not place a landmark")


def _depth_ranges(M, depth_mix):
    """Per-landmark (dmin, dmax) of a depth mixture [(fraction, dmin, dmax), ...]: the groups take consecutive
    landmark indices in proportion to their fractions (no random draw, so the mixture leaves the RNG stream alone).
    None: every landmark at 2-10 m."""
    if depth_mix is None:
        return [(2.0, 10.0)] * M
    fr = np.array([g[0] for g in depth_mix], dtype=float)
    edges = np.rint(np.cumsum(fr) / fr.sum() * M)
    return [depth_mix[min(int(np.searchsorted(edges, l, side='right')), len(depth_mix) - 1)][1:] for l in range(M)]


# 70 % of the landmarks at 2-10 m, 20 % at 20-60 m, 10 % at 60-400 m (beyond the post-pass's 50 m: rejected)
DEPTH_MIX_OUTDOOR = ((0.7, 2.0, 10.0), (0.2, 20.0, 60.0), (0.1, 60.0, 400.0))


def _fill_observations(rng, cal, w, q_t, p_t, lm_frames, depth_mix=None):
    """lm_frames: per-landmark sorted frame lists (anchor first).  Adds pixel noise."""
    fx, fy = cal['K'][0], cal['K'][1]
    s = np.sqrt(cal['noise_px2'])
    M = len(lm_frames)
    anchors, zrefs, begins, of, oz, rho_t = [], [], [0], [], [], []
    for frames, (dmin, dmax) in zip(lm_frames, _depth_ranges(M, depth_mix)):
        x, zr, d = _sample_landmark(rng, cal, w, q_t, p_t, frames, dmin, dmax)
        anchors.append(frames[0])
        zrefs.append(zr + rng.normal(0, s, 2) / np.array([fx, fy]))
        for f in frames[1:]:
            z, _ = _project(q_t[f], p_t[f], w, x)
            of.append(f)
            oz.append(z + rng.normal(0, s, 2) / np.array([fx, fy]))
        begins.append(len(of))
        rho_t.append(1.0 / d)
    w.M, w.K = M, len(of)
    w.lm_anchor = np.array(anchors, dtype=np.int32)
    w.lm_z_ref = np.array(zrefs).reshape(M, 2)
    w.lm_obs_begin = np.array(begins, dtype=np.int32)
    w.obs_frame = np.array(of, dtype=np.int32)
    w.obs_z = np.array(oz).reshape(len(of), 2)
    w.lm_in_victim = np.array([1 if fr[0] == 0 else 0 for fr in lm_frames], dtype=np.uint8)
    return np.array(rho_t)


def _perturb(rng, w, truth, sig_p=0.01, sig_th=np.deg2rad(0.5), sig_rho=0.05, sig_v=0.02,
             sig_bg=1e-4, sig_ba=5e-3):
    st = truth.copy()
    for f in range(w.N):
        if w.frame_fixed[f]:
            continue
        st.q[f] = so3.qnormalize(so3.qmul(truth.q[f], so3.qexp(rng.normal(0, sig_th, 3))))
        st.p[f] = truth.p[f] + rng.normal(0, sig_p, 3)
    if w.use_inertial:
        st.v = truth.v + rng.normal(0, sig_v, truth.v.shape)
        st.bg = truth.bg + rng.normal(0, sig_bg, truth.bg.shape)
        st.ba = truth.ba + rng.normal(0, sig_ba, truth.ba.shape)
    st.rho = truth.rho * (1.0 + rng.normal(0, sig_rho, truth.rho.shape))
    return st


def make_cfg2(seed=648, N=10, M=500, staggered=False, cal=EUROC, depth_mix=None, baseline=1.0):
    """BASELINE config 2: N keyframes x M landmarks, reprojection-only GN, frames 0 and 1
    FF_FIX_POSE (gauge + scale), every landmark anchored in frame 0 and seen in all frames
    (K_res = M(N-1)).  staggered=True is config 2b: landmark l first observed in frame
    l mod 5, last in frame N-1.  depth_mix: landmark depths (see _depth_ranges); baseline
    scales the frame positions (1e-3: a camera hovering at start-up)."""
    rng = np.random.default_rng(seed)
    w = _base_window(cal, N, use_inertial=False)
    w.frame_fixed[:2] = 1
    # arc: 0.25 m spacing sideways (camera x), <= 10 deg total yaw
    q_t, p_t = np.zeros((N, 4)), np.zeros((N, 3))
    R_wb0 = R_WC0 @ so3.qmat(w.cam_q_cs).T
    for k in range(N):
        yaw = np.deg2rad(10.0) * k / max(N - 1, 1)
        Rz = np.array([[np.cos(yaw), -np.sin(yaw), 0.], [np.sin(yaw), np.cos(yaw), 0.], [0., 0., 1.]])
        q_t[k] = so3.mat2quat(Rz @ R_wb0)
        p_t[k] = baseline * np.array([0.3 * np.sin(yaw) * 4.0, -0.25 * k, 0.02 * np.sin(0.7 * k)])
    lm_frames = []
    for l in range(M):
        a = (l % min(5, N - 1)) if staggered else 0
        lm_frames.append(list(range(a, N)))
    rho_t = _fill_observations(rng, cal, w, q_t, p_t, lm_frames, depth_mix)
    truth = State(q_t, p_t, np.zeros((N, 3)), np.zeros((N, 3)), np.zeros((N, 3)), rho_t)
    w.validate()
    return w, _perturb(rng, w, truth), truth


def _trajectory(t):
    """Smooth body trajectory: position, velocity, acceleration (world), rotation vector
    theta(t) and its rate, for orientation R_wb(t) = R_wb0 Exp(theta(t))."""
    w1 = 0.9
    p = np.array([0.6 * np.sin(0.5 * w1 * t), -0.9 * t + 0.2 * np.sin(w1 * t), 0.15 * np.sin(1.3 * w1 * t)])
    v = np.array([0.3 * w1 * np.cos(0.5 * w1 * t), -0.9 + 0.2 * w1 * np.cos(w1 * t),
                  0.195 * w1 * np.cos(1.3 * w1 * t)])
    a = np.array([-0.15 * w1 * w1 * np.sin(0.5 * w1 * t), -0.2 * w1 * w1 * np.sin(w1 * t),
                  -0.2535 * w1 * w1 * np.sin(1.3 * w1 * t)])
    th = np.array([0.06 * np.sin(1.1 * t), 0.05 * np.sin(0.8 * t + 0.3), 0.12 * np.sin(0.6 * t)])
    thd = np.array([0.066 * np.cos(1.1 * t), 0.04 * np.cos(0.8 * t + 0.3), 0.072 * np.cos(0.6 * t)])
    return p, v, a, th, thd


def synth_prior(rng, w, st, n):
    """A steady-state marginalisation prior over frames 0..n-1: S = sqrt(Lambda) V^T of a
    synthetic SPD information matrix with realistic per-component scales and mild
    correlations, linearised at a point close to the current guess
    (shape of what bundle_adjustor.cpp:583-597 produces)."""
    d = 15 * n
    sc = np.tile(np.concatenate([np.full(3, 300.0), np.full(3, 150.0), np.full(3, 60.0),
                                 np.full(3, 8.0e3), np.full(3, 150.0)]), n)
    L = np.triu(rng.normal(0, 0.08, (d, d)), 1) + np.eye(d)
    L = L * sc[None, :]
    Lam = L.T @ L
    lam, V = np.linalg.eigh(Lam)
    S = np.sqrt(np.maximum(lam, 0))[:, None] * V.T
    w.n_prior = n
    w.prior_frames = np.arange(n, dtype=np.int32)
    w.prior_S = S
    w.prior_e = rng.normal(0, 0.3, d)
    w.prior_q0 = np.array([so3.qnormalize(so3.qmul(st.q[i], so3.qexp(rng.normal(0, 2e-3, 3)))) for i in range(n)])
    w.prior_p0 = st.p[:n] + rng.normal(0, 3e-3, (n, 3))
    w.prior_v0 = st.v[:n] + rng.normal(0, 5e-3, (n, 3))
    w.prior_bg0 = st.bg[:n] + rng.normal(0, 2e-5, (n, 3))
    w.prior_ba0 = st.ba[:n] + rng.normal(0, 1e-3, (n, 3))


def gauge_prior(w, st):
    """The first-window prior of core/sliding_window_tracker.cpp:100-112: sqrt-information
    1e15 on the pose of frame 0, zero elsewhere, over frames 0..N-2."""
    n = w.N - 1
    d = 15 * n
    S = np.zeros((d, d))
    S[0:3, 0:3] = 1.0e15 * np.eye(3)
    S[3:6, 3:6] = 1.0e15 * np.eye(3)
    w.n_prior = n
    w.prior_frames = np.arange(n, dtype=np.int32)
    w.prior_S = S
    w.prior_e = np.zeros(d)
    w.prior_q0, w.prior_p0 = st.q[:n].copy(), st.p[:n].copy()
    w.prior_v0, w.prior_bg0, w.prior_ba0 = st.v[:n].copy(), st.bg[:n].copy(), st.ba[:n].copy()


def make_cfg3(seed=649, N=9, M=300, cal=EUROC, planes=0, tracks_per_plane=40, prior='synthetic',
              kf_dt=0.25, imu_hz=200.0, depth_mix=None, plane_noise_px=None, plane_range=(1.0, 15.0)):
    """BASELINE config 3 (planes=0) / config 4 (planes=2, TUM-VI calibration): full window
    with reprojection + IMU pre-integration + marginalisation prior (+ plane factors).
    depth_mix: landmark depths (see _depth_ranges).  plane_noise_px: the keypoint noise (px) of the plane tracks,
    None: the calibration's; plane_range: the distances from the first camera at which plane tracks are drawn"""
    rng = np.random.default_rng(seed)
    w = _base_window(cal, N, use_inertial=True)
    R_wb0 = R_WC0 @ so3.qmat(w.cam_q_cs).T
    q_t, p_t, v_t = np.zeros((N, 4)), np.zeros((N, 3)), np.zeros((N, 3))
    for k in range(N):
        p, v, _, th, _ = _trajectory(k * kf_dt)
        q_t[k] = so3.mat2quat(R_wb0 @ so3.qmat(so3.qexp(th)))
        p_t[k], v_t[k] = p, v
    bg_t = np.tile(rng.normal(0, 2e-3, 3), (N, 1)) + rng.normal(0, 1e-5, (N, 3))
    ba_t = np.tile(rng.normal(0, 2e-2, 3), (N, 1)) + rng.normal(0, 1e-3, (N, 3))
    # landmarks: truncated-geometric track lengths on [2, N]
    lm_frames = []
    for l in range(M):
        L = 2
        while L < N and rng.random() < 0.72:
            L += 1
        a = int(rng.integers(0, N - L + 1))
        if l < M // 3:
            a = 0               # plenty of victim-frame tracks for the marginaliser
            L = min(L, N)
        lm_frames.append(list(range(a, a + L)))
    rho_t = _fill_observations(rng, cal, w, q_t, p_t, lm_frames, depth_mix)
    truth = State(q_t, p_t, v_t, bg_t, ba_t, rho_t)
    st = _perturb(rng, w, truth)
    # IMU factors: synthetic gyro/accel at imu_hz, pre-integrated at the GUESS biases
    # (bundle_adjustor.cpp:224 re-integrates with frame_i's current bg/ba)
    n_imu = N - 1
    w.n_imu = n_imu
    w.imu_frame_i = np.arange(0, N - 1, dtype=np.int32)
    w.imu_frame_j = np.arange(1, N, dtype=np.int32)
    recs = []
    raw_factors = []            # (samples [K][7], t_end, bg, ba) per factor, for the device pre-integrator
    dt = 1.0 / imu_hz
    for j in range(1, N):
        pre = so3.PreIntegrator(cal['cov_g'], cal['cov_a'], cal['cov_bg'], cal['cov_ba'])
        t0, t1 = (j - 1) * kf_dt, j * kf_dt
        ns = int(round((t1 - t0) * imu_hz))
        for s in range(ns):
            t = t0 + s * dt
            _, _, a, th, thd = _trajectory(t + 0.5 * dt)
            Rwb = R_wb0 @ so3.qmat(so3.qexp(th))
            w_true = so3.right_jacobian(th) @ thd
            a_true = Rwb.T @ (a - GRAVITY)
            gyro = w_true + bg_t[j - 1] + rng.normal(0, np.sqrt(cal['cov_g'] * imu_hz), 3)
            acc = a_true + ba_t[j - 1] + rng.normal(0, np.sqrt(cal['cov_a'] * imu_hz), 3)
            pre.data.append((t, gyro, acc))
        recs.append(pre.integrate(t1, st.bg[j - 1], st.ba[j - 1]))
        raw_factors.append((np.array([np.r_[t_, g_, a_] for t_, g_, a_ in pre.data]), t1, st.bg[j - 1].copy(), st.ba[j - 1].copy()))
    truth.imu_factors = raw_factors
    truth.imu_noise = tuple(np.eye(3) * cal[k] for k in ('cov_g', 'cov_a', 'cov_bg', 'cov_ba'))
    w.imu_dt = np.array([r['dt'] for r in recs])
    w.imu_dq = np.array([r['dq'] for r in recs])
    w.imu_dp = np.array([r['dp'] for r in recs])
    w.imu_dv = np.array([r['dv'] for r in recs])
    w.imu_sqrt_inv_cov = np.array([r['sqrt_inv_cov'] for r in recs])
    for k in ('dq_dbg', 'dp_dbg', 'dp_dba', 'dv_dbg', 'dv_dba'):
        setattr(w, 'imu_' + k, np.array([r[k] for r in recs]))
    w.imu_bg0 = st.bg[:N - 1].copy()
    w.imu_ba0 = st.ba[:N - 1].copy()
    if prior == 'synthetic':
        synth_prior(rng, w, st, N - 1)
    elif prior == 'gauge':
        st.q[0], st.p[0] = truth.q[0].copy(), truth.p[0].copy()   # gravity-aligned first pose
        gauge_prior(w, st)
    # planes: floor (z = -1.4) and a wall ahead (x = 7), plane tracks seen in 2..N frames
    if planes > 0:
        fx, fy = cal['K'][0], cal['K'][1]
        s = np.sqrt(cal['noise_px2']) if plane_noise_px is None else plane_noise_px
        defs = [(np.array([0., 0., 1.]), -1.4), (np.array([1., 0., 0.]), 7.0)][:planes]
        w.n_planes = len(defs)
        w.plane_normal = np.array([d[0] for d in defs])
        w.plane_distance = np.array([d[1] for d in defs])
        w.plane_sqrt_inv_cov = np.sqrt(1.0 / 1.0e-4)
        pt_plane, begins, pf, pz = [], [0], [], []
        for pi, (nrm, dist) in enumerate(defs):
            cnt = 0
            while cnt < tracks_per_plane:
                L = int(rng.integers(2, N + 1))
                a = int(rng.integers(0, N - L + 1))
                frames = list(range(a, a + L))
                qc, pc = _cam_pose(q_t[a], p_t[a], w)
                u, v = rng.uniform(25, cal['size'][0] - 25), rng.uniform(25, cal['size'][1] - 25)
                ray = so3.qrot(qc, np.array([(u - cal['K'][2]) / fx, (v - cal['K'][3]) / fy, 1.0]))
                den = nrm @ ray
                if abs(den) < 1e-3:
                    continue
                lam = (dist - nrm @ pc) / den
                if lam < plane_range[0] or lam > plane_range[1]:
                    continue
                x = pc + lam * ray
                zs, ok = [], True
                for f in frames:
                    z, dep = _project(q_t[f], p_t[f], w, x)
                    if not _in_view(z, dep, cal):
                        ok = False
                        break
                    zs.append(z + rng.normal(0, s, 2) / np.array([fx, fy]))
                if not ok:
                    continue
                pt_plane.append(pi)
                pf += frames
                pz += zs
                begins.append(len(pf))
                cnt += 1
        w.n_ptracks = len(pt_plane)
        w.pt_plane = np.array(pt_plane, dtype=np.int32)
        w.pt_obs_begin = np.array(begins, dtype=np.int32)
        w.pt_obs_frame = np.array(pf, dtype=np.int32)
        w.pt_obs_z = np.array(pz).reshape(len(pf), 2)
    w.validate()
    return w, st, truth


def make_cfg4(seed=650, **kw):
    return make_cfg3(seed=seed, cal=TUMVI, planes=2, **kw)


# ------------------------------------------------------------------ hard windows: post-transforms
# Each takes a generated (Window, State guess, State truth) and returns new copies; the inputs are left alone.
def _copies(w, st, truth):
    import copy
    return copy.deepcopy(w), st.copy(), copy.deepcopy(truth)


def _px_offsets(rng, n, px, fx, fy):
    """n displacements of uniform direction and a length uniform in px = (lo, hi) pixels, in normalised coordinates."""
    ang = rng.uniform(0.0, 2.0 * np.pi, n)
    r = rng.uniform(px[0], px[1], n)
    return np.stack([r * np.cos(ang) / fx, r * np.sin(ang) / fy], axis=1)


def with_outliers(w, st, truth, seed=0, frac=0.07, px=(15.0, 300.0), n_tracks=2):
    """Mismatched keypoints: a fraction `frac` of the observations displaced by px pixels, and n_tracks whole tracks
    with a wrong keypoint (a different one) in every observing frame.  Returns (w, st, truth, outlier observation mask)."""
    w, st, truth = _copies(w, st, truth)
    rng = np.random.default_rng(seed)
    bad = np.zeros(w.K, dtype=bool)
    bad[rng.choice(w.K, int(round(frac * w.K)), replace=False)] = True
    nobs = np.diff(w.lm_obs_begin)
    for l in rng.choice(np.nonzero(nobs >= 2)[0], n_tracks, replace=False):
        bad[w.lm_obs_begin[l]:w.lm_obs_begin[l + 1]] = True
    w.obs_z = w.obs_z.copy()
    w.obs_z[bad] += _px_offsets(rng, int(bad.sum()), px, w.K_fx, w.K_fy)
    return w, st, truth, bad


def general_sqrt_info(w, sigma_px=None, ratio=1.6, corr=0.55, angle=0.5):
    """A full 2x2 square-root information of correlated keypoint noise: the upper Cholesky factor U of
    Lambda = Sigma^-1 (Sigma: sigma_px and ratio * sigma_px pixel deviations with correlation corr) turned by `angle`,
    W = Rot(angle) U.  W^T W = Lambda as for U, but W is not symmetric and its two off-diagonals are non-zero and
    different, so a transposed or swapped entry changes every residual."""
    if sigma_px is None:
        sigma_px = w.K_fx / w.sqrt_inv_cov[0, 0]
    sx, sy = sigma_px / w.K_fx, ratio * sigma_px / w.K_fy
    Sig = np.array([[sx * sx, corr * sx * sy], [corr * sx * sy, sy * sy]])
    U = np.linalg.cholesky(np.linalg.inv(Sig)).T
    c, s = np.cos(angle), np.sin(angle)
    return np.array([[c, -s], [s, c]]) @ U


def with_general_w(w, st, truth, **kw):
    w, st, truth = _copies(w, st, truth)
    w.sqrt_inv_cov = general_sqrt_info(w, **kw)
    return w, st, truth


def with_cauchy(w, st, truth, a):
    w, st, truth = _copies(w, st, truth)
    w.cauchy_a = float(a)
    return w, st, truth


FAR_OFFSET = np.array([4000.0, -3000.0, 120.0])      # 5.0 km from the world origin


def with_offset(w, st, truth, offset=FAR_OFFSET):
    """The whole window translated by `offset` (a long sequence far from its start): frame positions of the guess and
    the truth, the prior's linearisation point, and each plane's distance (n.x = d becomes n.x = d + n.offset).  The
    inverse-depth landmarks move with their anchors; IMU factors are translation invariant.  The plane factors are not:
    the reference's functor regularises its point towards n.x = -d and measures n.x - d, so their cost changes."""
    w, st, truth = _copies(w, st, truth)
    o = np.asarray(offset, dtype=float)
    st.p = st.p + o
    truth.p = truth.p + o
    if w.n_prior > 0:
        w.prior_p0 = w.prior_p0 + o
    if w.n_planes > 0:
        w.plane_distance = w.plane_distance + w.plane_normal @ o
    return w, st, truth


def _anchor_point(w, st, l, rho):
    a = int(w.lm_anchor[l])
    qc, pc = _cam_pose(st.q[a], st.p[a], w)
    return so3.qrot(qc, np.array([w.lm_z_ref[l][0], w.lm_z_ref[l][1], 1.0])) / rho + pc


def with_rejected_landmarks(w, st, truth, seed=0, n_behind=3, n_far=3, far=(55.0, 90.0)):
    """Landmarks the post-pass rejects: n_behind with an inverse depth of the wrong sign in the guess (behind the
    anchor camera), n_far moved to far = (lo, hi) metres along their anchor ray, observations re-projected from the truth
    poses with their pixel noise kept.  Returns (w, st, truth, behind indices, far indices)."""
    w, st, truth = _copies(w, st, truth)
    rng = np.random.default_rng(seed)
    nobs = np.diff(w.lm_obs_begin)
    pick = rng.choice(np.nonzero(nobs >= 1)[0], n_behind + n_far, replace=False)
    behind, farl = np.sort(pick[:n_behind]), np.sort(pick[n_behind:])
    st.rho[behind] = -st.rho[behind]
    w.obs_z = w.obs_z.copy()
    for l in farl:
        d = rng.uniform(*far)
        x_old, x_new = _anchor_point(w, truth, l, truth.rho[l]), _anchor_point(w, truth, l, 1.0 / d)
        for k in range(int(w.lm_obs_begin[l]), int(w.lm_obs_begin[l + 1])):
            f = int(w.obs_frame[k])
            z_old, _ = _project(truth.q[f], truth.p[f], w, x_old)
            z_new, _ = _project(truth.q[f], truth.p[f], w, x_new)
            w.obs_z[k] = z_new + (w.obs_z[k] - z_old)
        st.rho[l] = st.rho[l] / truth.rho[l] / d
        truth.rho[l] = 1.0 / d
    return w, st, truth, behind, farl


def with_offplane_tracks(w, st, truth, seed=0, frac=0.3, dist=(0.3, 1.0)):
    """Plane tracks of points off their plane (a wrong plane association): a fraction `frac` of the tracks moved by
    dist = (lo, hi) metres along the plane normal, either side; the point is triangulated from the truth poses and the
    observations, the observations are re-projected with their pixel noise kept.  Returns (w, st, truth, moved tracks,
    signed displacements)."""
    w, st, truth = _copies(w, st, truth)
    rng = np.random.default_rng(seed)
    n = int(round(frac * w.n_ptracks))
    tracks = np.sort(rng.choice(w.n_ptracks, n, replace=False))
    shift = rng.uniform(*dist, n) * rng.choice([-1.0, 1.0], n)
    w.pt_obs_z = w.pt_obs_z.copy()
    for t, dd in zip(tracks, shift):
        ks = range(int(w.pt_obs_begin[t]), int(w.pt_obs_begin[t + 1]))
        A, b = np.zeros((3, 3)), np.zeros(3)
        for k in ks:                                         # least-squares intersection of the observation rays
            qc, pc = _cam_pose(truth.q[w.pt_obs_frame[k]], truth.p[w.pt_obs_frame[k]], w)
            u = so3.qrot(qc, np.array([w.pt_obs_z[k][0], w.pt_obs_z[k][1], 1.0]))
            P = np.eye(3) - np.outer(u, u) / (u @ u)
            A += P
            b += P @ pc
        x = np.linalg.solve(A, b)
        x_new = x + dd * w.plane_normal[w.pt_plane[t]]
        for k in ks:
            f = int(w.pt_obs_frame[k])
            z_old, _ = _project(truth.q[f], truth.p[f], w, x)
            z_new, _ = _project(truth.q[f], truth.p[f], w, x_new)
            w.pt_obs_z[k] = z_new + (w.pt_obs_z[k] - z_old)
    return w, st, truth, tracks, shift



def f32_keypoints(w):
    """The keypoints rounded to fp32, as the device keeps them (the oracle then sees the values the kernels see)."""
    w.obs_z = w.obs_z.astype(np.float32).astype(np.float64)
    w.lm_z_ref = w.lm_z_ref.astype(np.float32).astype(np.float64)
    w.pt_obs_z = w.pt_obs_z.astype(np.float32).astype(np.float64)
    return w


HARD_KINDS_VISUAL = ("far_depths", "low_baseline", "outliers", "general_w", "cauchy_0.3", "cauchy_0.01", "offset",
                     "rejected", "all")
HARD_KINDS_INERTIAL = ("far_depths", "outliers", "general_w", "cauchy_0.01", "offset", "rejected", "all")


def hard_base(inertial, kind, N, M, seed):
    """The generated window a hard kind starts from: cfg3 (inertial) or cfg2, with the outdoor depth mixture for
    far_depths / all and a 1/1000 baseline for low_baseline."""
    mix = DEPTH_MIX_OUTDOOR if kind in ("far_depths", "all") else None
    if inertial:
        return make_cfg3(N=N, M=M, seed=seed, depth_mix=mix)
    return make_cfg2(N=N, M=M, seed=seed, depth_mix=mix, baseline=1e-3 if kind == "low_baseline" else 1.0)


def hard_window(kind, inertial=False, N=8, M=200, seed=800):
    """(Window, State) of one hard kind: plain, far_depths, low_baseline, outliers, general_w, cauchy_0.3,
    cauchy_0.01, offset, rejected, or all (outliers, full W, Cauchy 0.3, rejected landmarks, 5 km offset on the
    outdoor depth mixture), keypoints rounded to fp32."""
    w, st, truth = hard_base(inertial, kind, N, M, seed)
    if kind in ("plain", "far_depths", "low_baseline"):
        pass                                    # made by the generator itself
    elif kind == "outliers":
        w, st, truth, _ = with_outliers(w, st, truth, seed=1)
    elif kind == "general_w":
        w, st, truth = with_general_w(w, st, truth)
    elif kind in ("cauchy_0.3", "cauchy_0.01"):
        w, st, truth, _ = with_outliers(w, st, truth, seed=2)
        w, st, truth = with_cauchy(w, st, truth, float(kind.split("_")[1]))
    elif kind == "offset":
        w, st, truth = with_offset(w, st, truth)
    elif kind == "rejected":
        w, st, truth, _, _ = with_rejected_landmarks(w, st, truth, seed=3)
    elif kind == "all":
        w, st, truth, _ = with_outliers(w, st, truth, seed=4)
        w, st, truth = with_general_w(w, st, truth)
        w, st, truth = with_cauchy(w, st, truth, 0.3)
        w, st, truth, _, _ = with_rejected_landmarks(w, st, truth, seed=5)
        w, st, truth = with_offset(w, st, truth)
    else:
        raise ValueError(kind)
    return f32_keypoints(w), st

# ----------------------------------------------------------------------------- KLT inputs
def _texture(rng, w, h):
    """Band-limited noise (sum of octaves), 8-bit, with good corners everywhere."""
    acc = np.zeros((h, w))
    for octave, amp in ((4, 1.0), (8, 0.8), (16, 0.6), (32, 0.4)):
        gh, gw = h // octave + 3, w // octave + 3
        g = rng.normal(0, 1, (gh, gw))
        ys, xs = np.arange(h) / octave + 1, np.arange(w) / octave + 1
        y0, x0 = ys.astype(int), xs.astype(int)
        fy, fx = (ys - y0)[:, None], (xs - x0)[None, :]
        acc += amp * ((1 - fy) * (1 - fx) * g[y0][:, x0] + (1 - fy) * fx * g[y0][:, x0 + 1]
                      + fy * (1 - fx) * g[y0 + 1][:, x0] + fy * fx * g[y0 + 1][:, x0 + 1])
    acc = (acc - acc.min()) / (acc.max() - acc.min())
    return acc


def make_klt_pair(seed=648, size=(752, 480), n_points=500, max_shift=8.0):
    """Two 8-bit frames related by a small homography (<= max_shift px), points on a jittered
    25-px grid >= 30 px from the border, initial guess = previous position (SURVEY.md 8d KLT row).
    Returns prev, next (uint8 [h,w]), pts (float32 [n,2]), true next positions."""
    rng = np.random.default_rng(seed)
    w, h = size
    tex = _texture(rng, w + 64, h + 64)
    prev = tex[32:32 + h, 32:32 + w]
    # homography close to identity (in pixel coordinates centred on the image)
    ang = np.deg2rad(rng.uniform(-0.6, 0.6))
    sc = 1.0 + rng.uniform(-0.008, 0.008)
    Hm = np.array([[sc * np.cos(ang), -sc * np.sin(ang), rng.uniform(-0.5, 0.5) * max_shift],
                   [sc * np.sin(ang), sc * np.cos(ang), rng.uniform(-0.5, 0.5) * max_shift],
                   [rng.uniform(-2e-6, 2e-6), rng.uniform(-2e-6, 2e-6), 1.0]])
    cx, cy = w / 2.0, h / 2.0

    def warp_pts(p):
        q = np.stack([p[:, 0] - cx, p[:, 1] - cy, np.ones(len(p))], axis=1) @ Hm.T
        return np.stack([q[:, 0] / q[:, 2] + cx, q[:, 1] / q[:, 2] + cy], axis=1)
    # next(x') = prev(H^-1 x'): sample the texture with bilinear interpolation
    Hi = np.linalg.inv(Hm)
    yy, xx = np.mgrid[0:h, 0:w]
    q = np.stack([xx.ravel() - cx, yy.ravel() - cy, np.ones(w * h)], axis=1) @ Hi.T
    sx, sy = q[:, 0] / q[:, 2] + cx + 32, q[:, 1] / q[:, 2] + cy + 32
    x0, y0 = np.floor(sx).astype(int), np.floor(sy).astype(int)
    fx, fy = sx - x0, sy - y0
    x0, y0 = np.clip(x0, 0, w + 62), np.clip(y0, 0, h + 62)
    nxt = ((1 - fy) * (1 - fx) * tex[y0, x0] + (1 - fy) * fx * tex[y0, x0 + 1]
           + fy * (1 - fx) * tex[y0 + 1, x0] + fy * fx * tex[y0 + 1, x0 + 1]).reshape(h, w)
    to_u8 = lambda a: np.clip(np.rint(a * 235.0 + 10.0 + rng.normal(0, 1.0, a.shape)), 0, 255).astype(np.uint8)
    prev8, next8 = to_u8(prev), to_u8(nxt)
    gx, gy = np.meshgrid(np.arange(35, w - 35, 25.0), np.arange(35, h - 35, 25.0))
    pts = np.stack([gx.ravel(), gy.ravel()], axis=1) + rng.uniform(-6, 6, (gx.size, 2))
    sel = rng.permutation(len(pts))[:n_points]
    pts = pts[np.sort(sel)].astype(np.float32)
    return prev8, next8, pts, warp_pts(pts.astype(np.float64)).astype(np.float32)


# ----------------------------------------------------------------------------- PnP inputs
def make_pnp(seed=651, n_points=150, cal=EUROC, use_inertial=True, kf_dt=0.05, imu_hz=200.0, depth=(2.0, 10.0),
             outlier_frac=0.0, outlier_px=(15.0, 300.0), W=None, cauchy_a=1.0, offset=None):
    """Inputs of visual_inertial_pnp (estimation/pnp.cpp:32-100): the last frame (constant), the new
    frame's predicted state, the IMU pre-integration between them and the world points of the tracks
    both frames see, with pixel noise.  Returns a dict of arrays (16-vectors: q xyzw, p, v, bg, ba).
    Hard inputs: depth = (dmin, dmax) of the points; a fraction outlier_frac of the keypoints displaced by
    outlier_px pixels; W a full 2x2 square-root information (general_sqrt_info); cauchy_a of the loss (the dict
    carries it only when it is not 1); offset translates the scene (frames and points)."""
    rng = np.random.default_rng(seed)
    w = _base_window(cal, 2, use_inertial)
    R_wb0 = R_WC0 @ so3.qmat(w.cam_q_cs).T
    t0, t1 = 0.4, 0.4 + kf_dt
    st = []
    for t in (t0, t1):
        p, v, _, th, _ = _trajectory(t)
        st.append((so3.mat2quat(R_wb0 @ so3.qmat(so3.qexp(th))), p, v))
    bg = rng.normal(0, 2e-3, 3)
    ba = rng.normal(0, 2e-2, 3)
    last = np.concatenate([st[0][0], st[0][1], st[0][2], bg, ba])
    truth = np.concatenate([st[1][0], st[1][1], st[1][2], bg, ba])
    pre = so3.PreIntegrator(cal['cov_g'], cal['cov_a'], cal['cov_bg'], cal['cov_ba'])
    dt = 1.0 / imu_hz
    for s in range(int(round(kf_dt * imu_hz))):
        t = t0 + s * dt
        _, _, a, th, thd = _trajectory(t + 0.5 * dt)
        Rwb = R_wb0 @ so3.qmat(so3.qexp(th))
        gyro = so3.right_jacobian(th) @ thd + bg + rng.normal(0, np.sqrt(cal['cov_g'] * imu_hz), 3)
        acc = Rwb.T @ (a - GRAVITY) + ba + rng.normal(0, np.sqrt(cal['cov_a'] * imu_hz), 3)
        pre.data.append((t, gyro, acc))
    imu = pre.integrate(t1, bg, ba)
    q_t = np.stack([st[0][0], st[1][0]])
    p_t = np.stack([st[0][1], st[1][1]])
    fx, fy = cal['K'][0], cal['K'][1]
    s_px = np.sqrt(cal['noise_px2'])
    pts, zs = [], []
    for _ in range(n_points):
        x, _, _ = _sample_landmark(rng, cal, w, q_t, p_t, [0, 1], depth[0], depth[1])
        z, _ = _project(q_t[1], p_t[1], w, x)
        pts.append(x + rng.normal(0, 0.02, 3))                 # landmark estimate, not the true point
        zs.append(z + rng.normal(0, s_px, 2) / np.array([fx, fy]))
    guess = truth.copy()
    guess[0:4] = so3.qnormalize(so3.qmul(truth[0:4], so3.qexp(rng.normal(0, np.deg2rad(0.7), 3))))
    guess[4:7] += rng.normal(0, 0.03, 3)
    guess[7:10] += rng.normal(0, 0.05, 3)
    pts, zs = np.array(pts), np.array(zs)
    if outlier_frac > 0:                                       # own stream: the draws above do not move
        r2 = np.random.default_rng(seed + 7919)
        bad = r2.choice(n_points, int(round(outlier_frac * n_points)), replace=False)
        zs[bad] += _px_offsets(r2, len(bad), outlier_px, fx, fy)
    if offset is not None:
        o = np.asarray(offset, dtype=float)
        for v in (guess, last, truth):
            v[4:7] += o
        pts = pts + o
    d = dict(frame=guess, last=last, truth=truth, imu=imu, pts=pts, zs=zs,
             cam_q=w.cam_q_cs, cam_p=w.cam_p_cs, imu_q=w.imu_q_cs, imu_p=w.imu_p_cs,
             W=w.sqrt_inv_cov if W is None else np.asarray(W, dtype=float), use_inertial=use_inertial)
    if cauchy_a != 1.0:
        d['cauchy_a'] = float(cauchy_a)
    return d


def make_fm_matches(seed=652, n=300, outlier_frac=0.2, noise=0.3, planar=False, cal=EUROC):
    """Matched keypoints (float32 pixels) of n world points seen from two nearby camera poses, Gaussian pixel noise,
    the first int(outlier_frac n) matches displaced by up to 40 px: the input of the F-matrix RANSAC of
    OpenCvImage::track_keypoints (opencv_image.cpp:121-129).  Returns (p, q)."""
    r = np.random.default_rng(seed)
    fx, fy, cx, cy = 458.0, 457.0, 367.0, 248.0
    X = np.stack([r.uniform(-4, 4, n), r.uniform(-3, 3, n), r.uniform(3, 12, n)], 1)
    if planar:
        X[:, 2] = 6.0 + 0.01 * r.standard_normal(n)
    w = r.normal(0, 0.05, 3)
    t = r.normal(0, 0.3, 3)
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    R = np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
    x1 = np.stack([fx * X[:, 0] / X[:, 2] + cx, fy * X[:, 1] / X[:, 2] + cy], 1)
    X2 = X @ R.T + t
    x2 = np.stack([fx * X2[:, 0] / X2[:, 2] + cx, fy * X2[:, 1] / X2[:, 2] + cy], 1)
    x1 = x1 + r.normal(0, noise, x1.shape)
    x2 = x2 + r.normal(0, noise, x2.shape)
    no = int(outlier_frac * n)
    if no:
        x2[:no] += r.uniform(-40, 40, (no, 2))
    return x1.astype(np.float32), x2.astype(np.float32)


def make_two_view(seed=660, n=150, outlier_frac=0.0, noise_px=0.5, kind="general", cal=EUROC):
    """Frames i and j of init_sfm's two-view step (initializer.cpp:117-127): n world points seen from two camera poses,
    Gaussian pixel noise, the first int(outlier_frac n) matches of frame j displaced by 20 to 80 pixels.
    kind: 'general' (depths 3..12 m, a 1 m baseline), 'plane' (every point on one tilted plane), 'rotation' (no
    translation), 'small' (a 2 cm baseline and a
    small rotation: too little parallax).  Returns a dict: p1, p2 [n][2] normalised keypoints,
    fx, fy, R, t (x_j = R x_i + t), X [n][3] the points in frame i."""
    r = np.random.default_rng(seed)
    fx, fy = cal["K"][0], cal["K"][1]
    X = np.stack([r.uniform(-4, 4, n), r.uniform(-3, 3, n), r.uniform(3, 12, n)], 1)
    if kind == "plane":
        X[:, 2] = 7.0 + 0.3 * X[:, 0] - 0.2 * X[:, 1]
    w = r.normal(0, 0.08, 3) * (0.05 if kind == "small" else 1.0)
    R = _rodrigues(w)
    b = {"general": 1.0, "plane": 1.0, "rotation": 0.0, "small": 0.02}[kind]
    d = r.normal(0, 1, 3)
    d[2] *= 0.3
    t = b * d / np.linalg.norm(d)
    Xj = X @ R.T + t
    p1 = X[:, :2] / X[:, 2:]
    p2 = Xj[:, :2] / Xj[:, 2:]
    px = np.array([fx, fy])
    p1 = p1 + r.normal(0, noise_px, p1.shape) / px
    p2 = p2 + r.normal(0, noise_px, p2.shape) / px
    no = int(outlier_frac * n)
    if no:
        off = r.uniform(20, 80, (no, 2)) * r.choice([-1, 1], (no, 2))
        p2[:no] += off / px
    return dict(p1=p1, p2=p2, fx=fx, fy=fy, R=R, t=t, X=X)


def _rodrigues(w):
    th = np.linalg.norm(w)
    k = w / th
    Kx = np.array([[0, -k[2], k[1]], [k[2], 0, -k[0]], [-k[1], k[0], 0]])
    return np.eye(3) + np.sin(th) * Kx + (1 - np.cos(th)) * Kx @ Kx
