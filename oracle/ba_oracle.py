"""TEST INFRASTRUCTURE ONLY -- fp64 NumPy oracle for PVIO's sliding-window BA hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference leg
may import this module; the product (pvio_b200/) never does and fails loudly without its
CUDA library.

What is restated (reference paths relative to /root/reference/pvio/src/pvio):
  R  estimation/ceres/reprojection_error_cost.h:40-120      reprojection_evaluate
  I  estimation/ceres/preintegration_error_cost.h:40-160     preintegration_evaluate
  P  estimation/ceres/marginalization_error_cost.h:53-94     marginalization_evaluate
  A  estimation/ceres/augmented_plane_distance_error_cost.h:53-136  plane_evaluate
  Q  estimation/ceres/quaternion_parameterization.h:27-44    (oracle/lie.py quat_plus)
  S  estimation/bundle_adjustor.cpp:63-299  problem assembly (which blocks exist, which
     are constant, which carry CauchyLoss(1.0)) and the post-pass :277-296
  M  estimation/bundle_adjustor.cpp:348-599 marginalize()
  C  Ceres Solver 1.14.0 (pvio/depends/CMakeLists.txt:31-35; NOT in /root/reference, not
     installed here): loss Corrector, Jacobi scaling, TRADITIONAL_DOGLEG trust region,
     step acceptance and the convergence tests, restated from the published algorithm
     (trust_region_minimizer.cc, dogleg_strategy.cc, corrector.cc, defaults in
     solver.h) with the options PVIO sets (estimation/ceres/solver_options.h:26-33).

PARITY PINNING: the functor restatements (R, I, P, A) are pinned by finite-difference
checks in the style of estimation/ceres/cost_function_validator.h:39-43,270-323 because
the reference ships no tests or golden vectors and cannot be compiled here (Eigen/Ceres
absent).  The optimiser loop C is "PARITY UNPINNED": no Ceres result exists to check it
against; parity on dx is therefore defined against this oracle's fp64 step.

Window / State are duck-typed containers of NumPy arrays (see pvio_b200/window.py for
the product-side definition of the same fields).
"""
import numpy as np
from .lie import (hat, qmul, qconj, qmat, qrot, expmap, logmap, right_jacobian,
                  quat_plus, qnormalized)

GRAVITY = np.array([0.0, 0.0, -9.80665])  # PVIO_GRAVITY_NOMINAL, preintegration_error_cost.h:41
ES_Q, ES_P, ES_V, ES_BG, ES_BA, ES_SIZE = 0, 3, 6, 9, 12, 15  # estimation/state.h:29-36


# ----------------------------------------------------------------------------- functors
def reprojection_evaluate(q_tgt, p_tgt, q_ref, p_ref, rho, z_tgt, z_ref,
                          cam_q, cam_p, sqrt_inv_cov, jac=True):
    """reprojection_error_cost.h:40-120.  Returns r[2] and (if jac) the LOCAL Jacobians
    (2x3 each; the reference's 4th quaternion column is zero) J_qt, J_pt, J_qr, J_pr, J_rho."""
    y_ref = np.array([z_ref[0], z_ref[1], 1.0]) / rho                    # :58
    y_ref_center = qrot(cam_q, y_ref) + cam_p                             # :59
    x = qrot(q_ref, y_ref_center) + p_ref                                 # :60
    y_tgt_center = qrot(qconj(q_tgt), x - p_tgt)                          # :61
    y_tgt = qrot(qconj(cam_q), y_tgt_center - cam_p)                      # :62
    r = y_tgt[:2] / y_tgt[2] - z_tgt                                      # :63
    out = [sqrt_inv_cov @ r]                                              # :117
    if jac:
        zz = y_tgt[2]
        dproj = np.array([[1.0 / zz, 0.0, -y_tgt[0] / (zz * zz)],
                          [0.0, 1.0 / zz, -y_tgt[1] / (zz * zz)]])
        dr_dy_tgt = sqrt_inv_cov @ dproj                                  # :66-69
        dr_dy_tgt_center = dr_dy_tgt @ qmat(qconj(cam_q))                 # :75
        dr_dx = dr_dy_tgt_center @ qmat(qconj(q_tgt))                     # :79
        dr_dy_ref_center = dr_dx @ qmat(q_ref)                            # :86
        J_qt = dr_dy_tgt_center @ hat(y_tgt_center)                       # :95
        J_pt = -dr_dx                                                     # :100
        J_qr = -dr_dy_ref_center @ hat(y_ref_center)                      # :104
        J_pr = dr_dx                                                      # :109
        J_rho = -dr_dy_ref_center @ qmat(cam_q) @ y_ref / rho             # :113
        out += [J_qt, J_pt, J_qr, J_pr, J_rho]
    return out


def preintegration_evaluate(qi_c, pi_c, vi, bgi, bai, qj_c, pj_c, vj, bgj, baj,
                            imu, imu_q, imu_p, jac=True):
    """preintegration_error_cost.h:40-160.  `imu` is a dict with dt,dq,dp,dv,sqrt_inv_cov,
    dq_dbg,dp_dbg,dp_dba,dv_dbg,dv_dba,bg0,ba0 (the PreIntegrator outputs,
    estimation/preintegrator.h:29-44, plus the bias linearisation point -- SURVEY quirk Q1).
    Returns whitened r[15] and J[15,30] in local coordinates [th_i p_i v_i bg_i ba_i | ..j]."""
    dt, dq, dp, dv = imu['dt'], imu['dq'], imu['dp'], imu['dv']
    W = imu['sqrt_inv_cov']
    q_i = qmul(qi_c, imu_q)                                               # :60
    p_i = pi_c + qrot(qi_c, imu_p)                                        # :61
    q_j = qmul(qj_c, imu_q)                                               # :62
    p_j = pj_c + qrot(qj_c, imu_p)                                        # :63
    dbg = bgi - imu['bg0']                                                # :69
    dba = bai - imu['ba0']                                                # :70
    r = np.zeros(15)
    r[ES_Q:ES_Q + 3] = logmap(qmul(qmul(qconj(qmul(dq, expmap(imu['dq_dbg'] @ dbg))),
                                        qconj(q_i)), q_j))                 # :79
    Rit = qmat(qconj(q_i))
    r[ES_P:ES_P + 3] = Rit @ (p_j - p_i - dt * vi - 0.5 * dt * dt * GRAVITY) \
        - (dp + imu['dp_dbg'] @ dbg + imu['dp_dba'] @ dba)                # :80
    r[ES_V:ES_V + 3] = Rit @ (vj - vi - dt * GRAVITY) \
        - (dv + imu['dv_dbg'] @ dbg + imu['dv_dba'] @ dba)                # :81
    r[ES_BG:ES_BG + 3] = bgj - bgi                                        # :82
    r[ES_BA:ES_BA + 3] = baj - bai                                        # :83
    if not jac:
        return [W @ r]
    J = np.zeros((15, 30))
    rq = r[ES_Q:ES_Q + 3]
    Jr_inv = np.linalg.inv(right_jacobian(rq))
    Rimu_t = qmat(qconj(imu_q))
    Rci_t = qmat(qconj(qi_c))
    # dq_i :86-93
    J[ES_Q:ES_Q + 3, 0:3] = -Jr_inv @ qmat(qconj(q_j)) @ qmat(qi_c)
    J[ES_P:ES_P + 3, 0:3] = Rimu_t @ hat(Rci_t @ (p_j - pi_c - dt * vi - 0.5 * dt * dt * GRAVITY))
    J[ES_V:ES_V + 3, 0:3] = Rimu_t @ hat(Rci_t @ (vj - vi - dt * GRAVITY))
    # dp_i :94-99
    J[ES_P:ES_P + 3, 3:6] = -Rit
    # dv_i :100-106
    J[ES_P:ES_P + 3, 6:9] = -dt * Rit
    J[ES_V:ES_V + 3, 6:9] = -Rit
    # dbg_i :107-115
    J[ES_Q:ES_Q + 3, 9:12] = -Jr_inv @ qmat(qconj(expmap(rq))) \
        @ right_jacobian(imu['dq_dbg'] @ dbg) @ imu['dq_dbg']
    J[ES_P:ES_P + 3, 9:12] = -imu['dp_dbg']
    J[ES_V:ES_V + 3, 9:12] = -imu['dv_dbg']
    J[ES_BG:ES_BG + 3, 9:12] = -np.eye(3)
    # dba_i :116-123
    J[ES_P:ES_P + 3, 12:15] = -imu['dp_dba']
    J[ES_V:ES_V + 3, 12:15] = -imu['dv_dba']
    J[ES_BA:ES_BA + 3, 12:15] = -np.eye(3)
    # dq_j :124-130
    J[ES_Q:ES_Q + 3, 15:18] = Jr_inv @ Rimu_t
    J[ES_P:ES_P + 3, 15:18] = -Rit @ qmat(qj_c) @ hat(imu_p)
    # dp_j, dv_j, dbg_j, dba_j :131-154
    J[ES_P:ES_P + 3, 18:21] = Rit
    J[ES_V:ES_V + 3, 21:24] = Rit
    J[ES_BG:ES_BG + 3, 24:27] = np.eye(3)
    J[ES_BA:ES_BA + 3, 27:30] = np.eye(3)
    return [W @ r, W @ J]


def marginalization_evaluate(win, st, jac=True):
    """marginalization_error_cost.h:53-94.  Returns r[15n] (and J[15n,15n] w.r.t. the
    local coordinates of the n related frames, in prior order)."""
    n = win.n_prior
    S, e = win.prior_S, win.prior_e
    r = np.zeros(15 * n)
    E = np.eye(15 * n)
    for i in range(n):
        f = int(win.prior_frames[i])
        rq = logmap(qmul(qconj(win.prior_q0[i]), st.q[f]))                # :65
        r[15 * i + ES_Q:15 * i + ES_Q + 3] = rq
        r[15 * i + ES_P:15 * i + ES_P + 3] = st.p[f] - win.prior_p0[i]
        r[15 * i + ES_V:15 * i + ES_V + 3] = st.v[f] - win.prior_v0[i]
        r[15 * i + ES_BG:15 * i + ES_BG + 3] = st.bg[f] - win.prior_bg0[i]
        r[15 * i + ES_BA:15 * i + ES_BA + 3] = st.ba[f] - win.prior_ba0[i]
        if jac:
            E[15 * i:15 * i + 3, 15 * i:15 * i + 3] = np.linalg.inv(right_jacobian(rq))  # :76
    out = [S @ r + e]                                                     # :91
    if jac:
        out.append(S @ E)                                                 # :77,:84
    return out


def plane_evaluate(qs, ps, zs, normal, distance, cam_q, cam_p, sqrt_inv_cov,
                   regularization_weight=1.0, jac=True):
    """augmented_plane_distance_error_cost.h:53-136.  qs/ps/zs: the K observing body
    poses and keypoints.  Returns r (scalar) and J[6K] local ([th_0 p_0 th_1 p_1 ...]).
    Plane parameters are constant in the reference solve (bundle_adjustor.cpp:108-109),
    so their Jacobians (:121-130) are not produced."""
    K = len(qs)
    A = np.zeros((2 * K + 1, 3))
    b = np.zeros(2 * K + 1)
    Rsw_l = []
    for i in range(K):
        Rsw = qmat(qmul(qconj(cam_q), qconj(qs[i])))                      # :68
        Tsw = -Rsw @ ps[i] - qrot(qconj(cam_q), cam_p)                    # :69
        A[2 * i + 0] = zs[i][0] * Rsw[2] - Rsw[0]                         # :71
        A[2 * i + 1] = zs[i][1] * Rsw[2] - Rsw[1]
        b[2 * i + 0] = zs[i][0] * Tsw[2] - Tsw[0]
        b[2 * i + 1] = zs[i][1] * Tsw[2] - Tsw[1]
        Rsw_l.append(Rsw)
    A[2 * K] = regularization_weight * normal                             # :84
    b[2 * K] = regularization_weight * distance
    ATA = A.T @ A
    ATb = A.T @ b
    lam, V = np.linalg.eigh(ATA)                                          # :90
    lam_inv = np.where(lam > 1.0e-8, 1.0 / np.where(lam > 1.0e-8, lam, 1.0), 0.0)
    ATAinv = V @ np.diag(lam_inv) @ V.T
    x = -ATAinv @ ATb                                                     # :94
    r = normal @ x - distance                                             # :96
    if not jac:
        return [r * sqrt_inv_cov]
    J = np.zeros(6 * K)
    Rcs = qmat(cam_q)
    for i in range(K):
        Jb = np.array([[-1.0, 0.0, zs[i][0]], [0.0, -1.0, zs[i][1]]])
        A0, A1 = A[2 * i], A[2 * i + 1]
        dxdA0 = (b[2 * i] + A0 @ x) * ATAinv + np.outer(x, A0 @ ATAinv).T      # :105
        dxdA1 = (b[2 * i + 1] + A1 @ x) * ATAinv + np.outer(x, A1 @ ATAinv).T
        Rwc = qmat(qs[i])
        dA0dq = Rwc @ hat(Rcs @ Jb[0])                                    # :107
        dA1dq = Rwc @ hat(Rcs @ Jb[1])
        dxdAdq = dxdA0 @ dA0dq + dxdA1 @ dA1dq
        dxdbdq = ATAinv @ A[2 * i:2 * i + 2].T @ Jb @ Rcs.T @ hat(qrot(qconj(qs[i]), ps[i]))  # :110
        J[6 * i:6 * i + 3] = normal @ (dxdAdq + dxdbdq)
        J[6 * i + 3:6 * i + 6] = normal @ (ATAinv @ A[2 * i:2 * i + 2].T @ Jb @ Rsw_l[i])  # :117
    return [r * sqrt_inv_cov, J * sqrt_inv_cov]


# ------------------------------------------------------------------- Ceres loss corrector
def cauchy_rho(s, a=1.0):
    """ceres::CauchyLoss(a): rho(s) = b log(1 + s/b), b = a^2 (loss_function.cc).
    Returns rho, rho', rho''."""
    b = a * a
    c = 1.0 / b
    t = 1.0 + s * c
    inv = 1.0 / t
    return b * np.log(t), max(inv, np.finfo(float).tiny), -c * inv * inv


def corrector_scale(r, a=1.0):
    """ceres Corrector (corrector.cc): rho'' <= 0 for Cauchy => residual and Jacobian are
    both scaled by sqrt(rho'); the block's cost is rho(s)/2."""
    s = float(r @ r)
    rho0, rho1, rho2 = cauchy_rho(s, a)
    return np.sqrt(rho1), 0.5 * rho0


# --------------------------------------------------------------------------- assembly
def local_dim(win):
    return 15 * win.N + win.M


def free_mask(win):
    """Which local coordinates are parameters of the reference problem
    (bundle_adjustor.cpp:75-88): q,p constant for FF_FIX_POSE frames; v,bg,ba exist only
    if use_inertial."""
    m = np.ones(local_dim(win), dtype=bool)
    for f in range(win.N):
        if win.frame_fixed[f]:
            m[15 * f:15 * f + 6] = False
        if not win.use_inertial:
            m[15 * f + 6:15 * f + 15] = False
    # a landmark without residual blocks is dropped from ceres' reduced program (stays constant)
    m[15 * win.N:] = np.diff(win.lm_obs_begin) > 0
    return m


def iter_residual_blocks(win, st, jac=True):
    """Yield (r, [(col0, Jblock), ...], cost) for every residual block, already
    loss-corrected, in the order bundle_adjustor.cpp adds them (:126-242)."""
    N = win.N
    # prior :126-139 (no loss)
    if win.n_prior > 0:
        out = marginalization_evaluate(win, st, jac)
        r = out[0]
        blocks = []
        if jac:
            for i in range(win.n_prior):
                blocks.append((15 * int(win.prior_frames[i]), out[1][:, 15 * i:15 * i + 15]))
        yield r, blocks, 0.5 * float(r @ r)
    # reprojection :142-161 (CauchyLoss(1.0))
    for l in range(win.M):
        a = int(win.lm_anchor[l])
        for k in range(int(win.lm_obs_begin[l]), int(win.lm_obs_begin[l + 1])):
            t = int(win.obs_frame[k])
            out = reprojection_evaluate(st.q[t], st.p[t], st.q[a], st.p[a], st.rho[l],
                                        win.obs_z[k], win.lm_z_ref[l],
                                        win.cam_q_cs, win.cam_p_cs, win.sqrt_inv_cov, jac)
            sc, cost = corrector_scale(out[0], win.cauchy_a)
            blocks = []
            if jac:
                Jt = np.hstack([out[1], out[2]]) * sc
                Jr = np.hstack([out[3], out[4]]) * sc
                blocks = [(15 * t, Jt), (15 * a, Jr), (15 * N + l, (out[5] * sc).reshape(2, 1))]
            yield out[0] * sc, blocks, cost
    # plane :162-196 (CauchyLoss(1.0)), only planes with >= 20 tracks reach the window
    for t_ in range(win.n_ptracks):
        pl = int(win.pt_plane[t_])
        ks = range(int(win.pt_obs_begin[t_]), int(win.pt_obs_begin[t_ + 1]))
        fr = [int(win.pt_obs_frame[k]) for k in ks]
        out = plane_evaluate([st.q[f] for f in fr], [st.p[f] for f in fr],
                             [win.pt_obs_z[k] for k in ks], win.plane_normal[pl],
                             float(win.plane_distance[pl]), win.cam_q_cs, win.cam_p_cs,
                             win.plane_sqrt_inv_cov, 1.0, jac)
        r = np.array([out[0]])
        sc, cost = corrector_scale(r, win.cauchy_a)
        blocks = []
        if jac:
            for i, f in enumerate(fr):
                blocks.append((15 * f, (out[1][6 * i:6 * i + 6] * sc).reshape(1, 6)))
        yield r * sc, blocks, cost
    # IMU :220-242 (no loss)
    if win.use_inertial:
        for n in range(win.n_imu):
            i, j = int(win.imu_frame_i[n]), int(win.imu_frame_j[n])
            out = preintegration_evaluate(st.q[i], st.p[i], st.v[i], st.bg[i], st.ba[i],
                                          st.q[j], st.p[j], st.v[j], st.bg[j], st.ba[j],
                                          imu_record(win, n), win.imu_q_cs, win.imu_p_cs, jac)
            r = out[0]
            blocks = [(15 * i, out[1][:, :15]), (15 * j, out[1][:, 15:])] if jac else []
            yield r, blocks, 0.5 * float(r @ r)


def imu_record(win, n):
    return dict(dt=float(win.imu_dt[n]), dq=win.imu_dq[n], dp=win.imu_dp[n], dv=win.imu_dv[n],
                sqrt_inv_cov=win.imu_sqrt_inv_cov[n], dq_dbg=win.imu_dq_dbg[n],
                dp_dbg=win.imu_dp_dbg[n], dp_dba=win.imu_dp_dba[n], dv_dbg=win.imu_dv_dbg[n],
                dv_dba=win.imu_dv_dba[n], bg0=win.imu_bg0[n], ba0=win.imu_ba0[n])


def total_cost(win, st):
    return sum(c for _, _, c in iter_residual_blocks(win, st, jac=False))


def dense_jacobian(win, st):
    """Stacked (loss-corrected, local) J and r -- small windows / FD tests only."""
    rows, rs = [], []
    n = local_dim(win)
    for r, blocks, _ in iter_residual_blocks(win, st):
        Jrow = np.zeros((len(r), n))
        for c0, Jb in blocks:
            Jrow[:, c0:c0 + Jb.shape[1]] += Jb
        rows.append(Jrow)
        rs.append(r)
    return np.vstack(rows), np.concatenate(rs)


def normal_equations(win, st):
    """H = J^T J, g = J^T r over all residual blocks (dense, (15N+M)^2), and the cost."""
    n = local_dim(win)
    H = np.zeros((n, n))
    g = np.zeros(n)
    cost = 0.0
    for r, blocks, c in iter_residual_blocks(win, st):
        cost += c
        for ci, Ji in blocks:
            g[ci:ci + Ji.shape[1]] += Ji.T @ r
            for cj, Jj in blocks:
                H[ci:ci + Ji.shape[1], cj:cj + Jj.shape[1]] += Ji.T @ Jj
    return H, g, cost


def apply_step(win, st, dx):
    """QuaternionParameterization::Plus for q, plain addition elsewhere."""
    out = st.copy()
    N = win.N
    for f in range(N):
        d = dx[15 * f:15 * f + 15]
        out.q[f] = quat_plus(st.q[f], d[0:3])
        out.p[f] = st.p[f] + d[3:6]
        out.v[f] = st.v[f] + d[6:9]
        out.bg[f] = st.bg[f] + d[9:12]
        out.ba[f] = st.ba[f] + d[12:15]
    out.rho = st.rho + dx[15 * N:]
    return out


MIN_DIAG, MAX_DIAG = 1.0e-6, 1.0e32    # ceres Solver::Options min/max_lm_diagonal defaults
MIN_MU, MAX_MU, MU_INC = 1.0e-8, 1.0, 10.0  # dogleg_strategy.cc


def jacobi_scaling(H):
    """trust_region_minimizer.cc: scale_i = 1 / (1 + sqrt(sum_rows J_i^2)), fixed at iter 0."""
    return 1.0 / (1.0 + np.sqrt(np.maximum(np.diag(H), 0.0)))


def lm_regulariser(H, scale, mu):
    """The term the regularised GN solve adds to diag(H) in UNSCALED coordinates:
    mu * clamp(scale_i^2 H_ii, 1e-6, 1e32) / scale_i^2 (dogleg_strategy.cc ComputeStep +
    ComputeGaussNewtonStep with D = sqrt(mu) * diagonal)."""
    d2 = np.clip(scale * scale * np.diag(H), MIN_DIAG, MAX_DIAG)
    return mu * d2 / (scale * scale), d2


def gn_step(win, st, mu=MIN_MU, scale=None, schur=False):
    """One regularised Gauss-Newton step dx = -(H + reg)^-1 g on the free coordinates.
    Returns dict(dx, H, g, cost, reg, free [, Hred, gred])."""
    H, g, cost = normal_equations(win, st)
    if scale is None:
        scale = jacobi_scaling(H)
    reg, d2 = lm_regulariser(H, scale, mu)
    free = free_mask(win)
    n = local_dim(win)
    dx = np.zeros(n)
    Hr = H + np.diag(reg)
    out = dict(H=H, g=g, cost=cost, reg=reg, free=free, scale=scale, d2=d2)
    if not schur:
        idx = np.where(free)[0]
        dx[idx] = -np.linalg.solve(Hr[np.ix_(idx, idx)], g[idx])
    else:
        P = 15 * win.N
        pf = np.where(free[:P])[0]
        Hpp = Hr[:P, :P]
        Hpl = Hr[:P, P:]
        Hll = np.where(free[P:], np.diag(Hr)[P:], 1.0)
        Hred = Hpp - (Hpl / Hll) @ Hpl.T
        gred = g[:P] - Hpl @ (g[P:] / Hll)
        dx[pf] = -np.linalg.solve(Hred[np.ix_(pf, pf)], gred[pf])
        dx[P:] = np.where(free[P:], -(g[P:] + Hpl.T @ dx[:P]) / Hll, 0.0)
        out.update(Hred=Hred, gred=gred)
    out['dx'] = dx
    return out


# --------------------------------------------------------------- Ceres trust-region loop
def trust_region(normal, cost_fn, plus, ambient, x0, idx, ndim, max_iter=10, radius0=1.0e4, verbose=False,
                 on_accept=None):
    """Generic restatement of ceres' TrustRegionMinimizer + TRADITIONAL_DOGLEG (Ceres 1.14, options as
    PVIO sets them, estimation/ceres/solver_options.h:26-33): jacobi_scaling=true fixed at iteration
    0, initial radius 1e4, mu in [1e-8, 1] x10 on linear-solver failure, min_relative_decrease 1e-3,
    function / gradient / parameter tolerances 1e-6 / 1e-10 / 1e-8.
      normal(x) -> (H, g, cost) dense local normal equations;  cost_fn(x) -> cost;
      plus(x, dx) -> x';  ambient(x) -> ambient parameter vector (ceres takes norms of it);
      idx: free local coordinates;  on_accept(x): hook run before re-linearising an accepted point.
    PARITY UNPINNED against Ceres itself (not installed); see the module docstring."""
    x = x0
    H, g, cost = normal(x)
    scale = jacobi_scaling(H)
    radius, mu, reuse = radius0, MIN_MU, False
    summ = dict(iterations=0, initial_cost=cost, final_cost=cost, termination='NO_CONVERGENCE',
                usable=True, steps=[], accepted=[])
    if np.max(np.abs(g[idx])) <= 1e-10:
        summ['termination'] = 'CONVERGENCE'
        return x, summ
    x_norm = float(np.linalg.norm(ambient(x)))
    it = 0
    gn_s = None
    while True:
        if it >= max_iter:
            break
        it += 1
        # ---- DoglegStrategy::ComputeStep (all in Jacobi-scaled coordinates)
        Hs = (H * scale[:, None] * scale[None, :])[np.ix_(idx, idx)]
        gs = (g * scale)[idx]
        if not reuse:
            diag = np.sqrt(np.clip(np.diag(Hs), MIN_DIAG, MAX_DIAG))
            grad = gs / diag
            sg = grad / diag
            alpha = float(grad @ grad) / float(sg @ Hs @ sg)
            while True:
                lm = diag * np.sqrt(mu)
                try:
                    xs = np.linalg.solve(Hs + np.diag(lm * lm), gs)
                    ok = bool(np.all(np.isfinite(xs)))
                except np.linalg.LinAlgError:
                    ok = False
                if ok:
                    break
                mu *= MU_INC
                if mu > MAX_MU:
                    summ['termination'] = 'FAILURE'
                    summ['usable'] = False
                    return x, summ
            gn_s = -diag * xs
        gn_norm = float(np.linalg.norm(gn_s))
        g_norm = float(np.linalg.norm(grad))
        if gn_norm <= radius:
            step_s, step_norm = gn_s.copy(), gn_norm
        elif g_norm * alpha >= radius:
            step_s, step_norm = -(radius / g_norm) * grad, radius
        else:
            b_dot_a = -alpha * float(grad @ gn_s)
            a2 = (alpha * g_norm) ** 2
            bma2 = a2 - 2.0 * b_dot_a + gn_norm ** 2
            c = b_dot_a - a2
            d = np.sqrt(c * c + bma2 * (radius ** 2 - a2))
            beta = (d - c) / bma2 if c <= 0 else (radius ** 2 - a2) / (d + c)
            step_s, step_norm = (-alpha * (1.0 - beta)) * grad + beta * gn_s, radius
        step_s = step_s / diag
        # ---- model cost change (trust_region_minimizer.cc ComputeTrustRegionStep)
        model_change = -float(step_s @ gs + 0.5 * step_s @ Hs @ step_s)
        dx = np.zeros(ndim)
        dx[idx] = step_s * scale[idx]
        if model_change < 0:                       # invalid step
            radius *= 0.5
            reuse = True
            continue
        cand = plus(x, dx)
        cand_cost = cost_fn(cand)
        summ['steps'].append(dx.copy())
        # parameter tolerance
        if np.linalg.norm(ambient(cand) - ambient(x)) <= 1e-8 * (x_norm + 1e-8):
            summ['termination'] = 'CONVERGENCE'
            break
        if abs(cost - cand_cost) <= 1e-6 * cost:
            summ['termination'] = 'CONVERGENCE'
            break
        rel = (cost - cand_cost) / model_change
        if verbose:
            print(f"it {it} cost {cost:.6e} -> {cand_cost:.6e} rel {rel:.3f} radius {radius:.3e}")
        if rel > 1e-3:
            x, cost = cand, cand_cost
            if on_accept is not None:
                on_accept(x)
            x_norm = float(np.linalg.norm(ambient(x)))
            H, g, cost = normal(x)
            summ['accepted'].append(True)
            if rel < 0.25:
                radius *= 0.5
            if rel > 0.75:
                radius = max(radius, 3.0 * step_norm)
            mu = max(MIN_MU, 2.0 * mu / MU_INC)
            reuse = False
            if np.max(np.abs(g[idx])) <= 1e-10:
                summ['termination'] = 'CONVERGENCE'
                break
        else:
            summ['accepted'].append(False)
            radius *= 0.5
            reuse = True
        if radius <= 1e-32:
            summ['termination'] = 'CONVERGENCE'
            break
    summ['iterations'] = it
    summ['final_cost'] = cost
    return x, summ


def solve(win, st0, max_iter=10, verbose=False, alias_bias=True, radius0=1.0e4):
    """ceres::Solve on the sliding window as PVIO configures it (bundle_adjustor.cpp:244-249;
    SPARSE_SCHUR is an exact solver, so only the minimiser logic of trust_region() matters).
    Quirk Q1 (SURVEY 8a): the IMU bias linearisation point aliases the parameter
    (preintegration_error_cost.h:57-58 reads frame_i->motion, which ceres refreshes after
    every successful iteration because update_state_every_iteration=true), so with
    alias_bias=True bg0/ba0 follow the accepted state and only the current step's bias
    change is ever applied to the pre-integrated deltas.  alias_bias=False freezes the
    linearisation point at solve entry (the proper first-order correction).  The exact
    point inside a ceres iteration at which the user state is refreshed (before or after
    the re-linearisation of an accepted step) cannot be verified without Ceres; this
    restatement refreshes BEFORE re-linearising.  Returns (state, summary dict)."""
    alias = alias_bias and win.use_inertial
    box = [win.with_bias_lin_point(st0) if alias else win]
    free = free_mask(win)
    idx = np.where(free)[0]

    def on_accept(st):
        if alias:
            box[0] = box[0].with_bias_lin_point(st)
    return trust_region(lambda st: normal_equations(box[0], st), lambda st: total_cost(box[0], st),
                        lambda st, dx: apply_step(box[0], st, dx), lambda st: _x_vec(box[0], st, free),
                        st0.copy(), idx, local_dim(win), max_iter, radius0, verbose, on_accept)


def _x_vec(win, st, free):
    """The AMBIENT parameter vector ceres takes norms of (q has 4 coordinates)."""
    parts = []
    for f in range(win.N):
        if not win.frame_fixed[f]:
            parts += [st.q[f], st.p[f]]
        if win.use_inertial:
            parts += [st.v[f], st.bg[f], st.ba[f]]
    parts.append(st.rho)
    return np.concatenate(parts)


def _x_norm(win, st, free):
    return float(np.linalg.norm(_x_vec(win, st, free)))


# ------------------------------------------------------------------------- post-pass
def landmark_postpass(win, st):
    """bundle_adjustor.cpp:277-296 restricted to the window's landmarks: depth check
    1e-3 < z <= 50 in every observing camera (anchor included) and mean pixel error.
    Returns (valid[M] bool, quality[M])."""
    M = win.M
    valid = np.ones(M, dtype=bool)
    quality = np.zeros(M)
    fx, fy = win.K_fx, win.K_fy
    for l in range(M):
        a = int(win.lm_anchor[l])
        qa = qmul(st.q[a], win.cam_q_cs)
        pa = st.p[a] + qrot(st.q[a], win.cam_p_cs)
        x = qrot(qa, np.array([win.lm_z_ref[l][0], win.lm_z_ref[l][1], 1.0])) / st.rho[l] + pa
        obs = [(a, win.lm_z_ref[l])]
        obs += [(int(win.obs_frame[k]), win.obs_z[k])
                for k in range(int(win.lm_obs_begin[l]), int(win.lm_obs_begin[l + 1]))]
        obs.sort(key=lambda o: o[0])          # keypoint_map is ordered by frame id
        qsum, qn = 0.0, 0.0
        for f, z in obs:
            qc = qmul(st.q[f], win.cam_q_cs)
            pc = st.p[f] + qrot(st.q[f], win.cam_p_cs)
            y = qrot(qconj(qc), x - pc)
            if y[2] <= 1.0e-3 or y[2] > 50:
                valid[l] = False
                break
            d = np.array([(y[0] / y[2] - z[0]) * fx, (y[1] / y[2] - z[1]) * fy])
            qsum += np.sqrt(d @ d)
            qn += 1.0
        if valid[l]:
            quality[l] = qsum / max(qn, 1.0)
    return valid, quality


def reprojection_error(win, st):
    """BundleAdjustor::compute_reprojection_error (bundle_adjustor.cpp:321-336) over the window's landmarks, which are
    the TF_VALID tracks the shim packs: the mean pixel error of every observation (anchor included) of every landmark.
    No depth test: a landmark the post-pass would reject still counts, in the sum and in the count."""
    fx, fy = win.K_fx, win.K_fy
    qsum, qn = 0.0, 0
    for l in range(win.M):
        a = int(win.lm_anchor[l])
        qa = qmul(st.q[a], win.cam_q_cs)
        x = qrot(qa, np.array([win.lm_z_ref[l][0], win.lm_z_ref[l][1], 1.0])) / st.rho[l] + st.p[a] + qrot(st.q[a], win.cam_p_cs)
        obs = [(a, win.lm_z_ref[l])] + [(int(win.obs_frame[k]), win.obs_z[k])
                                        for k in range(int(win.lm_obs_begin[l]), int(win.lm_obs_begin[l + 1]))]
        for f, z in obs:
            y = qrot(qconj(qmul(st.q[f], win.cam_q_cs)), x - st.p[f] - qrot(st.q[f], win.cam_p_cs))
            d = np.array([(y[0] / y[2] - z[0]) * fx, (y[1] / y[2] - z[1]) * fy])
            qsum += np.sqrt(d @ d)
            qn += 1
    return qsum / max(qn, 1)


# ----------------------------------------------------------------------- marginaliser
def marginalize(win, st, index=0):
    """bundle_adjustor.cpp:348-599.  `win.lm_in_victim[M]` flags the landmarks observed by
    the victim frame (only those contribute, :454-457).  No robust loss, no plane factors,
    FF_FIX_POSE ignored (quirk Q3); all in-window observations of a victim-seen landmark
    are linearised (quirk Q2).  Returns (S[15(N-1),15(N-1)], e[15(N-1)], Hm, bm) where
    Hm,bm is the information before the eigen-factorisation (for well-posed comparisons)."""
    N = win.N
    n = 15 * N
    H = np.zeros((n, n))
    b = np.zeros(n)
    # prior :369-413
    if win.n_prior > 0:
        r, J = marginalization_evaluate(win, st, True)
        Jf = np.zeros((len(r), n))
        for i in range(win.n_prior):
            f = int(win.prior_frames[i])
            Jf[:, 15 * f:15 * f + 15] = J[:, 15 * i:15 * i + 15]
        H += Jf.T @ Jf
        b += Jf.T @ r
    # IMU factors adjacent to the victim :416-450
    for m in range(win.n_imu):
        i, j = int(win.imu_frame_i[m]), int(win.imu_frame_j[m])
        if j != index and j != index + 1:
            continue
        r, J = preintegration_evaluate(st.q[i], st.p[i], st.v[i], st.bg[i], st.ba[i],
                                       st.q[j], st.p[j], st.v[j], st.bg[j], st.ba[j],
                                       imu_record(win, m), win.imu_q_cs, win.imu_p_cs, True)
        sl = np.r_[15 * i:15 * i + 15, 15 * j:15 * j + 15]
        H[np.ix_(sl, sl)] += J.T @ J
        b[sl] += J.T @ r
    # reprojection factors of victim-seen landmarks :453-533, landmark Schur :536-545
    for l in range(win.M):
        if not win.lm_in_victim[l]:
            continue
        a = int(win.lm_anchor[l])
        mat, vec = 0.0, 0.0
        h = {}
        for k in range(int(win.lm_obs_begin[l]), int(win.lm_obs_begin[l + 1])):
            t = int(win.obs_frame[k])
            r, Jqt, Jpt, Jqr, Jpr, Jrho = reprojection_evaluate(
                st.q[t], st.p[t], st.q[a], st.p[a], st.rho[l], win.obs_z[k], win.lm_z_ref[l],
                win.cam_q_cs, win.cam_p_cs, win.sqrt_inv_cov, True)
            Jt = np.hstack([Jqt, Jpt])
            Jr = np.hstack([Jqr, Jpr])
            st_, sr_ = slice(15 * t, 15 * t + 6), slice(15 * a, 15 * a + 6)
            H[st_, st_] += Jt.T @ Jt
            H[sr_, st_] += Jr.T @ Jt
            H[st_, sr_] += Jt.T @ Jr
            H[sr_, sr_] += Jr.T @ Jr
            b[st_] += Jt.T @ r
            b[sr_] += Jr.T @ r
            mat += float(Jrho @ Jrho)
            vec += float(Jrho @ r)
            h[t] = h.get(t, np.zeros(6)) + Jrho @ Jt
            h[a] = h.get(a, np.zeros(6)) + Jrho @ Jr
        if mat == 0.0 or not np.isfinite(1.0 / mat):
            continue
        inv = 1.0 / mat
        for fi, hi in h.items():
            for fj, hj in h.items():
                H[15 * fi:15 * fi + 6, 15 * fj:15 * fj + 6] -= np.outer(hi, hj) * inv
            b[15 * fi:15 * fi + 6] -= hi * inv * vec
    # frame Schur :547-581
    v = slice(15 * index, 15 * index + 15)
    keep = np.r_[0:15 * index, 15 * index + 15:n]
    inv_vv = np.linalg.inv(H[v, v])
    Hk = H[np.ix_(keep, keep)] - H[keep][:, v] @ inv_vv @ H[v][:, keep]
    bk = b[keep] - H[keep][:, v] @ inv_vv @ b[v]
    # the reference mirrors the upper-right block into the lower-left (:572-577)
    if 0 < index < N - 1:
        i0 = 15 * index
        Hk[i0:, :i0] = Hk[:i0, i0:].T
    # eigen factorisation :583-590
    lam, V = np.linalg.eigh(Hk)
    pos = lam > 1.0e-8
    lam_c = np.where(pos, lam, 0.0)
    lam_inv = np.where(pos, 1.0 / np.where(pos, lam, 1.0), 0.0)
    S = np.sqrt(lam_c)[:, None] * V.T
    e = np.sqrt(lam_inv) * (V.T @ bk)
    return S, e, Hk, bk
