"""Reference of the resident slots' map output (pvio_b200_batch_window_landmarks): the world point of a landmark of a
packed window (Track::get_landmark_point) and its 3 x 3 covariance, in two forms:
  point_covariance       dense: Sigma over the free coordinates (cov_oracle.covariance) propagated through the Jacobian
                         of the world point with respect to the anchor's free pose coordinates and rho_l, taken by
                         central differences through ba_oracle.apply_step (independent of the xi derivation);
  point_covariance_elim  the elimination form the device uses: Sigma_xi = T Sigma_delta T^T of the frames (the inverse of
                         the landmark-reduced system), h_l in xi coordinates and H_ll, with
                         Sigma_x = X Sigma_aa X^T - X C c^T - c C^T X^T + c c^T Var(rho), C = -(Sigma_xi h_l)_a / H_ll."""
import numpy as np

from oracle import ba_oracle, cov_oracle
from oracle.lie import hat, qmat, qrot


def landmark_point(win, st, l):
    """Track::get_landmark_point() of landmark l: the anchor frame's camera pose applied to [z_anchor; 1] / rho_l
    (reprojection_error_cost.h:58-60)."""
    a = int(win.lm_anchor[l])
    z = win.lm_z_ref[l]
    y = np.array([z[0], z[1], 1.0]) / st.rho[l]
    return qrot(st.q[a], qrot(win.cam_q_cs, y) + win.cam_p_cs) + st.p[a]


def camera_pose(win, st, f):
    """the camera pose (q, p) in the world of frame f"""
    from oracle.lie import qmul
    return qmul(st.q[f], win.cam_q_cs), st.p[f] + qrot(st.q[f], win.cam_p_cs)


def _coords(win, l):
    """the local coordinates the world point of landmark l depends on: the anchor's pose (when free) and rho_l"""
    free = ba_oracle.free_mask(win)
    a = int(win.lm_anchor[l])
    return [c for c in range(15 * a, 15 * a + 6) if free[c]] + [15 * win.N + l]


def point_jacobian(win, st, l, h=1e-5):
    """d x_l / d(coordinates of _coords) by central differences through apply_step (relative step on rho)"""
    cols = _coords(win, l)
    J = np.zeros((3, len(cols)))
    for k, c in enumerate(cols):
        d = h * (abs(st.rho[l]) if c >= 15 * win.N else 1.0)
        e = np.zeros(ba_oracle.local_dim(win))
        e[c] = d
        J[:, k] = (landmark_point(win, ba_oracle.apply_step(win, st, e), l)
                   - landmark_point(win, ba_oracle.apply_step(win, st, -e), l)) / (2 * d)
    return J


def point_covariance(win, st, tracks, Sig=None):
    """[len(tracks), 3, 3] the dense form; NaN for an entry that is None / < 0.  Sig: cov_oracle.covariance's Sigma over
    the free coordinates (computed with refinement when None)."""
    if Sig is None:
        Sig = cov_oracle.covariance(win, st, [], [], refine=True)[2]
    free = ba_oracle.free_mask(win)
    pos = -np.ones(ba_oracle.local_dim(win), dtype=int)
    pos[free] = np.arange(int(free.sum()))
    out = np.full((len(tracks), 3, 3), np.nan)
    for k, l in enumerate(tracks):
        if l is None or l < 0:
            continue
        p = pos[_coords(win, l)]
        J = point_jacobian(win, st, l)
        out[k] = J @ Sig[np.ix_(p, p)] @ J.T
    return out


def xi_transform(q, p):
    """T of DESIGN 4: xi = T [dtheta; dp] = [R dtheta; -[p]x R dtheta - dp]"""
    R = qmat(q)
    T = np.zeros((6, 6))
    T[:3, :3] = R
    T[3:, :3] = -hat(p) @ R
    T[3:, 3:] = -np.eye(3)
    return T


def point_covariance_elim(win, st, tracks):
    """[len(tracks), 3, 3] the elimination form, and Var(rho) [len(tracks)]; NaN for an entry that is None / < 0"""
    H, _, _ = ba_oracle.normal_equations(win, st)
    free = ba_oracle.free_mask(win)
    N = win.N
    ff = np.flatnonzero(free[:15 * N])
    fl = 15 * N + np.flatnonzero(free[15 * N:])
    Hff, Hfl, Hll = H[np.ix_(ff, ff)], H[np.ix_(ff, fl)], H[np.ix_(fl, fl)]
    Sig_ff = np.linalg.inv(Hff - Hfl @ np.diag(1.0 / np.diag(Hll)) @ Hfl.T)
    # Sigma_delta over every frame's 6 pose coordinates (0 where not free), then Sigma_xi = T Sigma_delta T^T
    pose = np.concatenate([15 * f + np.arange(6) for f in range(N)])
    Sd = np.zeros((15 * N, 15 * N))
    Sd[np.ix_(ff, ff)] = Sig_ff
    Sd = Sd[np.ix_(pose, pose)]
    T = np.zeros((6 * N, 6 * N))
    for f in range(N):
        T[6 * f:6 * f + 6, 6 * f:6 * f + 6] = xi_transform(st.q[f], st.p[f])
    Sxi = T @ Sd @ T.T
    Tinv_t = np.linalg.inv(T).T
    out, var = np.full((len(tracks), 3, 3), np.nan), np.full(len(tracks), np.nan)
    for k, l in enumerate(tracks):
        if l is None or l < 0:
            continue
        c = 15 * N + l
        hd = np.where(free[pose], H[pose, c], 0.0)          # coupling to the free pose coordinates, delta coordinates
        h = Tinv_t @ hd                                       # ... in xi coordinates
        hll = H[c, c]
        v = Sxi @ h
        var[k] = 1.0 / hll + h @ v / hll ** 2
        a = int(win.lm_anchor[l])
        C = -v[6 * a:6 * a + 6] / hll
        x = landmark_point(win, st, l)
        ca = camera_pose(win, st, a)[1]
        cl = -(x - ca) / st.rho[l]
        X = np.hstack([hat(x), np.eye(3)])
        Saa = Sxi[6 * a:6 * a + 6, 6 * a:6 * a + 6]
        XC = X @ C
        out[k] = X @ Saa @ X.T - np.outer(XC, cl) - np.outer(cl, XC) + np.outer(cl, cl) * var[k]
    return out, var
