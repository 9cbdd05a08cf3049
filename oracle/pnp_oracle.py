"""TEST INFRASTRUCTURE ONLY -- fp64 NumPy restatement of PVIO's visual-inertial PnP
(pvio/src/pvio/estimation/pnp.cpp:32-100): a single-frame ceres::Solve over the new frame's pose
(and, with use_inertial, its v / bg / ba) with
  * PreIntegrationPriorCost  (estimation/ceres/preintegration_error_cost.h:167-206): the IMU factor
    between last_frame (constant) and the frame, no loss;
  * PoseOnlyReprojectionErrorCost / PoseOnlyReprojectionXYZErrorCost
    (estimation/ceres/reprojection_error_cost.h:128-203) with CauchyLoss(1.0): the landmark is a
    constant world point (Track::get_landmark_point(), or the plane-cast point for TF_PLANE tracks).
The minimiser is oracle.ba_oracle.trust_region (Ceres dogleg restatement, parity unpinned).
Only tests/ and bench.py's CPU-baseline legs may import this module."""
import numpy as np
from .lie import hat, qmat, qconj, qrot, quat_plus
from . import ba_oracle as bo


def reproj_xyz(q, p, x_w, z, cam_q, cam_p, W, jac=True):
    """reprojection_error_cost.h:168-197 (PoseOnlyReprojectionXYZErrorCost::Evaluate)."""
    y_c = qrot(qconj(q), x_w - p)                                 # :174
    y = qrot(qconj(cam_q), y_c - cam_p)                           # :175
    r = W @ (y[:2] / y[2] - z)                                    # :180,:195
    if not jac:
        return [r]
    zz = y[2]
    dproj = np.array([[1 / zz, 0, -y[0] / zz ** 2], [0, 1 / zz, -y[1] / zz ** 2]])
    A = W @ dproj                                                 # :182-185
    Jq = A @ qmat(qconj(cam_q)) @ hat(y_c)                        # :188
    Jp = -A @ qmat(qmul_conj(cam_q, q))                           # :192
    return [r, np.hstack([Jq, Jp])]


def qmul_conj(cam_q, q):
    """(q_cs^-1 * q^-1) as a quaternion."""
    from .lie import qmul
    return qmul(qconj(cam_q), qconj(q))


class PnpProblem:
    def __init__(self, last, imu, pts, zs, cam_q, cam_p, imu_q, imu_p, W, use_inertial, cauchy_a=1.0):
        self.last, self.imu, self.pts, self.zs = last, imu, np.asarray(pts), np.asarray(zs)
        self.cam_q, self.cam_p, self.imu_q, self.imu_p, self.W = cam_q, cam_p, imu_q, imu_p, np.asarray(W).reshape(2, 2)
        self.use_inertial, self.a = use_inertial, cauchy_a
        self.idx = np.arange(15 if use_inertial else 6)

    def blocks(self, x, jac=True):
        q, p, v, bg, ba = x[0:4], x[4:7], x[7:10], x[10:13], x[13:16]
        if self.use_inertial:
            lq, lp, lv, lbg, lba = self.last[0:4], self.last[4:7], self.last[7:10], self.last[10:13], self.last[13:16]
            imu = dict(self.imu, bg0=lbg, ba0=lba)                # frame_i_0 aliases the constant frame_i
            out = bo.preintegration_evaluate(lq, lp, lv, lbg, lba, q, p, v, bg, ba, imu, self.imu_q, self.imu_p, jac)
            yield out[0], (out[1][:, 15:] if jac else None), 0.5 * float(out[0] @ out[0])
        for x_w, z in zip(self.pts, self.zs):
            out = reproj_xyz(q, p, x_w, z, self.cam_q, self.cam_p, self.W, jac)
            sc, cost = bo.corrector_scale(out[0], self.a)
            J = None
            if jac:
                J = np.zeros((2, 15))
                J[:, :6] = out[1] * sc
            yield out[0] * sc, J, cost

    def normal(self, x):
        H, g, cost = np.zeros((15, 15)), np.zeros(15), 0.0
        for r, J, c in self.blocks(x):
            H += J.T @ J
            g += J.T @ r
            cost += c
        return H, g, cost

    def cost(self, x):
        return sum(c for _, _, c in self.blocks(x, jac=False))

    @staticmethod
    def plus(x, dx):
        o = x.copy()
        o[0:4] = quat_plus(x[0:4], dx[0:3])
        o[4:16] = x[4:16] + dx[3:15]
        return o

    def ambient(self, x):
        return x if self.use_inertial else x[:7]


def pnp_solve(frame, last, imu, pts, zs, cam_q, cam_p, imu_q, imu_p, W, use_inertial=True, max_iter=10,
              radius0=1.0e4, verbose=False, cauchy_a=1.0):
    """frame / last: 16-vectors (q xyzw, p, v, bg, ba).  cauchy_a: the scale of the reprojection blocks' CauchyLoss.
    Returns (frame', summary)."""
    prob = PnpProblem(np.asarray(last, float), imu, pts, zs, cam_q, cam_p, imu_q, imu_p, W, use_inertial, cauchy_a)
    return bo.trust_region(prob.normal, prob.cost, prob.plus, prob.ambient, np.array(frame, float), prob.idx, 15,
                           max_iter, radius0, verbose)
