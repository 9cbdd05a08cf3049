"""Host mirror of visual_inertial_pnp (pvio/src/pvio/estimation/pnp.cpp:32-100) over the C-ABI:
one kernel launch runs the whole single-frame trust-region solve on the GPU."""
import ctypes as C

import numpy as np

from . import _lib


def imu_record(imu):
    """PreIntegrator outputs (dict as pvio_b200.so3.PreIntegrator.integrate returns) -> [288] record."""
    return _lib.imu_records(imu['dt'], imu['dq'], imu['dp'], imu['dv'], imu['sqrt_inv_cov'], imu['dq_dbg'], imu['dp_dbg'],
                            imu['dp_dba'], imu['dv_dbg'], imu['dv_dba'])[0]


def _fill_problem(pb, keep, last_frame, imu, points, z, cam_q, cam_p, imu_q, imu_p, sqrt_inv_cov, use_inertial,
                  cauchy_a):
    """Fills the CPnpProblem pb; keep (a list) holds the arrays it points into alive until the call returns."""
    pts = np.ascontiguousarray(points, dtype=np.float64).reshape(-1, 3)
    zz = np.ascontiguousarray(z, dtype=np.float64).reshape(-1, 2)
    last = np.ascontiguousarray(last_frame, dtype=np.float64)
    rec = imu_record(imu) if use_inertial else np.zeros(_lib.IMU_STRIDE)
    keep += [pts, zz, last, rec]
    pb.n_points, pb.use_inertial = len(pts), 1 if use_inertial else 0
    pb.cam_q_cs[:], pb.cam_p_cs[:] = list(cam_q), list(cam_p)
    pb.imu_q_cs[:], pb.imu_p_cs[:] = list(imu_q), list(imu_p)
    pb.sqrt_inv_cov[:] = list(np.asarray(sqrt_inv_cov, dtype=np.float64).reshape(4))
    pb.cauchy_a = cauchy_a
    _lib.set_ptrs(pb, points=pts, z=zz, last_frame=last, imu_data=rec)


def visual_inertial_pnp(ba, frame, last_frame, imu, points, z, cam_q, cam_p, imu_q, imu_p, sqrt_inv_cov,
                        use_inertial=True, max_iterations=10, initial_radius=0.0, cauchy_a=1.0):
    """ba: a BundleAdjustor (device handle).  frame / last_frame: 16-vectors (q xyzw, p, v, bg, ba).
    Returns (frame', summary dict)."""
    pb, keep = _lib.CPnpProblem(), []
    _fill_problem(pb, keep, last_frame, imu, points, z, cam_q, cam_p, imu_q, imu_p, sqrt_inv_cov, use_inertial,
                  cauchy_a)
    out = np.array(frame, dtype=np.float64, copy=True)
    opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
    sm = _lib.CSummary()
    ba._ck(ba.lib.pvio_b200_pnp_solve(ba.h, C.byref(pb), _lib.ptr(out), C.byref(opt), C.byref(sm)))
    return out, _lib.summary(sm)


def batch_visual_inertial_pnp(ba, problems, max_iterations=10, initial_radius=0.0):
    """visual_inertial_pnp for n independent problems (e.g. the new frame of n sequences) in one kernel launch.
    problems: dicts with the keys synthetic.synth.make_pnp returns (frame, last, imu, pts, zs, cam_q, cam_p, imu_q,
    imu_p, W), plus optional use_inertial (default True) and cauchy_a (default 1.0).  The solver options are shared.
    Returns (frames [n, 16], [summary dict] * n); solve_seconds is the device time of the whole batch."""
    n = len(problems)
    pbs, keep = (_lib.CPnpProblem * max(n, 1))(), []
    frames = np.zeros((n, _lib.FRAME_STRIDE))
    for i, d in enumerate(problems):
        _fill_problem(pbs[i], keep, d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'], d['imu_q'],
                      d['imu_p'], d['W'], d.get('use_inertial', True), d.get('cauchy_a', 1.0))
        frames[i] = d['frame']
    opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
    sms = (_lib.CSummary * max(n, 1))()
    ba._ck(ba.lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), _lib.FRAME_STRIDE, C.byref(opt), sms))
    return frames, [_lib.summary(sms[i]) for i in range(n)]
