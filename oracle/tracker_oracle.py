"""TEST INFRASTRUCTURE (CPU oracle) -- the host steps of SlidingWindowTracker::track that
pvio_b200_batch_window_track_frame runs on the device, restated in NumPy fp64 on the arrays the call takes:
PreIntegrator::predict (pvio/src/pvio/estimation/preintegrator.cpp:102-109) and SlidingWindowTracker::keyframe_check
(pvio/src/pvio/core/sliding_window_tracker.cpp:255-296).  Only tests/ and tools/ may import it."""
import numpy as np

from . import lie

GRAVITY = np.array([0.0, 0.0, -9.80665])                      # PVIO_GRAVITY_NOMINAL (common.h)


def predict(state16, rec):
    """PreIntegrator::predict: the new frame's state [16] (q, p, v, bg, ba) from the old frame's state and the [288]
    record (PVIO_B200_IMU_* layout) of the factor between them.  Biases copied; the quaternion is not normalised."""
    x, rec = np.asarray(state16, dtype=np.float64), np.asarray(rec, dtype=np.float64)
    q, p, v = x[0:4], x[4:7], x[7:10]
    dt, dq, dp, dv = rec[0], rec[1:5], rec[5:8], rec[8:11]
    out = x.copy()
    out[7:10] = v + GRAVITY * dt + lie.qrot(q, dv)
    out[4:7] = p + 0.5 * GRAVITY * dt * dt + v * dt + lie.qrot(q, dp)
    out[0:4] = lie.qmul(q, dq)
    return out


def keyframe_check(z_i, z_j, dq, cam_q_cs, imu_q_cs, fx, fy, cx, cy, skipped):
    """z_i, z_j: [m][2] the normalised keypoints of the m tracks of the new frame that have a keypoint in frame_i, in
    frame_i and in the new frame; dq: the new frame's pre-integrated rotation; the extrinsics and camera matrix are
    frame_i's and the new frame's (the same camera); skipped: the tracker's counter before the check.
    Returns (keyframe, parallax (NaN with fewer than 50 pairs), m, skipped after the check)."""
    z_i = np.asarray(z_i, dtype=np.float64).reshape(-1, 2)
    z_j = np.asarray(z_j, dtype=np.float64).reshape(-1, 2)
    cq, iq = np.asarray(cam_q_cs, dtype=np.float64), np.asarray(imu_q_cs, dtype=np.float64)
    q = lie.qmul(lie.qmul(lie.qmul(lie.qmul(lie.qconj(cq), iq), np.asarray(dq, dtype=np.float64)), lie.qconj(iq)), cq)
    qij = lie.qconj(q)                                                     # :267
    par = []
    for a, b in zip(z_i, z_j):                                             # :269-277
        y = lie.qrot(qij, np.array([a[0], a[1], 1.0]))
        pi = np.array([y[0] / y[2] * fx + cx, y[1] / y[2] * fy + cy])
        pj = np.array([b[0] * fx + cx, b[1] * fy + cy])
        par.append(np.linalg.norm(pi - pj))
    m, parallax = len(par), np.nan
    if m < 50:                                                             # :278-280
        keyframe = True
    else:
        parallax = sorted(par)[m * 4 // 5]                                 # :281-282
        keyframe = parallax > 50
        if not keyframe:
            skipped += 1
    if skipped > 10:                                                       # :290-292
        keyframe = True
    if keyframe:
        skipped = 0
    return keyframe, parallax, m, skipped
