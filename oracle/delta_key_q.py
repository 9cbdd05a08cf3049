"""delta_key_q of Frame::track_keypoints (frame.cpp:98) in NumPy: (cam_q^* imu_q dq imu_q^* cam_q)^*, quaternions
(x, y, z, w), each Hamilton product summed in the order of Eigen's scalar quat_product, left to right.  The device
composes it in this order without contraction (feature_track.cu, ft_predict_kernel); Eigen's SSE product in a
reference build may differ from it in the last bit."""
import numpy as np


def quat_product(a, b):
    """Eigen's scalar quat_product (Geometry/Quaternion.h) of (x, y, z, w) quaternions, term by term in its order"""
    ax, ay, az, aw = (float(v) for v in a)
    bx, by, bz, bw = (float(v) for v in b)
    w = aw * bw - ax * bx - ay * by - az * bz
    x = aw * bx + ax * bw + ay * bz - az * by
    y = aw * by + ay * bw + az * bx - ax * bz
    z = aw * bz + az * bw + ax * by - ay * bx
    return np.array([x, y, z, w])


def conjugate(q):
    return np.array([-q[0], -q[1], -q[2], q[3]], dtype=np.float64)


def delta_key_q(cam_q, imu_q, dq):
    """the rotation that takes a keypoint of the previous frame's camera to the new frame's, both cameras on the same
    body with extrinsics cam_q (camera to body) and imu_q (IMU to body), dq the pre-integrated IMU rotation"""
    u = quat_product(conjugate(cam_q), imu_q)
    u = quat_product(u, dq)
    u = quat_product(u, conjugate(imu_q))
    u = quat_product(u, cam_q)
    return conjugate(u)
