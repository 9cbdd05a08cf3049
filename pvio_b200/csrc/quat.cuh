// Quaternions on the device: (x, y, z, w), Hamilton product, q * v = rotate -- the reference's Eigen conventions
// (estimation/state.h).  Used by the resident windows (batch_window.cu) and the feature tracker's initial guesses
// (feature_track.cu); each file's -fmad setting decides whether the products are contracted.
#pragma once

namespace pvio {

__device__ inline void bw_qmul(const double *a, const double *b, double *o) {
    o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    o[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
    o[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
    o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
// the Hamilton product summed term by term in the order of Eigen's scalar quat_product (Geometry/Quaternion.h), for
// arithmetic that must match a reference build's Eigen products bit for bit in a -fmad=false unit
__device__ inline void eigen_qmul(const double *a, const double *b, double *o) {
    o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
    o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
}
__device__ inline void bw_qrot(const double *q, const double *v, double *o) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2.0 * (y * v[2] - z * v[1]), ty = 2.0 * (z * v[0] - x * v[2]), tz = 2.0 * (x * v[1] - y * v[0]);
    o[0] = v[0] + w * tx + (y * tz - z * ty);
    o[1] = v[1] + w * ty + (z * tx - x * tz);
    o[2] = v[2] + w * tz + (x * ty - y * tx);
}

}  // namespace pvio
