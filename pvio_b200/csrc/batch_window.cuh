// The pieces of the resident batched windows (batch_window.cu) that other calls on the slots share: the kernels' view of
// the track table, the CTA scan, the camera pose and world point of a slot row, and the row of a track id in a slot's
// host mirror.  Used by batch_window.cu and plane_ransac.cu; their calls stage through Stage (api_internal.h) in
// BatchWindows::stage and BatchWindows::scratch.
#pragma once

#include <algorithm>

#include "api_internal.h"
#include "quat.cuh"

namespace pvio {

// the handle's arrays (the plane tables null until a slot has plane tracks), the track table and the post-pass results
struct BwArgs : BatchArrays {
    int32_t *tid;
    uint32_t *tmask;
    double *trho;
    double2 *tz;
    uint8_t *tvalid;
    double *tqual;
    int8_t *trole;
    double *tplane;
    int32_t *lm_row;
    const uint8_t *valid;
    const double *quality;
    double *imu_s, *imu_aux;
    int Scap;
    int32_t *tkp;
};

constexpr int kBwThreads = 256;
constexpr int kBwWarps = kBwThreads / 32;

// exclusive scan of one int per thread over the CTA (kBwThreads); total: the sum
__device__ inline int bw_block_scan(int v, int *sh, int &total) {
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    int x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= o) x += y; }
    if (lane == 31) sh[wv] = x;
    __syncthreads();
    if (threadIdx.x == 0) { int s = 0; for (int k = 0; k < kBwWarps; ++k) { const int t = sh[k]; sh[k] = s; s += t; } sh[kBwWarps] = s; }
    __syncthreads();
    const int r = sh[wv] + x - v;
    total = sh[kBwWarps];
    __syncthreads();
    return r;
}

// the kernels' view of the handle's arrays and the track table
template <>
BwArgs launch_args<BwArgs>(const Handle *h);

__device__ inline void bw_cam_pose(const double *fs, const WinConst &c, double *qc, double *pc) {
    bw_qmul(fs, c.cam_q, qc);
    double t[3];
    bw_qrot(fs, c.cam_p, t);
    for (int i = 0; i < 3; ++i) pc[i] = fs[4 + i] + t[i];
}
// the world point at inverse depth rho along keypoint (zx, zy) of the camera at pose (qc, pc) (Track::get_landmark_point)
__device__ __forceinline__ void bw_world_point(const double *qc, const double *pc, double zx, double zy, double rho,
                                               double *x) {
    const double ray[3] = {zx / rho, zy / rho, 1.0 / rho};
    double y[3];
    bw_qrot(qc, ray, y);
    for (int i = 0; i < 3; ++i) x[i] = y[i] + pc[i];
}
// Track::get_landmark_point() of track-table row R of the slot whose frames are fr: its anchor (lowest) frame's camera
// pose applied to the anchor keypoint at the row's inverse depth
__device__ __forceinline__ void bw_landmark_point(const BwArgs &a, size_t R, const double *fr, const WinConst &c, double *x) {
    const int an = __ffs(a.tmask[R]) - 1;
    const double2 z = a.tz[R * a.Ncap + an];
    const double rho = a.trho[R];
    double qc[4], pc[3];
    bw_cam_pose(fr + an * kFrameStride, c, qc, pc);
    bw_world_point(qc, pc, z.x, z.y, rho, x);
}
// the camera matrix [R | T] of a camera pose (R = q^-1, T = -R p, track.cpp:90-95), row-major 3 x 4
__device__ inline void loc_camera_matrix(const double *qc, const double *pc, double *P) {
    const double qi[4] = {-qc[0], -qc[1], -qc[2], qc[3]};
    for (int j = 0; j < 3; ++j) {
        const double e[3] = {j == 0 ? 1.0 : 0.0, j == 1 ? 1.0 : 0.0, j == 2 ? 1.0 : 0.0};
        double col[3];
        bw_qrot(qi, e, col);
        for (int i = 0; i < 3; ++i) P[4 * i + j] = col[i];
    }
    double t[3];
    bw_qrot(qi, pc, t);
    for (int i = 0; i < 3; ++i) P[4 * i + 3] = -t[i];
}

// the row of track `id` in a slot's host mirror, -1 for an unknown or dead track
inline int find_row(const WinSlot &s, int32_t id) {
    const auto it = std::lower_bound(s.ids.begin(), s.ids.end(), id);
    return (it == s.ids.end() || *it != id) ? -1 : (int)(it - s.ids.begin());
}

}  // namespace pvio
