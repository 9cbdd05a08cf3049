// The pieces of the resident batched windows that their files share: the kernels' view of the track table, the staged
// records of the edit, re-layout and set_imu kernels, the CTA scan, the camera pose and world point of a slot row, and the
// host side's slot checks and re-layout, defined in batch_window.cu.  Used by batch_window.cu, bw_frame.cu, bw_query.cu,
// bw_snapshot.cu and plane_ransac.cu; their calls stage through Stage (api_internal.h) in BatchWindows::stage / scratch.
#pragma once

#include <algorithm>
#include <cmath>

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
// the inverse depth of world point x in the camera at pose (qc, pc)
__device__ __forceinline__ double bw_inv_depth(const double *qc, const double *pc, const double *x) {
    const double qi[4] = {-qc[0], -qc[1], -qc[2], qc[3]};
    double d[3], y[3];
    for (int i = 0; i < 3; ++i) d[i] = x[i] - pc[i];
    bw_qrot(qi, d, y);
    return 1.0 / y[2];
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

// ------------------------------------------------------------------------ staged records (host -> device)
struct BwEdit {                       // one slot's edit, applied by bw_edit_kernel
    int32_t slot, N_old, T_old, replace_last;
    int32_t n_rm, rm_off;             // rows of the table BEFORE compaction
    int32_t frame, has_imu, x_off;    // new frame index (-1: none); its state [16] (+ IMU record) at doubles x_off
    int32_t n_new, new_off, n_obs, obs_off;
    int32_t out_off;                  // ints of the result: live rows after the edit, then the new ids
};
struct BwNew { int32_t row, id, frame, pad; double zx, zy, rho; };
struct BwObs { int32_t row, frame; double zx, zy; };
struct BwLayout { int32_t slot, N, T, fixed, n_prior, inertial, n_planes, smax; };  // a slot's window as the kernels rebuild
                                                                                    // it; smax: its longest sample list
struct BwImu {                                    // a factor with samples: n rows at row off (staged rows in set_imu,
    int32_t slot, factor, n, off;                 // rows of the sample store in a solve's work list)
    __device__ int begin() const { return off; }
    __device__ int end() const { return off + n; }
};
constexpr int kImuAux = 37;                                             // per factor: t_end, noise [4][9]

// One CTA per edit (each names a different slot): replace_last and removals clear mask bits, the table is compacted, then
// the new frame, the new tracks (appended) and the observations are written.  out: live rows, then the ids stored.
__global__ void __launch_bounds__(kBwThreads) bw_edit_kernel(BwArgs a, const BwEdit *eds, const int32_t *rm, const BwNew *nw,
                                                              const BwObs *ob, const double *x, int32_t *out);
// One CTA per set_imu record: the factor's samples, t_end and noise from the upload into the slot
__global__ void __launch_bounds__(kBwThreads) bw_set_imu_kernel(BwArgs a, const BwImu *recs, const double *smp,
                                                                const double *aux);

// a factor as imu_integrate_warp reads it: the sample rows [J.begin(), J.end()) of a job, t_end in aux[0], the noise at
// aux + 1, its record r.  The rows are read from the job where imu_integrate_warp asks for them.
template <typename Job>
struct BwFactor {
    const Job &J;
    const double *samples, *noise, *aux;
    double *r;
    __device__ int begin() const { return J.begin(); }
    __device__ int end() const { return J.end(); }
    __device__ double t_end() const { return aux[0]; }
    __device__ double *rec() const { return r; }
};

constexpr int kBwImuWarps = 4;

// PreIntegrator::predict (preintegrator.cpp:102-109): the state y [16] a factor of length dt and delta (dq, dp, dv)
// reaches from the state x [16]; the biases carry over
__device__ __forceinline__ void bw_imu_predict(const double *x, double dt, const double *dq, const double *dp,
                                               const double *dv, double *y) {
    const double g[3] = {0.0, 0.0, -9.80665};                // PVIO_GRAVITY_NOMINAL, as ba_factors.cuh
    double qdv[3], qdp[3];
    bw_qrot(x, dv, qdv);
    bw_qrot(x, dp, qdp);
    for (int k = 0; k < 3; ++k) {
        y[7 + k] = x[7 + k] + g[k] * dt + qdv[k];
        y[4 + k] = x[4 + k] + 0.5 * g[k] * dt * dt + x[7 + k] * dt + qdp[k];
    }
    bw_qmul(x, dq, y);
    for (int k = 10; k < 16; ++k) y[k] = x[k];
}

// ------------------------------------------------------------------------ host side (batch_window.cu)
// the row of track `id` in a slot's host mirror, -1 for an unknown or dead track
inline int find_row(const WinSlot &s, int32_t id) {
    const auto it = std::lower_bound(s.ids.begin(), s.ids.end(), id);
    return (it == s.ids.end() || *it != id) ? -1 : (int)(it - s.ids.begin());
}

inline bool all_finite(const double *x, int64_t n) {
    for (int64_t k = 0; k < n; ++k)
        if (!std::isfinite(x[k])) return false;
    return true;
}

// the track table, allocated with the first reset or restore of a slot
int ensure_bw(Handle *h);
// the sample store for factors of up to S samples: t_end / noise allocated with the first set_imu, the samples grown to
// the longest list seen, every slot's samples copied across to the new stride on the device
int ensure_imu_store(Handle *h, int S);
// 0, or PVIO_B200_EINVAL when slot window s exceeds the handle's capacities
int check_window(Handle *h, const WinSlot &s);
// the n slots of a list: distinct and resident (what: the message for a bad list)
int check_slots(Handle *h, int n, const int32_t *slots, const char *what);
// the rows of a mirror whose frame mask, shifted down by `shift` frames, is not 0, in order, with their shifted masks
void compact_rows(WinSlot &s, int shift);
// plane-table capacity for the windows the n slots of a call will hold, before anything of the call is staged
int ensure_plane_tables(Handle *h, const std::vector<WinSlot> &next);
// the mirrors of a call that has run into their slots, with their host headers
void commit(Handle *h, const int32_t *slots, std::vector<WinSlot> &next);

// the re-layout of a call's slots to their new mirrors next[]: their BwLayouts and the slot list go with the call's
// upload; launch rebuilds the packed windows once the call's own kernels are queued
struct Relayout {
    std::vector<BwLayout> lays;
    Stage::Sec<BwLayout> lay;
    Stage::Sec<int32_t> slots;
    Relayout(Stage &S, const int32_t *sl, const std::vector<WinSlot> &next);
    int launch(Handle *h, const Stage &S, bool prior) const;
};

// The opening of a call on n records: the handle, the record list and, with `gather`, the records' slots, which must be
// distinct resident slots.  open is false when the call returns at once, with rc (0 for an empty list).  bad(why):
// PVIO_B200_EINVAL with the message "<call>: <why>".
struct BwCall {
    Handle *h;
    const char *what;
    std::vector<int32_t> slots;
    int rc = 0;
    BwCall(pvio_b200_handle hh, const char *call) : h(reinterpret_cast<Handle *>(hh)), what(call) {}
    int bad(const char *why) const { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); }
    template <typename R>
    bool open(int n, const R *records, bool gather = true) {
        if (!h) rc = PVIO_B200_EINVAL;
        else if (n < 0 || (n > 0 && !records)) rc = bad("bad record list");
        if (rc || n == 0) return false;
        for (int i = 0; gather && i < n; ++i) slots.push_back(records[i].slot);
        if (gather) rc = check_slots(h, n, slots.data(), what);
        return rc == 0;
    }
};

}  // namespace pvio
