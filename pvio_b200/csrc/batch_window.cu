// Resident sliding windows of the batched slots (pvio_b200_batch_window_*), and the single resident window
// (pvio_b200_window_*), which is slot 0 of them.  The window persists between keyframes instead of being rebuilt from
// Map / Frame / Track at every BundleAdjustor::solve (bundle_adjustor.cpp:75-242); its bookkeeping follows map.cpp:76-88
// and track.cpp:32-49.
// A resident slot keeps its whole window on the device -- frame states, IMU records, the prior, and a TRACK TABLE with
// every live track's frame mask, inverse depth and fp64 keypoint per window frame.  Per camera frame the host sends only
// what changed (edit records); the packed tables the solve kernels read (LmRec, ObsRec, rho, WinHdr, the frame-major
// table) are rebuilt from the track table on the device, exactly as pack_window packs the window of the tracks with
// >= 2 observations in id order: stably sorted by anchor (their lowest frame).
//
// The host keeps integers only (frame count, prior size, fixed mask, plane count, the id, frame mask and role of every
// live row), enough to check every call completely before anything is staged, and to know the launch shapes.  The rows
// of a slot's table are its live tracks in id order: removals compact the table (the storage of dead tracks is reused),
// new tracks append.
// Plane factors (bundle_adjustor.cpp:162-196): the role of a row (WinSlot) decides what it is in the solve.  Rows of
// role < 0 with >= 2 observations are the landmarks (role -2 ones stay out of the marginaliser's victim set,
// bundle_adjustor.cpp:456-457); rows of role p >= 0 are the plane tracks of plane p, packed in row (= id) order with all
// their observations, anchor included, into the plane tables the solve kernels read (pt_plane, pt_begin, pt_frame,
// pt_z), with the slot's plane parameters.  The caller decides the roles (pvio_b200_batch_window_set_planes).
// IMU factors with samples (pvio_b200_batch_window_set_imu): a factor's raw samples, t_end and noise stay on the device
// with it, indexed like its record (BatchWindows::imu_s / imu_aux), shift with it in a drop, and are re-integrated at
// the biases its first frame holds on the device before every solve that names the slot (bundle_adjustor.cpp:220-231);
// the host keeps the sample count of each factor.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstddef>
#include <cstring>
#include <memory>
#include <optional>
#include <vector>

#include <math_constants.h>

#include "api_internal.h"
#include "ba_cov_lm.cuh"
#include "batch_window.cuh"
#include "imu.cuh"
#include "imu_factor_cov.cuh"
#include "klt_border.cuh"
#include "tri.cuh"

namespace pvio {

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
struct BwDl { int32_t slot, N, T, pad; int64_t off; };                  // download: bytes into the result area
struct BwPlanes { int32_t slot, n_planes, n_set, set_off, param_off, pad; };   // one set_planes record (n_planes < 0: keep)
struct BwRole { int32_t row, role; double rho; };                       // rho NaN: keep the row's inverse depth
struct BwImu {                                    // a factor with samples: n rows at row off (staged rows in set_imu,
    int32_t slot, factor, n, off;                 // rows of the sample store in a solve's work list)
    __device__ int begin() const { return off; }
    __device__ int end() const { return off + n; }
};
constexpr int kImuAux = 37;                                             // per factor: t_end, noise [4][9]

// stable compaction of rows [0, T) of window w to the rows whose frame mask is not 0; returns the live count.  A row only
// moves down, chunk by chunk: each chunk is read completely before it is written.
__device__ int bw_compact(const BwArgs &a, int w, int T, int *sh) {
    const size_t base = (size_t)w * a.Mcap;
    int carry = 0;
    for (int c0 = 0; c0 < T; c0 += kBwThreads) {
        const int r = c0 + threadIdx.x;
        const bool live = r < T && a.tmask[base + r] != 0u;
        int tot;
        const int d = carry + bw_block_scan(live ? 1 : 0, sh, tot);
        int32_t id = 0, kp = -1; uint32_t m = 0; double rho = 0.0, q = 0.0; uint8_t v = 0; int8_t ro = -1;
        if (live) {
            id = a.tid[base + r]; m = a.tmask[base + r]; rho = a.trho[base + r]; v = a.tvalid[base + r]; q = a.tqual[base + r];
            ro = a.trole[base + r]; kp = a.tkp[base + r];
        }
        __syncthreads();
        if (live && d != r) {
            a.tid[base + d] = id; a.tmask[base + d] = m; a.trho[base + d] = rho; a.tvalid[base + d] = v; a.tqual[base + d] = q;
            a.trole[base + d] = ro; a.tkp[base + d] = kp;
        }
        __syncthreads();
        for (int f = 0; f < a.Ncap; ++f) {
            double2 z = make_double2(0.0, 0.0);
            if (live) z = a.tz[(base + r) * a.Ncap + f];
            __syncthreads();
            if (live && d != r) a.tz[(base + d) * a.Ncap + f] = z;
            __syncthreads();
        }
        carry += tot;
    }
    for (int r = carry + threadIdx.x; r < T; r += kBwThreads) { a.tmask[base + r] = 0u; a.trole[base + r] = -1; a.tkp[base + r] = -1; }
    __syncthreads();
    return carry;
}

// One CTA per edit (each names a different slot): replace_last and removals clear mask bits, the table is compacted, then
// the new frame, the new tracks (appended) and the observations are written.  out: live rows, then the ids stored.
__global__ void __launch_bounds__(kBwThreads) bw_edit_kernel(BwArgs a, const BwEdit *eds, const int32_t *rm, const BwNew *nw,
                                                              const BwObs *ob, const double *x, int32_t *out) {
    __shared__ int sh[kBwWarps + 1];
    const BwEdit e = eds[blockIdx.x];
    const int w = e.slot;
    const size_t base = (size_t)w * a.Mcap;
    if (e.replace_last)
        for (int r = threadIdx.x; r < e.T_old; r += kBwThreads) a.tmask[base + r] &= ~(1u << (e.N_old - 1));
    __syncthreads();
    for (int i = threadIdx.x; i < e.n_rm; i += kBwThreads) a.tmask[base + rm[e.rm_off + i]] = 0u;
    __syncthreads();
    const int T = bw_compact(a, w, e.T_old, sh);
    if (e.frame >= 0) {
        double *fr = a.frames + ((size_t)w * a.Ncap + e.frame) * kFrameStride;
        for (int i = threadIdx.x; i < kFrameStride; i += kBwThreads) fr[i] = x[e.x_off + i];
        if (e.has_imu) {
            double *rec = a.imu_data + ((size_t)w * a.Ncap + e.frame - 1) * kImuStride;
            for (int i = threadIdx.x; i < kImuStride; i += kBwThreads) rec[i] = x[e.x_off + kFrameStride + i];
        }
    }
    for (int i = threadIdx.x; i < e.n_new; i += kBwThreads) {
        const BwNew t = nw[e.new_off + i];
        const size_t R = base + t.row;
        a.tid[R] = t.id; a.tmask[R] = 1u << t.frame; a.trho[R] = t.rho; a.tvalid[R] = 0; a.tqual[R] = 0.0; a.trole[R] = -1;
        a.tz[R * a.Ncap + t.frame] = make_double2(t.zx, t.zy);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < e.n_obs; i += kBwThreads) {      // distinct frames per row: the masks meet in atomicOr only
        const BwObs o = ob[e.obs_off + i];
        atomicOr(&a.tmask[base + o.row], 1u << o.frame);
        a.tz[(base + o.row) * a.Ncap + o.frame] = make_double2(o.zx, o.zy);
    }
    __syncthreads();
    int live = 0;
    for (int r = threadIdx.x; r < T + e.n_new; r += kBwThreads) live += a.tmask[base + r] != 0u ? 1 : 0;
    for (int o = 16; o > 0; o >>= 1) live += __shfl_xor_sync(0xffffffffu, live, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = live;
    __syncthreads();
    if (threadIdx.x == 0) { int s = 0; for (int k = 0; k < kBwWarps; ++k) s += sh[k]; out[e.out_off] = s; }
    for (int i = threadIdx.x; i < e.n_new; i += kBwThreads) out[e.out_off + 1 + i] = a.tid[base + nw[e.new_off + i].row];
}

// the anchor of row r as a landmark (role < 0, >= 2 observations), kMaxFrames for the other rows
__device__ __forceinline__ int bw_lm_anchor(const BwArgs &a, size_t R) {
    const uint32_t m = a.tmask[R];
    return (a.trole[R] < 0 && __popc(m) >= 2) ? __ffs(m) - 1 : kMaxFrames;
}

// One CTA per slot: the packed window from the track table, as pack_window builds it from build_view's window.
__global__ void __launch_bounds__(kBwThreads) bw_layout_kernel(BwArgs a, const BwLayout *lay) {
    __shared__ int sh[kBwWarps + 1];
    __shared__ int cnt[kMaxFrames], first[kMaxFrames], run[kMaxFrames];
    __shared__ int wcnt[kBwWarps][kMaxFrames + 1];
    __shared__ int n_pl;
    const BwLayout L = lay[blockIdx.x];
    const int w = L.slot, N = L.N, T = L.T;
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const size_t base = (size_t)w * a.Mcap;
    if (threadIdx.x < kMaxFrames) { cnt[threadIdx.x] = 0; run[threadIdx.x] = 0; }
    if (threadIdx.x == 0) n_pl = 0;
    __syncthreads();
    for (int r = threadIdx.x; r < T; r += kBwThreads) {
        const int an = bw_lm_anchor(a, base + r);
        if (an < kMaxFrames) atomicAdd(&cnt[an], 1);
        else if (a.trole[base + r] >= 0) atomicAdd(&n_pl, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) { int s = 0; for (int k = 0; k < kMaxFrames; ++k) { first[k] = s; s += cnt[k]; } sh[kBwWarps] = s; }
    __syncthreads();
    const int M = sh[kBwWarps];
    __syncthreads();
    // landmark order: anchor, then row (= id) -- a counting sort, stable chunk by chunk
    for (int c0 = 0; c0 < T; c0 += kBwThreads) {
        const int r = c0 + threadIdx.x;
        const int an = r < T ? bw_lm_anchor(a, base + r) : kMaxFrames;
        for (int i = threadIdx.x; i < kBwWarps * (kMaxFrames + 1); i += kBwThreads) (&wcnt[0][0])[i] = 0;
        __syncthreads();
        const unsigned peers = __match_any_sync(0xffffffffu, an);
        const int rank = __popc(peers & ((1u << lane) - 1u));
        if (rank == 0) wcnt[wv][an] = __popc(peers);
        __syncthreads();
        if (threadIdx.x < kMaxFrames) {
            int s = run[threadIdx.x];
            for (int k = 0; k < kBwWarps; ++k) { const int c = wcnt[k][threadIdx.x]; wcnt[k][threadIdx.x] = s; s += c; }
            run[threadIdx.x] = s;
        }
        __syncthreads();
        if (an < kMaxFrames) a.lm_row[base + first[an] + wcnt[wv][an] + rank] = r;
        __syncthreads();
    }
    // records: LmRec, rho, ObsRec in increasing frame order per landmark
    int carry = 0;
    for (int c0 = 0; c0 < M; c0 += kBwThreads) {
        const int lp = c0 + threadIdx.x;
        const bool ok = lp < M;
        const int row = ok ? a.lm_row[base + lp] : 0;
        const uint32_t m = ok ? a.tmask[base + row] : 0u;
        const int an = ok ? __ffs(m) - 1 : 0;
        const uint32_t seen = m & ~(1u << an);
        const int n = ok ? __popc(seen) : 0;
        int tot;
        const int ob = carry + bw_block_scan(n, sh, tot);
        if (ok) {
            const double2 *z = a.tz + (base + row) * a.Ncap;
            LmRec lr;
            lr.zrx = (float)z[an].x; lr.zry = (float)z[an].y;
            lr.meta = lm_meta(an, (an == 0 && a.trole[base + row] != -2) ? 1 : 0, n, seen);
            lr.obs_begin = ob;
            a.lms[base + lp] = lr;
            a.rho[base + lp] = a.trho[base + row];
            ObsRec *o = a.obs + (size_t)w * a.Kcap + ob;
            int k = 0;
            for (uint32_t s = seen; s; s &= s - 1) {
                const int f = __ffs(s) - 1;
                o[k].zx = (float)z[f].x; o[k].zy = (float)z[f].y;
                ++k;
            }
        }
        carry += tot;
    }
    // plane tracks in row order: plane index, CSR of their observations (every frame of the mask, increasing), fp32
    // keypoints; the host grew the tables to the slot's counts before the launch
    const int T_pl = n_pl;
    if (T_pl > 0) {
        const size_t pb = (size_t)w * a.Tcap, ob0 = (size_t)w * a.Ocap;
        int t_carry = 0, o_carry = 0;
        for (int c0 = 0; c0 < T; c0 += kBwThreads) {
            const int r = c0 + threadIdx.x;
            const int ro = r < T ? a.trole[base + r] : -1;
            const uint32_t m = ro >= 0 ? a.tmask[base + r] : 0u;
            int t_tot, o_tot;
            const int t = t_carry + bw_block_scan(ro >= 0 ? 1 : 0, sh, t_tot);
            const int ob = o_carry + bw_block_scan(__popc(m), sh, o_tot);
            if (ro >= 0) {
                a.pt_plane[pb + t] = ro;
                a.pt_begin[pb + (size_t)w + t] = ob;          // pt_begin: Tcap + 1 entries per window
                const double2 *z = a.tz + (base + r) * a.Ncap;
                int k = 0;
                for (uint32_t s = m; s; s &= s - 1) {
                    const int f = __ffs(s) - 1;
                    a.pt_frame[ob0 + ob + k] = f;
                    a.pt_z[2 * (ob0 + ob + k)] = (float)z[f].x; a.pt_z[2 * (ob0 + ob + k) + 1] = (float)z[f].y;
                    ++k;
                }
            }
            t_carry += t_tot; o_carry += o_tot;
        }
        if (threadIdx.x == 0) a.pt_begin[pb + (size_t)w + T_pl] = o_carry;
    }
    if (a.plane_param)
        for (int i = threadIdx.x; i < 4 * L.n_planes; i += kBwThreads)
            a.plane_param[(size_t)w * a.Pcap * 4 + i] = a.tplane[(size_t)w * a.Pcap * 4 + i];
    WinHdr &H = a.hdr[w];
    for (int i = threadIdx.x; i < kMaxChunks; i += kBwThreads) { H.chunk_begin[i] = 0; H.chunk_meta[i] = 0; }
    __syncthreads();
    if (threadIdx.x == 0) {
        const int n_imu = L.inertial ? max(N - 1, 0) : 0;
        H.N = N; H.M = M; H.K = carry; H.use_inertial = L.inertial;
        H.n_imu = n_imu; H.n_prior = L.inertial ? L.n_prior : 0; H.n_planes = L.n_planes; H.n_ptracks = T_pl;
        H.fixed_mask = L.fixed; H.pad0 = 0; H.pad1 = 0;
        int nch = 0;
        for (int an = 0; an < N; ++an)
            for (int j = 0; j < cnt[an]; j += 32) {
                H.chunk_begin[nch] = first[an] + j;
                H.chunk_meta[nch] = (an << 8) + min(32, cnt[an] - j);
                ++nch;
            }
        H.n_chunks = nch;
        // the mean frame position, summed in frame order as pack_window sums it
        const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
        double o[3] = {0.0, 0.0, 0.0};
        for (int f = 0; f < N; ++f) for (int k = 0; k < 3; ++k) o[k] += fr[f * kFrameStride + 4 + k];
        for (int k = 0; k < 3; ++k) a.cst[w].origin[k] = N > 0 ? o[k] / N : 0.0;
        if (a.imu_idx) {
            for (int k = 0; k < n_imu; ++k) { a.imu_idx[((size_t)w * a.Ncap + k) * 2] = k; a.imu_idx[((size_t)w * a.Ncap + k) * 2 + 1] = k + 1; }
            for (int k = 0; k < H.n_prior; ++k) a.prior_frames[(size_t)w * a.Ncap + k] = k;
        }
    }
}

// After a solve and its post-pass, one CTA per named slot: solved inverse depths back into the tracks, the post-pass
// flags of the landmarks into their rows (0 / 0 for the rows that did not take part -- plane tracks among them, as
// ba_solve gives them no flags -- and for every row when the solve ran no post-pass: flags == 0)
__global__ void __launch_bounds__(kBwThreads) bw_writeback_kernel(BwArgs a, const BwLayout *lay, int flags) {
    const BwLayout L = lay[blockIdx.x];
    const int w = L.slot;
    const size_t base = (size_t)w * a.Mcap;
    for (int r = threadIdx.x; r < L.T; r += kBwThreads) { a.tvalid[base + r] = 0; a.tqual[base + r] = 0.0; }
    __syncthreads();
    const int M = a.hdr[w].M;
    for (int lp = threadIdx.x; lp < M; lp += kBwThreads) {
        const int row = a.lm_row[base + lp];
        a.trho[base + row] = a.rho[base + lp];
        if (flags) { a.tvalid[base + row] = a.valid[base + lp]; a.tqual[base + row] = a.quality[base + lp]; }
    }
}

// One CTA per set_planes record (each names a different slot): the slot's plane parameters, then the roles and inverse
// depths of the named rows
__global__ void __launch_bounds__(kBwThreads) bw_planes_kernel(BwArgs a, const BwPlanes *recs, const BwRole *roles,
                                                                const double *params) {
    const BwPlanes p = recs[blockIdx.x];
    const int w = p.slot;
    const size_t base = (size_t)w * a.Mcap;
    for (int i = threadIdx.x; i < 4 * p.n_planes; i += kBwThreads) a.tplane[(size_t)w * a.Pcap * 4 + i] = params[p.param_off + i];
    for (int i = threadIdx.x; i < p.n_set; i += kBwThreads) {
        const BwRole r = roles[p.set_off + i];
        a.trole[base + r.row] = (int8_t)r.role;
        if (!isnan(r.rho)) a.trho[base + r.row] = r.rho;
    }
}

// the inverse depth of world point x in the camera at pose (qc, pc)
__device__ __forceinline__ double bw_inv_depth(const double *qc, const double *pc, const double *x) {
    const double qi[4] = {-qc[0], -qc[1], -qc[2], qc[3]};
    double d[3], y[3];
    for (int i = 0; i < 3; ++i) d[i] = x[i] - pc[i];
    bw_qrot(qi, d, y);
    return 1.0 / y[2];
}

// rows [0, n) of p down by one row over the CTA, chunk by chunk, each chunk read completely before it is written (every
// chunk reads above every address an earlier chunk wrote).  kW > 0: rows of kW doubles back to back; kW == 0: rows of w
// doubles at stride s.
template <int kW>
__device__ __forceinline__ void bw_shift_down(double *p, int n, int w = kW, int s = kW) {
    const int ne = n * w;
    for (int i0 = 0; i0 < ne; i0 += kBwThreads) {
        const int i = i0 + threadIdx.x, f = kW ? 0 : i / w, r = i - f * w;
        const double v = i < ne ? p[kW ? (size_t)(kW + i) : (size_t)(f + 1) * s + r] : 0.0;
        __syncthreads();
        if (i < ne) p[kW ? (size_t)i : (size_t)f * s + r] = v;
        __syncthreads();
    }
}

// Map::marginalize_frame(0) after the marginaliser, one CTA per slot (L.N, L.T: the window BEFORE the drop): a track
// anchored in the victim is re-anchored in its next frame from the current states (track.cpp:42-49, quirk Q5), the
// victim's observations leave their tracks, frames and IMU records shift down by one, dead tracks leave the table.
__global__ void __launch_bounds__(kBwThreads) bw_drop_kernel(BwArgs a, const BwLayout *lay) {
    __shared__ int sh[kBwWarps + 1];
    const BwLayout L = lay[blockIdx.x];
    const int w = L.slot, N = L.N, T = L.T;
    const size_t base = (size_t)w * a.Mcap;
    double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    for (int r = threadIdx.x; r < T; r += kBwThreads) {
        const uint32_t m = a.tmask[base + r];
        double2 *z = a.tz + (base + r) * a.Ncap;
        if ((m & 1u) && __popc(m) >= 2) {
            const int nx = __ffs(m & ~1u) - 1;
            double qa[4], pa[3], qn[4], pn[3];
            bw_cam_pose(fr, c, qa, pa);
            bw_cam_pose(fr + nx * kFrameStride, c, qn, pn);
            double x[3];
            bw_world_point(qa, pa, z[0].x, z[0].y, a.trho[base + r], x);
            a.trho[base + r] = bw_inv_depth(qn, pn, x);
        }
        for (int f = 0; f + 1 < N; ++f) z[f] = z[f + 1];
        a.tmask[base + r] = m >> 1;
    }
    __syncthreads();
    bw_shift_down<kFrameStride>(fr, N - 1);
    if (L.inertial && N > 2) {
        bw_shift_down<kImuStride>(a.imu_data + (size_t)w * a.Ncap * kImuStride, N - 2);
        if (L.smax > 0) {                     // the samples, t_end and noise of the factors that hold some
            bw_shift_down<kImuAux>(a.imu_aux + (size_t)w * a.Ncap * kImuAux, N - 2);
            // factor f + 1 -> f, rows [0, smax) of each
            const int fs = a.Scap * 7;
            bw_shift_down<0>(a.imu_s + (size_t)w * a.Ncap * fs, N - 2, L.smax * 7, fs);
        }
    }
    bw_compact(a, w, T, sh);
}

// One CTA per set_imu record: the factor's samples, t_end and noise from the upload into the slot
__global__ void __launch_bounds__(kBwThreads) bw_set_imu_kernel(BwArgs a, const BwImu *recs, const double *smp,
                                                                const double *aux) {
    const BwImu r = recs[blockIdx.x];
    const size_t F = (size_t)r.slot * a.Ncap + r.factor;
    double *dst = a.imu_s + F * a.Scap * 7;
    const double *src = smp + (size_t)r.off * 7;
    for (int i = threadIdx.x; i < 7 * r.n; i += kBwThreads) dst[i] = src[i];
    for (int i = threadIdx.x; i < kImuAux; i += kBwThreads) a.imu_aux[F * kImuAux + i] = aux[(size_t)blockIdx.x * kImuAux + i];
}

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

// Before a solve, one warp per factor with samples of the named slots: PreIntegrator::integrate(t, bg, ba, true, true)
// at the biases the factor's first frame holds now (frame state doubles 10 .. 15), into the slot's IMU record -- the
// arithmetic of pvio_b200_preintegrate (imu.cuh)
__global__ void __launch_bounds__(32 * kBwImuWarps) bw_reintegrate_kernel(BwArgs a, const BwImu *jobs, int n) {
    __shared__ ImuWarpSm sm[kBwImuWarps];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int j = blockIdx.x * kBwImuWarps + wv;
    if (j >= n) return;                                      // whole warps leave together
    const BwImu &J = jobs[j];
    const size_t F = (size_t)J.slot * a.Ncap + J.factor;
    const double *x = a.frames + F * kFrameStride;
    const double bg[3] = {x[10], x[11], x[12]}, ba[3] = {x[13], x[14], x[15]};
    const double *aux = a.imu_aux + F * kImuAux;
    imu_integrate_warp(sm[wv], lane, BwFactor<BwImu>{J, a.imu_s, aux + 1, aux, a.imu_data + F * kImuStride}, bg, ba);
}

// One CTA per slot: its N - 1 IMU records at dl.off (bytes)
__global__ void __launch_bounds__(kBwThreads) bw_imu_records_kernel(BwArgs a, const BwDl *dls, uint8_t *outb) {
    const BwDl d = dls[blockIdx.x];
    double *o = reinterpret_cast<double *>(outb + d.off);
    const double *rec = a.imu_data + (size_t)d.slot * a.Ncap * kImuStride;
    for (int i = threadIdx.x; i < (d.N - 1) * kImuStride; i += kBwThreads) o[i] = rec[i];
}

// one slot's record of pvio_b200_batch_window_download at byte b: its N frames, then per row of its T rows inverse depth,
// quality, id, anchor, observation count, valid; bytes: the record's size, rounded up to 16
struct BwDlRec {
    double *fo, *ro, *qo;
    int32_t *io, *ao, *no;
    uint8_t *vo;
    __host__ __device__ BwDlRec(uint8_t *b, int N, int T)
        : fo(reinterpret_cast<double *>(b)), ro(fo + (size_t)N * kFrameStride), qo(ro + T),
          io(reinterpret_cast<int32_t *>(qo + T)), ao(io + T), no(ao + T), vo(reinterpret_cast<uint8_t *>(no + T)) {}
    __host__ __device__ static int64_t bytes(int N, int T) {
        return ((int64_t)(N * kFrameStride + 2 * T) * 8 + (int64_t)T * 13 + 15) & ~(int64_t)15;
    }
};

// One CTA per slot: its download record at dl.off
__global__ void __launch_bounds__(kBwThreads) bw_download_kernel(BwArgs a, const BwDl *dls, uint8_t *outb) {
    const BwDl d = dls[blockIdx.x];
    const int w = d.slot, N = d.N, T = d.T;
    const size_t base = (size_t)w * a.Mcap;
    const BwDlRec o(outb + d.off, N, T);
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    for (int i = threadIdx.x; i < N * kFrameStride; i += kBwThreads) o.fo[i] = fr[i];
    for (int r = threadIdx.x; r < T; r += kBwThreads) {
        const uint32_t m = a.tmask[base + r];
        o.ro[r] = a.trho[base + r]; o.qo[r] = a.tqual[base + r];
        o.io[r] = a.tid[base + r]; o.ao[r] = m ? __ffs(m) - 1 : -1; o.no[r] = __popc(m); o.vo[r] = a.tvalid[base + r];
    }
}

// ------------------------------------------------------------------------ localize: PnP + triangulation of a new frame
// One record of pvio_b200_batch_window_localize as staged: the observations that take part (their rows, keypoints and
// points) at obs_off, the IMU record at imu_off (in records), the new tracks' keypoint pairs at new_off
struct BwLoc { int32_t slot, newest, inertial, n_obs, obs_off, imu_off, n_new, new_off; };
static_assert(sizeof(BwLoc) % sizeof(double) == 0, "records are staged as whole 8-byte words");

// the staged sections of one localize call (device pointers into the PnP staging)
struct LocArgs {
    const BwLoc *rec;        // [n]
    const int32_t *row;      // [n_obs] track-table row of each observation
    const double *z;         // [n_obs][2]
    const double *imu;       // [n_imu][kImuStride]
    const double *nz;        // [n_new][4] keypoint in the newest slot frame, keypoint in the new frame
    double *frames;          // [n][16] in: predicted state, out: solved
    double *pts;             // [n_obs][3] in: the given point or NaN, out: the point used
    double *out;             // [n][8] summary words of the PnP kernel
    double *rho, *rho_next;  // [n_new]
    uint8_t *valid;          // [n_new]
    PnpArgs *args;           // [n] written by the gather kernel
    int max_iter;
    double radius0;
};

constexpr int kLocGatherThreads = 128, kLocTriThreads = 64;

// One CTA per record: the world point of every observation without a given one (Track::get_landmark_point, the
// arithmetic of bw_drop_kernel's re-anchoring), and the record's PnP problem with the slot's constants and newest frame.
__global__ void __launch_bounds__(kLocGatherThreads) bw_localize_gather_kernel(BwArgs a, LocArgs L) {
    const BwLoc r = L.rec[blockIdx.x];
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    for (int i = threadIdx.x; i < r.n_obs; i += kLocGatherThreads) {
        const int k = r.obs_off + i;
        double *x = L.pts + 3 * (size_t)k;
        if (!isnan(x[0])) continue;
        bw_landmark_point(a, base + L.row[k], fr, c, x);
    }
    if (threadIdx.x == 0) {
        PnpArgs p{};                      // what batch_pnp_solve_impl stages for the same problem
        p.pts = L.pts + 3 * (size_t)r.obs_off; p.z = L.z + 2 * (size_t)r.obs_off;
        p.n = r.n_obs; p.inertial = r.inertial; p.max_iter = L.max_iter; p.radius0 = L.radius0;
        for (int j = 0; j < 4; ++j) { p.wc.cam_q[j] = c.cam_q[j]; p.wc.imu_q[j] = c.imu_q[j]; p.wc.sic[j] = c.sic[j]; }
        for (int j = 0; j < 3; ++j) { p.wc.cam_p[j] = c.cam_p[j]; p.wc.imu_p[j] = c.imu_p[j]; }
        p.wc.cauchy_a = c.cauchy_a;
        for (int j = 0; j < kFrameStride; ++j) p.last[j] = fr[r.newest * kFrameStride + j];
        p.imu_rec = r.inertial ? L.imu + (size_t)r.imu_off * kImuStride : nullptr;
        p.frame = L.frames + kFrameStride * (size_t)blockIdx.x;
        p.out = L.out + 8 * (size_t)blockIdx.x;
        L.args[blockIdx.x] = p;
    }
}

struct LocViews {                     // the two views of a new track: the newest slot frame, then the new frame
    const double *P0, *P1, *nz;
    __device__ const double *P(int o) const { return o ? P1 : P0; }
    __device__ const double *z(int o) const { return nz + 2 * o; }
};

// One CTA per record, one thread per new track: Track::triangulate over the newest slot frame and the new frame at its
// solved state, the inverse depth in the newest slot frame (set_landmark_point) and re-expressed in the new frame
// (track.cpp:42-49)
__global__ void __launch_bounds__(kLocTriThreads) bw_localize_triangulate_kernel(BwArgs a, LocArgs L) {
    const BwLoc r = L.rec[blockIdx.x];
    if (r.n_new == 0) return;
    const WinConst &c = a.cst[r.slot];
    double qa[4], pa[3], qn[4], pn[3], Pa[12], Pn[12];
    bw_cam_pose(a.frames + ((size_t)r.slot * a.Ncap + r.newest) * kFrameStride, c, qa, pa);
    bw_cam_pose(L.frames + kFrameStride * (size_t)blockIdx.x, c, qn, pn);
    loc_camera_matrix(qa, pa, Pa);
    loc_camera_matrix(qn, pn, Pn);
    for (int t = threadIdx.x; t < r.n_new; t += kLocTriThreads) {
        const int k = r.new_off + t;
        const double *nz = L.nz + 4 * (size_t)k;
        double p[3], score;
        const bool ok = tri_point_scored(LocViews{Pa, Pn, nz}, 0, 2, p, score);
        double rho = NAN, rho_next = NAN;
        if (ok) {
            rho = bw_inv_depth(qa, pa, p);
            double x[3];
            bw_world_point(qa, pa, nz[0], nz[1], rho, x);
            rho_next = bw_inv_depth(qn, pn, x);
        }
        L.valid[k] = ok ? 1 : 0;
        L.rho[k] = rho;
        L.rho_next[k] = rho_next;
    }
}

// ------------------------------------------------------------------------ track_frame: integrate, predict, keyframe check
// One record of pvio_b200_batch_window_track_frame beyond its localize half (same index): its samples' t_end and noise
// at aux_off (kImuAux doubles), frame_i of the keyframe check, the observed tracks with a keypoint in frame_i (rows and
// new-frame keypoints at kf_off), whether the new tracks count, where its parallax list starts in the scratch
struct BwTrack { int32_t merged, frame_i, n_kf, kf_off, use_new, par_off, skipped, aux_off; double cx, cy; };
// one warp job of the integrate launch: record `rec`, staged sample rows [b, e); merged: the merged list
struct BwTrackJob {
    int32_t rec, b, e, merged;
    __device__ int begin() const { return b; }
    __device__ int end() const { return e; }
};
static_assert(sizeof(BwTrack) % sizeof(double) == 0 && sizeof(BwTrackJob) % sizeof(double) == 0,
              "records are staged as whole 8-byte words");

struct TrackArgs {
    const BwTrack *tr;       // [n]
    const BwTrackJob *job;   // [n_jobs]
    const double *smp;       // [rows][7] per record merge_samples ++ samples
    const double *aux;       // [n][kImuAux] t_end, noise
    const int32_t *kf_row;   // [n_kf] track-table row of each observed pair
    const double *kf_z;      // [n_kf][2] its keypoint in the new frame
    double *rec1;            // [n][kImuStride] step-1 records (scratch; the PnP reads them through LocArgs::imu)
    double *rec_out;         // [n][kImuStride] the edit's records
    double *pred;            // [n][16]
    double *kfo;             // [n][4] keyframe, parallax, pairs, skipped
    double *par;             // parallax lists (scratch)
    int n_jobs;
};

// One warp per job: PreIntegrator::integrate(t, bg, ba, true, true) at the biases of the slot's newest frame
// (sliding_window_tracker.cpp:77, 118) -- the arithmetic of pvio_b200_preintegrate (imu.cuh); after the step-1 job,
// PreIntegrator::predict (preintegrator.cpp:102-109) into the PnP's initial state
__global__ void __launch_bounds__(32 * kBwImuWarps) bw_track_integrate_kernel(BwArgs a, LocArgs L, TrackArgs T) {
    __shared__ ImuWarpSm sm[kBwImuWarps];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int j = blockIdx.x * kBwImuWarps + wv;
    if (j >= T.n_jobs) return;                               // whole warps leave together
    const BwTrackJob &J = T.job[j];
    const BwLoc r = L.rec[J.rec];
    const double *x = a.frames + ((size_t)r.slot * a.Ncap + r.newest) * kFrameStride;
    const double bg[3] = {x[10], x[11], x[12]}, ba[3] = {x[13], x[14], x[15]};
    const double *aux = T.aux + (size_t)T.tr[J.rec].aux_off;
    double *rec = (J.merged ? T.rec_out : T.rec1) + (size_t)J.rec * kImuStride;
    imu_integrate_warp(sm[wv], lane, BwFactor<BwTrackJob>{J, T.smp, aux + 1, aux, rec}, bg, ba);
    if (J.merged) return;
    __syncwarp();
    if (!T.tr[J.rec].merged)                                 // the edit takes the step-1 record
        for (int i = lane; i < kImuStride; i += 32) T.rec_out[(size_t)J.rec * kImuStride + i] = rec[i];
    if (lane == 0) {
        double y[16];
        bw_imu_predict(x, rec[0], rec + 1, rec + 5, rec + 8, y);
        for (int k = 0; k < 16; ++k) {
            L.frames[kFrameStride * (size_t)J.rec + k] = y[k];
            T.pred[kFrameStride * (size_t)J.rec + k] = y[k];
        }
    }
}

// One CTA per record: SlidingWindowTracker::keyframe_check (sliding_window_tracker.cpp:255-296).  The parallax list goes
// to the scratch; its entry m * 4 / 5 in ascending order is found by a radix select over the fp64 bit patterns (the
// parallaxes are >= 0, so their bit patterns order as their values), eight 8-bit digits from the top, which returns
// exactly the element a sort would put there for any m.
__global__ void __launch_bounds__(kBwThreads) bw_track_keyframe_kernel(BwArgs a, LocArgs L, TrackArgs T) {
    __shared__ int sh[kBwWarps + 1];
    __shared__ unsigned int hist[256];
    __shared__ unsigned long long prefix;
    __shared__ int rank;
    const BwTrack t = T.tr[blockIdx.x];
    const BwLoc r = L.rec[blockIdx.x];
    const WinConst &c = a.cst[r.slot];
    const size_t base = (size_t)r.slot * a.Mcap;
    const double *dq = T.rec1 + (size_t)blockIdx.x * kImuStride + 1;
    double q[4], u[4], qij[4];
    const double cq[4] = {-c.cam_q[0], -c.cam_q[1], -c.cam_q[2], c.cam_q[3]};
    const double iq[4] = {-c.imu_q[0], -c.imu_q[1], -c.imu_q[2], c.imu_q[3]};
    bw_qmul(cq, c.imu_q, q);
    bw_qmul(q, dq, u);
    bw_qmul(u, iq, q);
    bw_qmul(q, c.cam_q, u);
    qij[0] = -u[0]; qij[1] = -u[1]; qij[2] = -u[2]; qij[3] = u[3];
    const int n_new = t.use_new ? r.n_new : 0, m = t.n_kf + n_new;
    double *par = T.par + t.par_off;
    for (int k = threadIdx.x; k < m; k += kBwThreads) {
        double zi[3], zj[2];
        if (k < t.n_kf) {
            const double2 z = a.tz[(base + T.kf_row[t.kf_off + k]) * a.Ncap + t.frame_i];
            zi[0] = z.x; zi[1] = z.y;
            zj[0] = T.kf_z[2 * ((size_t)t.kf_off + k)]; zj[1] = T.kf_z[2 * ((size_t)t.kf_off + k) + 1];
        } else {
            const double *nz = L.nz + 4 * ((size_t)r.new_off + k - t.n_kf);
            zi[0] = nz[0]; zi[1] = nz[1]; zj[0] = nz[2]; zj[1] = nz[3];
        }
        zi[2] = 1.0;
        double y[3];
        bw_qrot(qij, zi, y);
        const double pix = y[0] / y[2] * c.fx + t.cx, piy = y[1] / y[2] * c.fy + t.cy;
        const double pjx = zj[0] * c.fx + t.cx, pjy = zj[1] * c.fy + t.cy;
        const double dx = pix - pjx, dy = piy - pjy;
        par[k] = sqrt(dx * dx + dy * dy);
    }
    if (threadIdx.x == 0) { prefix = 0ull; rank = m * 4 / 5; }
    __syncthreads();
    if (m >= 50) {
        unsigned long long mask = 0ull;
        for (int shift = 56; shift >= 0; shift -= 8) {
            hist[threadIdx.x] = 0u;
            __syncthreads();
            const unsigned long long pre = prefix;
            for (int k = threadIdx.x; k < m; k += kBwThreads) {
                const unsigned long long v = (unsigned long long)__double_as_longlong(par[k]);
                if ((v & mask) == pre) atomicAdd(&hist[(v >> shift) & 255u], 1u);
            }
            __syncthreads();
            const int cnt = (int)hist[threadIdx.x], want = rank;
            int tot;
            const int below = bw_block_scan(cnt, sh, tot);   // ends with a barrier: every thread has read rank / prefix
            if (want >= below && want < below + cnt) {           // exactly one digit holds the wanted rank
                prefix = pre | ((unsigned long long)threadIdx.x << shift);
                rank = want - below;
            }
            mask |= 255ull << shift;
            __syncthreads();
        }
    }
    if (threadIdx.x == 0) {
        int skipped = t.skipped;
        bool kf;
        double p = NAN;
        if (m < 50) {
            kf = true;
        } else {
            p = __longlong_as_double((long long)prefix);
            kf = p > 50.0;
            if (!kf) ++skipped;
        }
        if (skipped > 10) kf = true;
        if (kf) skipped = 0;
        double *o = T.kfo + 4 * (size_t)blockIdx.x;
        o[0] = kf ? 1.0 : 0.0; o[1] = p; o[2] = m; o[3] = skipped;
    }
}

// ------------------------------------------------------------------------ set_keypoints / mirror_frame: the tracker link
// one set_keypoints record: the slot's T rows, its n (row, keypoint) pairs at off
struct BwKeys { int32_t slot, T, n, off; };

// One CTA per set_keypoints record: every row without a keypoint in the newest frame, then the named ones
__global__ void __launch_bounds__(kBwThreads) bw_set_keypoints_kernel(BwArgs a, const BwKeys *recs, const int2 *pairs) {
    const BwKeys k = recs[blockIdx.x];
    const size_t base = (size_t)k.slot * a.Mcap;
    for (int r = threadIdx.x; r < k.T; r += kBwThreads) a.tkp[base + r] = -1;
    __syncthreads();
    for (int i = threadIdx.x; i < k.n; i += kBwThreads) { const int2 p = pairs[k.off + i]; a.tkp[base + p.x] = p.y; }
}

// One record of pvio_b200_batch_window_mirror_frame as staged.  Its lists start at kp_off, the earlier records' new-frame
// keypoint counts summed (each list holds at most one entry per new-frame keypoint): PnP observations, new-track
// candidates, parallax pairs, continued rows, kp_track, the edit's new tracks and observations.
struct BwMirror {
    const double2 *zi, *zj;           // the tracker slot's previous frame (the slot's newest) and new frame
    const int32_t *prev;              // the new frame's prev_index
    int32_t slot, T, n_i, n_j;        // live rows; keypoints of the two frames
    int32_t tab_off, kp_off, g_off, n_g;          // keypoint tables (2 n_i ints); given points (rows ascending)
    int32_t rm_off, merge_row, n_merge, replace;  // row map (T ints); the merge list's staged rows
    int32_t N_old, next_id, pad0, pad1;
};
static_assert(sizeof(BwMirror) % sizeof(double) == 0, "records are staged as whole 8-byte words");

// the device view of a mirror_frame call: the mirror's records and lists, and the sections of track_frame's kernels
// (LocArgs, TrackArgs) and bw_edit_kernel it writes
struct MirArgs {
    const BwMirror *rec;
    BwLoc *loc;              // [n] n_obs, n_new written by the mirror
    BwTrack *tr;             // [n] n_kf written by the mirror
    int32_t *tab;            // row of each keypoint of frame i (-1: none), then the new-frame keypoint continuing it
    const int32_t *grow;     // given points: rows, ascending per record
    const double *gpt;       //   [3] each
    int32_t *row;            // LocArgs::row
    double *z, *pts, *nz;    // LocArgs::z, pts, nz
    int32_t *kf_row;         // TrackArgs::kf_row
    double *kf_z, *smp;      // TrackArgs::kf_z, smp (the merge rows are copied from the slot)
    int2 *cont;              // continued tracks in new-frame order: (row, kj)
    int32_t *cand;           // the new-frame keypoint of each candidate
    int32_t *rmap;           // row after the edit's compaction, -1: the track ends with the replaced frame
    int32_t *lrow;           // row after the edit of each new-frame keypoint, -1: none
    int32_t *kp;             // kp_track
    int32_t *cnt;            // [n][4] continued, PnP observations, candidates, new tracks
    const int32_t *eout;     // bw_edit_kernel's results (live rows at each edit's out_off)
    int32_t *live;           // [n] live rows after the edit (downloaded)
    BwEdit *ed;              // [n] host-filled but for n_new, n_obs
    BwNew *nw;
    BwObs *ob;
    double *x;               // [n][16 + kImuStride] the edit's state and IMU record
    BwLayout *lay;           // [n] the re-layout's records, T written by the append
};
constexpr int kMirX = kFrameStride + kImuStride;

// One CTA per record: SlidingWindowTracker::mirror_frame (sliding_window_tracker.cpp:52-73) into the lists track_frame's
// kernels read.  The slot's keypoint -> row table of the newest frame (frame i) and, for each keypoint of frame i, the
// new-frame keypoint kj continuing it; then the continued tracks in kj order (the PnP observations, the parallax pairs
// with a keypoint in frame_i) and the candidates in ki order; the merge list from the slot's newest factor.
__global__ void __launch_bounds__(kBwThreads) bw_mirror_kernel(BwArgs a, MirArgs M) {
    __shared__ int sh[kBwWarps + 1];
    const BwMirror r = M.rec[blockIdx.x];
    const BwLoc lc = M.loc[blockIdx.x];
    const BwTrack tk = M.tr[blockIdx.x];
    const size_t base = (size_t)r.slot * a.Mcap;
    int *row_of = M.tab + r.tab_off, *kj_of = row_of + r.n_i;
    for (int k = threadIdx.x; k < r.n_i; k += kBwThreads) { row_of[k] = -1; kj_of[k] = -1; }
    __syncthreads();
    for (int q = threadIdx.x; q < r.T; q += kBwThreads) {
        const int k = a.tkp[base + q];
        if (k >= 0) row_of[k] = q;
    }
    for (int kj = threadIdx.x; kj < r.n_j; kj += kBwThreads) {
        const int ki = r.prev[kj];
        if (ki >= 0) kj_of[ki] = kj;
    }
    __syncthreads();
    const uint32_t fi = 1u << tk.frame_i;
    int nc = 0, np = 0, nk = 0;
    for (int c0 = 0; c0 < r.n_j; c0 += kBwThreads) {
        const int kj = c0 + threadIdx.x;
        const int ki = kj < r.n_j ? r.prev[kj] : -1;
        const int row = ki >= 0 ? row_of[ki] : -1;
        int g = -1;
        bool pnp = false, kf = false;
        if (row >= 0) {
            int lo = 0, hi = r.n_g;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (M.grow[r.g_off + mid] < row) lo = mid + 1; else hi = mid;
            }
            if (lo < r.n_g && M.grow[r.g_off + lo] == row) g = r.g_off + lo;
            pnp = a.trole[base + row] == -1 || g >= 0;
            kf = (a.tmask[base + row] & fi) != 0u;
        }
        int tc, tp, tq;
        const int ic = nc + bw_block_scan(row >= 0 ? 1 : 0, sh, tc);
        const int ip = np + bw_block_scan(pnp ? 1 : 0, sh, tp);
        const int iq = nk + bw_block_scan(kf ? 1 : 0, sh, tq);
        if (row >= 0) {
            const double2 z = r.zj[kj];
            M.cont[r.kp_off + ic] = make_int2(row, kj);
            if (pnp) {
                const size_t k = (size_t)lc.obs_off + ip;
                M.row[k] = row;
                M.z[2 * k] = z.x; M.z[2 * k + 1] = z.y;
                for (int j = 0; j < 3; ++j) M.pts[3 * k + j] = g >= 0 ? M.gpt[3 * (size_t)g + j] : NAN;
            }
            if (kf) {
                const size_t k = (size_t)tk.kf_off + iq;
                M.kf_row[k] = row;
                M.kf_z[2 * k] = z.x; M.kf_z[2 * k + 1] = z.y;
            }
        }
        nc += tc; np += tp; nk += tq;
    }
    int nn = 0;
    for (int c0 = 0; c0 < r.n_i; c0 += kBwThreads) {
        const int ki = c0 + threadIdx.x;
        const int kj = ki < r.n_i ? kj_of[ki] : -1;
        const bool cand = kj >= 0 && row_of[ki] < 0;
        int tn;
        const int in = nn + bw_block_scan(cand ? 1 : 0, sh, tn);
        if (cand) {
            const size_t k = (size_t)lc.new_off + in;
            const double2 zi = r.zi[ki], zj = r.zj[kj];
            M.nz[4 * k] = zi.x; M.nz[4 * k + 1] = zi.y; M.nz[4 * k + 2] = zj.x; M.nz[4 * k + 3] = zj.y;
            M.cand[k] = kj;
        }
        nn += tn;
    }
    if (r.n_merge > 0) {                      // the newest factor's samples: factor N - 2 of the slot
        const double *src = a.imu_s + ((size_t)r.slot * a.Ncap + r.N_old - 2) * a.Scap * 7;
        for (int i = threadIdx.x; i < 7 * r.n_merge; i += kBwThreads) M.smp[7 * (size_t)r.merge_row + i] = src[i];
    }
    if (threadIdx.x == 0) {
        M.loc[blockIdx.x].n_obs = np; M.loc[blockIdx.x].n_new = nn; M.tr[blockIdx.x].n_kf = nk;
        int *c = M.cnt + 4 * (size_t)blockIdx.x;
        c[0] = nc; c[1] = np; c[2] = nn; c[3] = 0;
    }
}

// One CTA per record, after track_frame's kernels: the frame edit in bw_edit_kernel's layout.  replace_last follows the
// slot's newest frame; the continued tracks that outlive it observe the new frame (kj order); the valid candidates (ki
// order) become the slot's next ids, anchored in the newest frame with their observation in the new one, or anchored in
// the new frame after replace_last.  kp_track, the rows of the new frame's keypoints after the edit, the edit's state
// and IMU record, the re-layout's row count.
__global__ void __launch_bounds__(kBwThreads) bw_mirror_append_kernel(BwArgs a, LocArgs L, TrackArgs T, MirArgs M) {
    __shared__ int sh[kBwWarps + 1];
    const int b = blockIdx.x;
    const BwMirror r = M.rec[b];
    const BwLoc lc = M.loc[b];
    const BwEdit e = M.ed[b];
    const int nc = M.cnt[4 * b];
    const size_t base = (size_t)r.slot * a.Mcap;
    const int fnew = e.frame;
    int32_t *rmap = M.rmap + r.rm_off, *lrow = M.lrow + r.kp_off, *kp = M.kp + r.kp_off;
    const uint32_t keep = r.replace ? ~(1u << (r.N_old - 1)) : ~0u;
    int kept = 0;
    for (int c0 = 0; c0 < r.T; c0 += kBwThreads) {
        const int q = c0 + threadIdx.x;
        const bool live = q < r.T && (a.tmask[base + q] & keep) != 0u;
        int tot;
        const int d = kept + bw_block_scan(live ? 1 : 0, sh, tot);
        if (q < r.T) rmap[q] = live ? d : -1;
        kept += tot;
    }
    for (int kj = threadIdx.x; kj < r.n_j; kj += kBwThreads) { lrow[kj] = -1; kp[kj] = -1; }
    __syncthreads();
    int no = 0;
    for (int c0 = 0; c0 < nc; c0 += kBwThreads) {
        const int i = c0 + threadIdx.x;
        int row = -1, kj = 0, id = -1;
        if (i < nc) {
            const int2 c = M.cont[r.kp_off + i];
            row = rmap[c.x]; kj = c.y; id = a.tid[base + c.x];
        }
        int tot;
        const int o = no + bw_block_scan(row >= 0 ? 1 : 0, sh, tot);
        if (row >= 0) {
            const double2 z = r.zj[kj];
            M.ob[e.obs_off + o] = BwObs{row, fnew, z.x, z.y};
            lrow[kj] = row; kp[kj] = id;
        }
        no += tot;
    }
    int nv = 0;
    for (int c0 = 0; c0 < lc.n_new; c0 += kBwThreads) {
        const int t = c0 + threadIdx.x;
        const bool v = t < lc.n_new && L.valid[lc.new_off + t] != 0;
        int tot;
        const int k = nv + bw_block_scan(v ? 1 : 0, sh, tot);
        if (v) {
            const size_t q = (size_t)lc.new_off + t;
            const double *nz = M.nz + 4 * q;
            const int row = kept + k, kj = M.cand[q];
            if (r.replace) {
                M.nw[e.new_off + k] = BwNew{row, r.next_id + k, fnew, 0, nz[2], nz[3], L.rho_next[q]};
            } else {
                M.nw[e.new_off + k] = BwNew{row, r.next_id + k, fnew - 1, 0, nz[0], nz[1], L.rho[q]};
                M.ob[e.obs_off + no + k] = BwObs{row, fnew, nz[2], nz[3]};
            }
            lrow[kj] = row; kp[kj] = r.next_id + k;
        }
        nv += tot;
    }
    double *x = M.x + (size_t)b * kMirX;
    for (int i = threadIdx.x; i < kFrameStride; i += kBwThreads) x[i] = L.frames[(size_t)b * kFrameStride + i];
    for (int i = threadIdx.x; i < kImuStride; i += kBwThreads) x[kFrameStride + i] = T.rec_out[(size_t)b * kImuStride + i];
    if (threadIdx.x == 0) {
        M.ed[b].n_new = nv;
        M.ed[b].n_obs = no + (r.replace ? 0 : nv);
        M.cnt[4 * b + 3] = nv;
        M.lay[b].T = kept + nv;
    }
}

// One CTA per record, after the edit's compaction: the slot's keypoint index of every row in the new frame
__global__ void __launch_bounds__(kBwThreads) bw_mirror_link_kernel(BwArgs a, MirArgs M) {
    const BwMirror r = M.rec[blockIdx.x];
    const size_t base = (size_t)r.slot * a.Mcap;
    const int T = M.lay[blockIdx.x].T;
    if (threadIdx.x == 0) M.live[blockIdx.x] = M.eout[M.ed[blockIdx.x].out_off];
    for (int q = threadIdx.x; q < T; q += kBwThreads) a.tkp[base + q] = -1;
    __syncthreads();
    for (int kj = threadIdx.x; kj < r.n_j; kj += kBwThreads) {
        const int row = M.lrow[r.kp_off + kj];
        if (row >= 0) a.tkp[base + row] = kj;
    }
}

// ------------------------------------------------------------------------ host side
template <>
BwArgs launch_args<BwArgs>(const Handle *h) {
    const BatchWindows &b = h->bw;
    BwArgs a{};
    static_cast<BatchArrays &>(a) = h->arrays;
    a.tid = b.tid.d; a.tmask = b.tmask.d; a.trho = b.trho.d; a.tz = b.tz.d; a.tvalid = b.tvalid.d; a.tqual = b.tqual.d;
    a.trole = b.trole.d; a.tplane = b.tplane.d; a.lm_row = b.lm_row.d; a.valid = h->valid.d; a.quality = h->quality.d;
    a.imu_s = b.imu_s.d; a.imu_aux = b.imu_aux.d; a.Scap = b.Scap; a.tkp = b.tkp.d;
    return a;
}

static int ensure_bw(Handle *h) {
    BatchWindows &b = h->bw;
    if (b.lm_row.n) return 0;                 // allocated last: every table is there
    const size_t W = h->W, M = h->Mcap;
    TRY(alloc(h, b.tid, W * M, kDevice)); TRY(alloc(h, b.tmask, W * M, kDevice)); TRY(alloc(h, b.trho, W * M, kDevice));
    TRY(alloc(h, b.tz, W * M * h->Ncap, kDevice)); TRY(alloc(h, b.tvalid, W * M, kDevice)); TRY(alloc(h, b.tqual, W * M, kDevice));
    TRY(alloc(h, b.trole, W * M, kDevice)); TRY(alloc(h, b.tplane, W * h->Pcap * 4, kDevice));
    TRY(alloc(h, b.tkp, W * M, kDevice));
    TRY(alloc(h, b.lm_row, W * M, kDevice));
    return 0;
}

// the sample store for factors of up to S samples: t_end / noise allocated with the first set_imu, the samples grown to
// the longest list seen, every slot's samples copied across to the new stride on the device
static int ensure_imu_store(Handle *h, int S) {
    BatchWindows &b = h->bw;
    const size_t F = (size_t)h->W * h->Ncap;
    if (!b.imu_aux.n) TRY(alloc(h, b.imu_aux, F * kImuAux, kDevice));
    if (S <= b.Scap) return 0;
    DevBuf<double> next;
    TRY(alloc(h, next, F * S * 7, kDevice));
    if (b.Scap > 0) {
        CK(h, cudaMemcpy2DAsync(next.d, sizeof(double) * 7 * S, b.imu_s.d, sizeof(double) * 7 * b.Scap,
                                sizeof(double) * 7 * b.Scap, F, cudaMemcpyDeviceToDevice, h->stream));
        CK(h, cudaStreamSynchronize(h->stream));       // the old store is freed below
    }
    b.imu_s = std::move(next);
    b.Scap = S;
    return 0;
}

// the window of a slot as the checks and the launch shapes see it; T / O: plane tracks and their observations
struct BwShape { int M = 0, K = 0, chunks = 0, max_obs = 0, T = 0, O = 0; };
static BwShape shape_of(const WinSlot &s) {
    BwShape r;
    int cnt[kMaxFrames] = {};
    for (size_t i = 0; i < s.mask.size(); ++i) {
        const uint32_t m = s.mask[i];
        const int p = __builtin_popcount(m);
        if (s.role[i] >= 0) { ++r.T; r.O += p; continue; }
        if (p < 2) continue;
        ++cnt[__builtin_ctz(m)]; ++r.M; r.K += p - 1; r.max_obs = std::max(r.max_obs, p - 1);
    }
    for (int a = 0; a < kMaxFrames; ++a) r.chunks += (cnt[a] + 31) / 32;
    return r;
}

static int check_window(Handle *h, const WinSlot &s) {
    const BwShape sh = shape_of(s);
    if (s.N > h->Ncap) return fail(h, PVIO_B200_EINVAL, "batch_window: more frames than max_frames");
    if ((int)s.ids.size() > h->Mcap) return fail(h, PVIO_B200_EINVAL, "batch_window: more live tracks than max_landmarks");
    if (sh.K > h->Kcap) return fail(h, PVIO_B200_EINVAL, "batch_window: more observations than max_obs");
    if (sh.max_obs >= 16) return fail(h, PVIO_B200_EINVAL, "batch_window: a landmark with 16 or more observations");
    if (sh.chunks > kMaxChunks) return fail(h, PVIO_B200_EINVAL, "batch_window: too many landmark chunks");
    return 0;
}

// the shape fields of the slot's host header (batch_shape and the marginaliser read them); the device header is the
// re-layout kernel's
static void host_header(Handle *h, int slot) {
    const WinSlot &s = h->slots[slot];
    const BwShape sh = shape_of(s);
    WinHdr &H = h->hdr.h[slot];
    memset(&H, 0, sizeof(H));
    H.N = s.N; H.M = sh.M; H.K = sh.K; H.use_inertial = s.inertial; H.n_imu = s.inertial ? std::max(s.N - 1, 0) : 0;
    H.n_prior = s.inertial ? s.n_prior : 0; H.fixed_mask = s.fixed; H.n_chunks = sh.chunks;
    H.n_planes = s.n_planes; H.n_ptracks = sh.T;            // batch_shape: plane tracks take the full solve kernel
}

static BwLayout layout_of(int slot, const WinSlot &s) {
    int smax = 0;
    for (int32_t c : s.n_samples) smax = std::max(smax, (int)c);
    return BwLayout{slot, s.N, (int)s.ids.size(), s.fixed, s.n_prior, s.inertial, s.n_planes, smax};
}

// the rows of a mirror whose frame mask, shifted down by `shift` frames, is not 0, in order, with their shifted masks
static void compact_rows(WinSlot &s, int shift) {
    size_t o = 0;
    for (size_t r = 0; r < s.ids.size(); ++r) {
        const uint32_t m = s.mask[r] >> shift;
        if (m) { s.ids[o] = s.ids[r]; s.mask[o] = m; s.role[o] = s.role[r]; ++o; }
    }
    s.ids.resize(o); s.mask.resize(o); s.role.resize(o);
}

// the re-layout of a call's slots to their new mirrors next[]: their BwLayouts and the slot list go with the call's
// upload; launch rebuilds the packed windows once the call's own kernels are queued
struct Relayout {
    std::vector<BwLayout> lays;
    Stage::Sec<BwLayout> lay;
    Stage::Sec<int32_t> slots;
    Relayout(Stage &S, const int32_t *sl, const std::vector<WinSlot> &next) : lays(next.size()) {
        for (size_t i = 0; i < next.size(); ++i) lays[i] = layout_of(sl[i], next[i]);
        lay = S.up(lays);
        slots = S.add(Stage::kUp, next.size(), sl);
    }
    int launch(Handle *h, const Stage &S, bool prior) const {
        const int n = (int)lays.size();
        bw_layout_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(lay));
        ++h->launches;
        CK(h, cudaGetLastError());
        return launch_layout_tail(h, S.dev(slots), n, prior);
    }
};

// the mirrors of a call that has run into their slots, with their host headers
static void commit(Handle *h, const int32_t *slots, std::vector<WinSlot> &next) {
    for (size_t i = 0; i < next.size(); ++i) {
        h->slots[slots[i]] = std::move(next[i]);
        host_header(h, slots[i]);
    }
}

// plane-table capacity for the windows the n slots of a call will hold, before anything of the call is staged
static int ensure_plane_tables(Handle *h, const std::vector<WinSlot> &next) {
    int T = 0, O = 0;
    for (const WinSlot &s : next) { const BwShape sh = shape_of(s); T = std::max(T, sh.T); O = std::max(O, sh.O); }
    return T > 0 ? ensure_planes(h, T, O) : 0;
}

static int check_slots(Handle *h, int n, const int32_t *slots, const char *what) {
    if (n < 0 || (n > 0 && !slots)) return fail(h, PVIO_B200_EINVAL, what);
    std::vector<uint8_t> seen(h->W, 0);
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        if (s < 0 || s >= h->W || !h->slots[s].resident)
            return fail(h, PVIO_B200_EINVAL, "batch_window: slot out of range or not resident");
        if (seen[s]) return fail(h, PVIO_B200_EINVAL, "batch_window: a slot named twice");
        seen[s] = 1;
    }
    return 0;
}

// BundleAdjustor::solve on the n slots of a list; post: then the landmark post-pass
static int solve_slots(Handle *h, int n, const int32_t *slots, const pvio_b200_options *opt, bool post,
                       pvio_b200_summary *summaries) {
    TRY(check_slots(h, n, slots, "batch_window_solve: bad slot list"));
    if (n == 0) return 0;
    // the trust-region chain runs over windows [0, range) and skips the unnamed ones (init_ctrl_kernel marks them
    // finished before the first body; every kernel of the chain returns for a finished window before it reads anything
    // else of it); the post-pass and the write-back run over the named list only
    int range = 0;
    for (int i = 0; i < n; ++i) {
        if (h->slots[slots[i]].N < 1) return fail(h, PVIO_B200_EINVAL, "batch_window_solve: a window without frames");
        range = std::max(range, slots[i] + 1);
    }
    std::vector<uint8_t> named(range, 0);
    std::vector<BwLayout> lays(n);
    std::vector<BwImu> jobs;                  // the factors with samples: re-integrated before the chain
    for (int i = 0; i < n; ++i) {
        const WinSlot &s = h->slots[slots[i]];
        named[slots[i]] = 1; lays[i] = layout_of(slots[i], s);
        if (s.inertial)
            for (int k = 0; k + 1 < s.N; ++k)
                if (s.n_samples[k] > 0)
                    jobs.push_back(BwImu{slots[i], k, s.n_samples[k], (int32_t)(((size_t)slots[i] * h->Ncap + k) * h->bw.Scap)});
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto nm = S.up(named);
    const auto lay = S.up(lays);
    const auto sl = S.add(Stage::kUp, n, slots);
    const auto job = S.up(jobs);
    TRY(S.place(h, true));
    if (!jobs.empty()) {
        const int J = (int)jobs.size();
        bw_reintegrate_kernel<<<(J + kBwImuWarps - 1) / kBwImuWarps, 32 * kBwImuWarps, 0, h->stream>>>(
            launch_args<BwArgs>(h), S.dev(job), J);
        ++h->launches;
        CK(h, cudaGetLastError());
    }
    CK(h, cudaEventRecord(h->ev0, h->stream));
    TRY(run_named_solve(h, opt, range, S.dev(nm), named.data()));
    CK(h, cudaEventRecord(h->ev1, h->stream));
    if (post) TRY(run_postpass_slots(h, n, S.dev(sl)));
    bw_writeback_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(lay), post ? 1 : 0);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(h->ctrl.h, h->ctrl.d, sizeof(WinCtrl) * range, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev0, h->ev1);
    if (summaries)
        for (int i = 0; i < n; ++i) {
            fill_summary(h->ctrl.h[slots[i]], &summaries[i]);
            summaries[i].solve_seconds = ms * 1e-3;
        }
    return 0;
}

// The localize half of a batch of records (pvio_b200_batch_window_localize, pvio_b200_batch_window_track_frame): every
// record checked against its slot's host mirror, the observations that take part kept with the index they came from,
// the new tracks' keypoint pairs
struct LocPlan {
    const char *what;
    std::vector<BwLoc> recs;
    std::vector<int32_t> rows, from;
    std::vector<double> zs, pts, nzs;
    int n_imu = 0;
};

static int loc_fail(Handle *h, const LocPlan &P, const char *why) {
    return fail(h, PVIO_B200_EINVAL, (std::string(P.what) + ": " + why).c_str());
}

// checks record R (imu_given: it must carry its IMU record when inertial) and appends it to the plan
static int loc_add(Handle *h, LocPlan &P, const pvio_b200_window_localize &R, bool imu_given) {
    const WinSlot &s = h->slots[R.slot];
    if (s.N < 1) return loc_fail(h, P, "a window without frames");
    if (!R.state || R.n_obs < 0 || R.n_new < 0 || (R.n_obs > 0 && (!R.obs_track || !R.obs_z)) ||
        (R.n_new > 0 && (!R.new_z_last || !R.new_z || !R.new_valid || !R.new_inv_depth)))
        return loc_fail(h, P, "null array");
    if (imu_given && R.use_inertial && !R.imu_record)
        return loc_fail(h, P, "an inertial record needs the IMU record from the newest frame");
    P.recs.push_back(BwLoc{R.slot, s.N - 1, R.use_inertial ? 1 : 0, 0, (int32_t)P.rows.size(), R.use_inertial ? P.n_imu++ : -1,
                           R.n_new, (int32_t)(P.nzs.size() / 4)});
    BwLoc &L = P.recs.back();
    const uint32_t newest = 1u << (s.N - 1);
    std::vector<uint8_t> named(s.ids.size(), 0);
    for (int k = 0; k < R.n_obs; ++k) {
        const int r = find_row(s, R.obs_track[k]);
        if (r < 0) return loc_fail(h, P, "unknown or dead track");
        if (named[r]) return loc_fail(h, P, "a track named twice");
        named[r] = 1;
        const double *z = R.obs_z + 2 * k;
        if (!std::isfinite(z[0]) || !std::isfinite(z[1])) return loc_fail(h, P, "non-finite keypoint");
        const double *x = R.obs_point ? R.obs_point + 3 * k : nullptr;
        const bool given = x && std::isfinite(x[0]) && std::isfinite(x[1]) && std::isfinite(x[2]);
        if (x && !given && !(std::isnan(x[0]) && std::isnan(x[1]) && std::isnan(x[2])))
            return loc_fail(h, P, "a point row neither finite nor NaN");
        if (!(s.mask[r] & newest)) continue;                              // pnp.cpp:58
        if (!given && s.role[r] != -1) return loc_fail(h, P, "a plane track without its plane-cast point");
        P.rows.push_back(r);
        P.from.push_back(k);
        P.zs.insert(P.zs.end(), z, z + 2);
        for (int j = 0; j < 3; ++j) P.pts.push_back(given ? x[j] : NAN);
    }
    L.n_obs = (int32_t)P.rows.size() - L.obs_off;
    for (int k = 0; k < R.n_new; ++k) {
        const double *a = R.new_z_last + 2 * k, *b = R.new_z + 2 * k;
        if (!std::isfinite(a[0]) || !std::isfinite(a[1]) || !std::isfinite(b[0]) || !std::isfinite(b[1]))
            return loc_fail(h, P, "non-finite keypoint");
        P.nzs.insert(P.nzs.end(), {a[0], a[1], b[0], b[1]});
    }
    return 0;
}

// the staged sections of a plan: upload records | rows | keypoints | IMU records | new pairs; in/out states (in: the
// prediction, out: solved) | points (in: the given point or NaN, out: the point used); download summary words |
// inverse depths | re-anchored inverse depths | valid bytes; device only the PnP records
struct LocSecs {
    Stage::Sec<BwLoc> rec;
    Stage::Sec<int32_t> row;
    Stage::Sec<double> z, imu, nz, frames, pts, out, rho, next;
    Stage::Sec<uint8_t> valid;
    Stage::Sec<PnpArgs> args;
};

// imu: the IMU records of the inertial records are staged (the caller fills them)
static LocSecs loc_stage(Stage &S, const LocPlan &P, bool imu) {
    const size_t n = P.recs.size(), T = P.nzs.size() / 4;
    LocSecs s;
    s.rec = S.up(P.recs); s.row = S.up(P.rows); s.z = S.up(P.zs);
    s.imu = S.add<double>(Stage::kUp, imu ? (size_t)P.n_imu * kImuStride : 0); s.nz = S.up(P.nzs);
    s.frames = S.add<double>(Stage::kInOut, 16 * n); s.pts = S.add(Stage::kInOut, P.pts.size(), P.pts.data());
    s.out = S.add<double>(Stage::kDown, 8 * n); s.rho = S.add<double>(Stage::kDown, T);
    s.next = S.add<double>(Stage::kDown, T); s.valid = S.add<uint8_t>(Stage::kDown, T);
    s.args = S.add<PnpArgs>(Stage::kScratch, n);
    return s;
}

// the device view of the placed plan
static LocArgs loc_args(const Stage &S, const LocSecs &s, const pvio_b200_options *opt) {
    const SolveOptions so = solve_options(opt);
    LocArgs L;
    L.rec = S.dev(s.rec); L.row = S.dev(s.row); L.z = S.dev(s.z); L.imu = S.dev(s.imu); L.nz = S.dev(s.nz);
    L.frames = S.dev(s.frames); L.pts = S.dev(s.pts); L.out = S.dev(s.out); L.rho = S.dev(s.rho);
    L.rho_next = S.dev(s.next); L.valid = S.dev(s.valid); L.args = S.dev(s.args);
    L.max_iter = so.max_iter; L.radius0 = so.radius0;
    return L;
}

// gather, PnP, triangulation: three launches whatever n is
static int loc_launch(Handle *h, const LocArgs &L, int n) {
    const BwArgs a = launch_args<BwArgs>(h);
    bw_localize_gather_kernel<<<n, kLocGatherThreads, 0, h->stream>>>(a, L);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(launch_pnp(h, n, L.args));
    CK(h, cudaGetLastError());
    bw_localize_triangulate_kernel<<<n, kLocTriThreads, 0, h->stream>>>(a, L);
    ++h->launches;
    CK(h, cudaGetLastError());
    return 0;
}

// after the download: record i's localize outputs into R
static void loc_results(const Stage &S, const LocSecs &s, const LocPlan &P, int i, size_t &k,
                        const pvio_b200_window_localize &R, float ms) {
    const size_t w8 = sizeof(double);
    const BwLoc &L = P.recs[i];
    memcpy(R.state, S.host(s.frames) + 16 * (size_t)i, w8 * 16);
    if (R.points_out) {
        for (int j = 0; j < 3 * R.n_obs; ++j) R.points_out[j] = NAN;
        for (int j = 0; j < L.n_obs; ++j, ++k) memcpy(R.points_out + 3 * P.from[k], S.host(s.pts) + 3 * k, w8 * 3);
    } else {
        k += L.n_obs;
    }
    for (int t = 0; t < L.n_new; ++t) {
        const size_t q = (size_t)L.new_off + t;
        R.new_valid[t] = S.host(s.valid)[q];
        R.new_inv_depth[t] = S.host(s.rho)[q];
        if (R.new_inv_depth_next) R.new_inv_depth_next[t] = S.host(s.next)[q];
    }
    if (R.summary) pnp_summary(S.host(s.out) + 8 * (size_t)i, ms, R.summary);
}

// the localize half of a track_frame record
static pvio_b200_window_localize localize_view(const pvio_b200_window_track_frame &R) {
    pvio_b200_window_localize L{};
    L.slot = R.slot; L.use_inertial = 1; L.state = R.state;
    L.n_obs = R.n_obs; L.obs_track = R.obs_track; L.obs_z = R.obs_z; L.obs_point = R.obs_point; L.points_out = R.points_out;
    L.n_new = R.n_new; L.new_z_last = R.new_z_last; L.new_z = R.new_z; L.new_valid = R.new_valid;
    L.new_inv_depth = R.new_inv_depth; L.new_inv_depth_next = R.new_inv_depth_next; L.summary = R.summary;
    return L;
}

static bool all_finite(const double *x, int64_t n) {
    for (int64_t k = 0; k < n; ++k)
        if (!std::isfinite(x[k])) return false;
    return true;
}

// slot 0 as the single resident window (pvio_b200_window_*); null, with the error set, before pvio_b200_window_reset
static const WinSlot *window0(Handle *h) {
    if (!h->slots[0].resident) {
        fail(h, PVIO_B200_EINVAL, "window: no resident window: call pvio_b200_window_reset first");
        return nullptr;
    }
    return &h->slots[0];
}

// the host mirror of a slot after its mirror_frame record: replace_last when the newest frame is not a keyframe, the new
// frame (its factor holding n_kept samples), an observation there for each continued row (rows of s) that outlives the
// replaced frame, n_new new tracks with the slot's next ids
static WinSlot mirror_next(const WinSlot &s0, const std::vector<int> &rows, int n_new, int n_kept) {
    WinSlot s = s0;
    const bool replace = !s.newest_kf;
    if (replace) {
        for (uint32_t &m : s.mask) m &= ~(1u << (s.N - 1));
        s.fixed &= ~(1 << (s.N - 1));
        s.n_samples[s.N - 2] = 0;
        --s.N;
    }
    const int f = s.N;
    for (int r : rows)
        if (s.mask[r]) s.mask[r] |= 1u << f;
    compact_rows(s, 0);
    s.n_samples[f - 1] = n_kept;
    ++s.N;
    for (int k = 0; k < n_new; ++k) {
        s.ids.push_back(s.next_id++);
        s.mask.push_back(replace ? 1u << f : (1u << (f - 1)) | (1u << f));
        s.role.push_back(-1);
    }
    return s;
}

// ------------------------------------------------------------------------ snapshots (pvio_b200_batch_window_save / restore)
// A blob: SnapHead, then sections that each start at a multiple of 16 bytes, zero between them.  The host region (ids,
// frame masks, roles, per-factor sample counts: what the host mirror holds) follows the head; the device region, from
// dev0, holds what only the device keeps.  Sections of a part the blob lacks are empty.
constexpr int32_t kSnapWindow = 1, kSnapTracker = 2;
struct SnapHead {
    uint32_t magic, version;
    int64_t size;                                 // bytes of the blob
    int32_t parts;                                // kSnapWindow | kSnapTracker
    int32_t N, T, fixed, next_id, n_prior, inertial, n_planes, newest_kf, skipped;     // the window
    int32_t linked;                               // the window's link to the blob's tracker part (both parts held)
    int32_t n[2];                                 // the tracker: keypoints of its newest and its previous frame
    int32_t frame_no, w, h, levels;               //   the newest frame's number and pyramid shape (levels 0: none)
    int32_t pad[3];
    uint64_t frame_id, prev_frame_id;             //   its frame ids
    uint64_t link_frame;                          // the tracker frame id of the window's newest frame (linked)
    double K[4];                                  // fx, fy, cx, cy of the newest frame
    double clahe;                                 // the CLAHE clip its pyramid was built with
};
static_assert(sizeof(SnapHead) == 160 && offsetof(SnapHead, frame_id) == 96, "the head has no implicit padding");

// byte offsets of a blob's sections
struct SnapOff {
    int64_t ids, mask, role, nsmp, dev0;          // host region, then the start of the device region
    int64_t cst, tkp, valid, rho, qual, tz, frames, imu, pS, pe, px0, aux, smp, planes;   // window, device region
    int64_t kz, kb, kp, lvl[kMaxLevels];          // tracker: keypoints, births, prev_index (newest frame first), pyramid
    int64_t size;
};
static int64_t a16(int64_t x) { return (x + 15) & ~(int64_t)15; }

// the IMU factors of a blob's window
static int snap_factors(const SnapHead &H) { return (H.parts & kSnapWindow) && H.inertial ? std::max(H.N - 1, 0) : 0; }

// the sections of a blob with head H (its counts already in range), n_fac factors holding `rows` samples in all
static SnapOff snap_layout(const SnapHead &H, int64_t n_fac, int64_t rows) {
    const bool win = H.parts & kSnapWindow, trk = H.parts & kSnapTracker;
    const int64_t T = win ? H.T : 0, N = win ? H.N : 0, F = snap_factors(H), d = win ? 15 * (int64_t)H.n_prior : 0;
    const int64_t nk = trk ? (int64_t)H.n[0] + H.n[1] : 0;
    SnapOff o{};
    int64_t p = sizeof(SnapHead);
    auto sec = [&p](int64_t &at, int64_t bytes) { at = p; p += a16(bytes); };
    sec(o.ids, 4 * T); sec(o.mask, 4 * T); sec(o.role, T); sec(o.nsmp, 4 * F);
    o.dev0 = p;
    sec(o.cst, win ? (int64_t)sizeof(WinConst) : 0);
    sec(o.tkp, 4 * T); sec(o.valid, T); sec(o.rho, 8 * T); sec(o.qual, 8 * T); sec(o.tz, 16 * T * N);
    sec(o.frames, 8 * kFrameStride * N); sec(o.imu, 8 * kImuStride * F);
    sec(o.pS, 8 * d * d); sec(o.pe, 8 * d); sec(o.px0, 8 * kFrameStride * (d / 15));
    sec(o.aux, 8 * kImuAux * n_fac); sec(o.smp, 8 * 7 * rows); sec(o.planes, 32 * (int64_t)(win ? H.n_planes : 0));
    sec(o.kz, 16 * nk); sec(o.kb, 4 * nk); sec(o.kp, 4 * nk);
    if (trk && H.levels > 0) {
        KltPyramids k;
        klt_layout(k, H.w, H.h, H.levels);
        for (int l = 0; l < H.levels; ++l) sec(o.lvl[l], (int64_t)k.lw[l] * k.lh[l]);
    }
    o.size = p;
    return o;
}

// one record of a save or restore call as the kernels read it: its blob at byte `base` of the call's area (save: the
// area holds the device region only, so base + dev0 is where that region starts), the window slot (-1: none) and the
// tracker slot's buffers (trk 0: none)
struct SnapRec {
    SnapOff o;
    int64_t base;
    int32_t slot, N, T, F, n_prior, n_planes, fac_off, n_fac;
    int32_t rows, link, trk, levels;              // link: the rows' keypoint indices are kept (else -1)
    int32_t n[2];
    double2 *kz[2];                               // the tracker slot's keypoints, births, prev_index: newest, previous
    int32_t *kb[2], *kp[2];
    uint8_t *pyr;                                 // the newest frame's pyramid
    int64_t poff[kMaxLevels];
    int32_t lw[kMaxLevels], lh[kMaxLevels];
};
static_assert(sizeof(SnapRec) % 16 == 0, "the blob area after the records starts 16-byte aligned");
struct SnapFac { int32_t factor, n; int64_t smp; };     // a factor with samples: n rows at blob byte smp
static_assert(sizeof(SnapFac) == 16, "the blob area after the factors starts 16-byte aligned");

constexpr int kSnapThreads = 256;

template <typename T>
__device__ __forceinline__ void snap_copy(T *dst, const T *src, int64_t n) {
    for (int64_t i = threadIdx.x; i < n; i += kSnapThreads) dst[i] = src[i];
}
// zero bytes [bytes, a16(bytes)) of the section at p
__device__ __forceinline__ void snap_pad(uint8_t *p, int64_t bytes) {
    for (int64_t i = bytes; i & 15; ++i) p[i] = 0;
}
// the bytes of 4-byte word q of a 16-byte chunk below `left` bytes, the others 0
__device__ __forceinline__ unsigned snap_keep(unsigned x, int64_t left, int q) {
    const int64_t k = left - 4 * q;
    return k >= 4 ? x : k <= 0 ? 0u : x & ((1u << (8 * k)) - 1u);
}
// one pyramid level of `bytes` bytes in 16-byte copies, the last chunk's bytes past the level 0
__device__ __forceinline__ void snap_level(uint4 *dst, const uint4 *src, int64_t bytes) {
    const int64_t nc = (bytes + 15) >> 4;
    for (int64_t i = threadIdx.x; i < nc; i += kSnapThreads) {
        uint4 v = src[i];
        const int64_t left = bytes - 16 * i;
        if (left < 16) { v.x = snap_keep(v.x, left, 0); v.y = snap_keep(v.y, left, 1); v.z = snap_keep(v.z, left, 2); v.w = snap_keep(v.w, left, 3); }
        dst[i] = v;
    }
}

// One CTA per save record: the device region of its blob from the slot's track table, frames, IMU records, prior,
// samples and planes, and from the tracker slot's keypoint buffers and newest pyramid.  Keypoints of frames a row does
// not observe are written 0, keypoint indices -1 without the link, the sections' padding 0.
__global__ void __launch_bounds__(kSnapThreads) bw_save_kernel(BwArgs a, const SnapRec *recs, const SnapFac *facs,
                                                                uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    const SnapOff &o = R.o;
    uint8_t *b = area + R.base;
    if (R.slot >= 0) {
        const int w = R.slot, N = R.N, T = R.T;
        const size_t base = (size_t)w * a.Mcap;
        int32_t *kp = reinterpret_cast<int32_t *>(b + o.tkp);
        double *rho = reinterpret_cast<double *>(b + o.rho), *q = reinterpret_cast<double *>(b + o.qual);
#pragma unroll 1
        for (int r = threadIdx.x; r < T; r += kSnapThreads) {
            kp[r] = R.link ? a.tkp[base + r] : -1;
            b[o.valid + r] = a.tvalid[base + r];
            rho[r] = a.trho[base + r]; q[r] = a.tqual[base + r];
        }
        double2 *z = reinterpret_cast<double2 *>(b + o.tz);
        for (int i = threadIdx.x; i < T * N; i += kSnapThreads) {
            const int r = i / N, f = i - r * N;
            z[i] = ((a.tmask[base + r] >> f) & 1u) ? a.tz[(base + r) * a.Ncap + f] : make_double2(0.0, 0.0);
        }
        // the constants with the origin the slot's solves use (the mean frame position at its last re-layout)
        WinConst *c = reinterpret_cast<WinConst *>(b + o.cst);
        snap_copy(reinterpret_cast<double *>(c), reinterpret_cast<const double *>(&a.cst[w]),
                  (int64_t)(offsetof(WinConst, pad) / sizeof(double)));
        if (threadIdx.x == 0) c->pad = 0.0;
        const size_t dcap = 15 * (size_t)a.Ncap, d = 15 * (size_t)R.n_prior;
        snap_copy(reinterpret_cast<double *>(b + o.frames), a.frames + (size_t)w * a.Ncap * kFrameStride, (int64_t)N * kFrameStride);
        snap_copy(reinterpret_cast<double *>(b + o.imu), a.imu_data + (size_t)w * a.Ncap * kImuStride, (int64_t)R.F * kImuStride);
        snap_copy(reinterpret_cast<double *>(b + o.pS), a.prior_S + w * dcap * dcap, (int64_t)(d * d));
        snap_copy(reinterpret_cast<double *>(b + o.pe), a.prior_e + w * dcap, (int64_t)d);
        snap_copy(reinterpret_cast<double *>(b + o.px0), a.prior_x0 + (size_t)w * a.Ncap * kFrameStride, (int64_t)R.n_prior * kFrameStride);
        for (int j = 0; j < R.n_fac; ++j) {
            const SnapFac f = facs[R.fac_off + j];
            const size_t F = (size_t)w * a.Ncap + f.factor;
            snap_copy(reinterpret_cast<double *>(b + o.aux) + (size_t)j * kImuAux, a.imu_aux + F * kImuAux, kImuAux);
            snap_copy(reinterpret_cast<double *>(b + f.smp), a.imu_s + F * a.Scap * 7, (int64_t)f.n * 7);
        }
        snap_copy(reinterpret_cast<double *>(b + o.planes), a.tplane + (size_t)w * a.Pcap * 4, (int64_t)R.n_planes * 4);
        if (threadIdx.x == 0) {
            snap_pad(b + o.tkp, 4 * (int64_t)T); snap_pad(b + o.valid, T); snap_pad(b + o.rho, 8 * (int64_t)T);
            snap_pad(b + o.qual, 8 * (int64_t)T); snap_pad(b + o.pS, 8 * (int64_t)(d * d)); snap_pad(b + o.pe, 8 * (int64_t)d);
            snap_pad(b + o.aux, 8 * (int64_t)kImuAux * R.n_fac); snap_pad(b + o.smp, 56 * (int64_t)R.rows);
        }
    }
    if (R.trk) {
        const int64_t nk = (int64_t)R.n[0] + R.n[1];
        double2 *z = reinterpret_cast<double2 *>(b + o.kz);
        int32_t *kb = reinterpret_cast<int32_t *>(b + o.kb), *kp = reinterpret_cast<int32_t *>(b + o.kp);
        const int n0 = R.n[0], n1 = R.n[1];
        snap_copy(z, R.kz[0], n0); snap_copy(kb, R.kb[0], n0); snap_copy(kp, R.kp[0], n0);
        snap_copy(z + n0, R.kz[1], n1); snap_copy(kb + n0, R.kb[1], n1); snap_copy(kp + n0, R.kp[1], n1);
        if (threadIdx.x == 0) { snap_pad(b + o.kb, 4 * nk); snap_pad(b + o.kp, 4 * nk); }
        for (int l = 0; l < R.levels; ++l)
            snap_level(reinterpret_cast<uint4 *>(b + o.lvl[l]), reinterpret_cast<const uint4 *>(R.pyr + R.poff[l]),
                       (int64_t)R.lw[l] * R.lh[l]);
    }
}

// One CTA per restore record: the blob's window into the slot's track table (rows [0, T)), frames, IMU records, prior,
// samples, planes and constants; its tracker part into the tracker slot's buffers (newest frame in buffer 0) and the
// newest frame's pyramid
__global__ void __launch_bounds__(kSnapThreads) bw_restore_kernel(BwArgs a, const SnapRec *recs, const SnapFac *facs,
                                                                   const uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    const SnapOff &o = R.o;
    const uint8_t *b = area + R.base;
    if (R.slot >= 0) {
        const int w = R.slot, N = R.N, T = R.T;
        const size_t base = (size_t)w * a.Mcap;
        const int32_t *id = reinterpret_cast<const int32_t *>(b + o.ids), *kp = reinterpret_cast<const int32_t *>(b + o.tkp);
        const uint32_t *m = reinterpret_cast<const uint32_t *>(b + o.mask);
        const double *rho = reinterpret_cast<const double *>(b + o.rho), *q = reinterpret_cast<const double *>(b + o.qual);
#pragma unroll 1
        for (int r = threadIdx.x; r < T; r += kSnapThreads) {
            a.tid[base + r] = id[r]; a.tmask[base + r] = m[r]; a.trole[base + r] = static_cast<int8_t>(b[o.role + r]);
            a.tkp[base + r] = R.link ? kp[r] : -1;
            a.tvalid[base + r] = b[o.valid + r];
            a.trho[base + r] = rho[r]; a.tqual[base + r] = q[r];
        }
        const double2 *z = reinterpret_cast<const double2 *>(b + o.tz);
        for (int i = threadIdx.x; i < T * N; i += kSnapThreads) {
            const int r = i / N, f = i - r * N;
            a.tz[(base + r) * a.Ncap + f] = z[i];
        }
        const size_t dcap = 15 * (size_t)a.Ncap, d = 15 * (size_t)R.n_prior;
        snap_copy(a.frames + (size_t)w * a.Ncap * kFrameStride, reinterpret_cast<const double *>(b + o.frames), (int64_t)N * kFrameStride);
        snap_copy(a.imu_data + (size_t)w * a.Ncap * kImuStride, reinterpret_cast<const double *>(b + o.imu), (int64_t)R.F * kImuStride);
        snap_copy(const_cast<double *>(a.prior_S) + w * dcap * dcap, reinterpret_cast<const double *>(b + o.pS), (int64_t)(d * d));
        snap_copy(const_cast<double *>(a.prior_e) + w * dcap, reinterpret_cast<const double *>(b + o.pe), (int64_t)d);
        snap_copy(const_cast<double *>(a.prior_x0) + (size_t)w * a.Ncap * kFrameStride, reinterpret_cast<const double *>(b + o.px0),
                  (int64_t)R.n_prior * kFrameStride);
        for (int j = 0; j < R.n_fac; ++j) {
            const SnapFac f = facs[R.fac_off + j];
            const size_t F = (size_t)w * a.Ncap + f.factor;
            snap_copy(a.imu_aux + F * kImuAux, reinterpret_cast<const double *>(b + o.aux) + (size_t)j * kImuAux, kImuAux);
            snap_copy(a.imu_s + F * a.Scap * 7, reinterpret_cast<const double *>(b + f.smp), (int64_t)f.n * 7);
        }
        snap_copy(a.tplane + (size_t)w * a.Pcap * 4, reinterpret_cast<const double *>(b + o.planes), (int64_t)R.n_planes * 4);
        snap_copy(reinterpret_cast<double *>(&a.cst[w]), reinterpret_cast<const double *>(b + o.cst),
                  (int64_t)(sizeof(WinConst) / sizeof(double)));
    }
    if (R.trk) {
        const double2 *z = reinterpret_cast<const double2 *>(b + o.kz);
        const int32_t *kb = reinterpret_cast<const int32_t *>(b + o.kb), *kp = reinterpret_cast<const int32_t *>(b + o.kp);
        const int n0 = R.n[0], n1 = R.n[1];
        snap_copy(R.kz[0], z, n0); snap_copy(R.kb[0], kb, n0); snap_copy(R.kp[0], kp, n0);
        snap_copy(R.kz[1], z + n0, n1); snap_copy(R.kb[1], kb + n0, n1); snap_copy(R.kp[1], kp + n0, n1);
        for (int l = 0; l < R.levels; ++l)         // the level's storage is 256-byte aligned: the last chunk fits
            snap_level(reinterpret_cast<uint4 *>(R.pyr + R.poff[l]), reinterpret_cast<const uint4 *>(b + o.lvl[l]),
                       (int64_t)R.lw[l] * R.lh[l]);
    }
}

// After the re-layout of a restore (which sets each window's origin to its mean frame position), one CTA per record:
// the origin the window had when it was saved, so that its next solve or drop runs exactly as the source's would
__global__ void __launch_bounds__(32) bw_restore_origin_kernel(BwArgs a, const SnapRec *recs, const uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    if (R.slot < 0 || threadIdx.x >= 3) return;
    const WinConst *c = reinterpret_cast<const WinConst *>(area + R.base + R.o.cst);
    a.cst[R.slot].origin[threadIdx.x] = c->origin[threadIdx.x];
}

// a tracker slot's keypoint buffers as a SnapRec names them (the newest frame's first), and pyramid k of its cache c
// (c null or k < 0: none)
static void snap_tracker(SnapRec &r, const SlotKeypoints &K, const KltPyramids *c, int k) {
    r.trk = 1; r.n[0] = K.n; r.n[1] = K.prev_n;
    for (int j = 0; j < 2; ++j) {
        const int b = j ? 1 - K.cur : K.cur;
        r.kz[j] = K.z(b); r.kb[j] = K.birth(b); r.kp[j] = K.prev(b);
    }
    if (!c || k < 0) return;
    r.levels = c->levels; r.pyr = c->pyr[k].d;
    for (int l = 0; l < c->levels; ++l) { r.poff[l] = (int64_t)c->off[l]; r.lw[l] = c->lw[l]; r.lh[l] = c->lh[l]; }
}

// the pyramid of a tracker slot's newest frame in its cache, -1: none
static int snap_pyramid(const KltBatchState &B, int t) {
    if ((size_t)t >= B.slots.size()) return -1;
    for (int k = 0; k < 2; ++k)
        if (B.slots[t].pyr_id[k] == B.kps[t].frame_id && B.slots[t].pyr[k].d) return k;
    return -1;
}

// the kernels' record of blob H with sections o: window slot `slot` (-1: none), the tracker part when trk
static SnapRec snap_rec(const SnapHead &H, const SnapOff &o, int slot, int64_t base, int fac_off, int n_fac, int rows) {
    SnapRec r{};
    r.o = o; r.base = base; r.slot = slot; r.fac_off = fac_off;
    if (slot >= 0) {
        r.N = H.N; r.T = H.T; r.F = snap_factors(H); r.n_prior = H.n_prior; r.n_planes = H.n_planes;
        r.n_fac = n_fac; r.rows = rows;
    }
    return r;
}

// ---- pvio_b200_batch_window_landmarks: every row's world point, and for the rows the solve treats as landmarks the
// point's covariance from the covariance call's Sigma_xi and the landmark's Schur records
struct BwLmk {
    int32_t slot, n_rows, T;      // rows written; live rows of the slot
    int32_t rows_off;             // ints into the call's row list; -1: rows [0, n_rows) of the slot (every live track)
    int32_t out_off;              // rows into the call's points
    int32_t cov, cov_off, pad;    // index among the records with a covariance (-1: none); rows into its outputs
};
struct LmkArgs {
    const BwLmk *rec;             // [n]
    const int32_t *rows;          // the named rows of every record
    const int32_t *cov_rec;       // [n_cov] the record of each covariance record
    double *pts;                  // out: [rows][3]
    int32_t *role;                // out: [rows]
    int32_t *lm_of;               // scratch: [n_cov][Mcap] the packed landmark of each row of the slot, -1: none
    const int32_t *status;        // [n_cov] cov_kernel's status
    const double *sig_xi;         // [n_cov][Ncap][Ncap][36] Sigma_xi of every frame pair (cov_kernel)
    double *pcov, *var;           // out: [cov rows][9], [cov rows]
};
constexpr int kLmkWarps = 4;

// One CTA per record: Track::get_landmark_point() of every row; for a record with a covariance, the packed landmark of
// every row of its slot (bw_layout_kernel's lm_row inverted) for bw_landmark_cov_kernel
__global__ void __launch_bounds__(kBwThreads) bw_landmark_point_kernel(BwArgs a, LmkArgs L) {
    const BwLmk r = L.rec[blockIdx.x];
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    for (int k = threadIdx.x; k < r.n_rows; k += kBwThreads) {
        const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
        bw_landmark_point(a, base + row, fr, c, L.pts + 3 * ((size_t)r.out_off + k));
        L.role[r.out_off + k] = a.trole[base + row];
    }
    if (r.cov < 0) return;
    int32_t *lm = L.lm_of + (size_t)r.cov * a.Mcap;
    for (int q = threadIdx.x; q < r.T; q += kBwThreads) lm[q] = -1;
    __syncthreads();
    for (int lp = threadIdx.x; lp < a.hdr[w].M; lp += kBwThreads) lm[a.lm_row[base + lp]] = lp;
}

// row i of X_l = [[x]x, I]
__device__ __forceinline__ void lmk_xrow(const double *x, int i, double *o) {
    o[0] = i == 1 ? x[2] : (i == 2 ? -x[1] : 0.0);
    o[1] = i == 0 ? -x[2] : (i == 2 ? x[0] : 0.0);
    o[2] = i == 0 ? x[1] : (i == 1 ? -x[0] : 0.0);
    o[3] = i == 0 ? 1.0 : 0.0; o[4] = i == 1 ? 1.0 : 0.0; o[5] = i == 2 ? 1.0 : 0.0;
}

// One warp per row of a record with a covariance (grid: covariance records x row blocks).  Var(rho) as cov_lm_kernel
// forms it (ba_cov_lm.cuh), C = Cov(xi_a, rho) = -(Sigma_xi h_l)_a / H_ll from the same products, then
//   Sigma_x = X Sigma_aa X^T - X C c^T - c C^T X^T + c c^T Var(rho),  X = [[x - o]x, I], c = -(x - c_a) / rho,
// o the window's origin, about which frame_T takes xi,
// the upper triangle on six lanes, mirrored (exactly symmetric).  NaN for a row that is not a landmark of the solve and
// for every row of a record whose factorisation failed.
template <typename real>
__global__ void __launch_bounds__(32 * kLmkWarps) bw_landmark_cov_kernel(BwArgs a, LmkArgs L) {
    __shared__ double u_sm[kLmkWarps][6 * kMaxFrames];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int crec = blockIdx.x;                     // the covariance record
    const BwLmk r = L.rec[L.cov_rec[crec]];
    const int k = blockIdx.y * kLmkWarps + wv;
    if (k >= r.n_rows) return;
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
    const int lm = L.lm_of[(size_t)crec * a.Mcap + row];
    double *P = L.pcov + 9 * ((size_t)r.cov_off + k);
    double *V = L.var + r.cov_off + k;
    if (lm < 0 || L.status[crec] != PVIO_B200_OK) {
        if (lane < 9) P[lane] = CUDART_NAN;
        if (lane == 0) *V = CUDART_NAN;
        return;
    }
    const int N = a.hdr[w].N;
    const unsigned fixed = (unsigned)a.hdr[w].fixed_mask & ((1u << N) - 1u);
    const real *hs = reinterpret_cast<const real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    double *u = u_sm[wv];
    cov_lm_h(hs, a.Mcap, lm, N, fixed, lane, u);
    __syncwarp();
    const double *X = L.sig_xi + (size_t)crec * a.Ncap * a.Ncap * 36;
    const int an = __ffs(a.tmask[base + row]) - 1;
    double srow = 0.0;
    const double q = cov_lm_quad<true>(u, X, N, lane, an, srow);
    const double hll = a.lm_aux[base + lm].hll;
    const double var = cov_lm_var(hll, q);
    double C[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) C[i] = -__shfl_sync(0xffffffffu, srow, (6 * an + i) & 31) / hll;
    const double2 z = a.tz[(base + row) * a.Ncap + an];
    const double rho = a.trho[base + row];
    double qc[4], pc[3], x[3];
    bw_cam_pose(a.frames + ((size_t)w * a.Ncap + an) * kFrameStride, a.cst[w], qc, pc);
    bw_world_point(qc, pc, z.x, z.y, rho, x);
    const double cl[3] = {-(x[0] - pc[0]) / rho, -(x[1] - pc[1]) / rho, -(x[2] - pc[2]) / rho};
    const double *o = a.cst[w].origin;                  // xi is taken about the window's origin (frame_T)
    const double xo[3] = {x[0] - o[0], x[1] - o[1], x[2] - o[2]};
    if (lane < 6) {
        const int i = lane < 3 ? 0 : (lane < 5 ? 1 : 2), j = lane < 3 ? lane : (lane < 5 ? lane - 2 : 2);
        double Xi[6], Xj[6];
        lmk_xrow(xo, i, Xi);
        lmk_xrow(xo, j, Xj);
        const double *S = X + ((size_t)an * N + an) * 36;
        double s = 0.0, bi = 0.0, bj = 0.0;
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            double t = 0.0;
#pragma unroll
            for (int n = 0; n < 6; ++n) t += S[m * 6 + n] * Xj[n];
            s += Xi[m] * t;
            bi += Xi[m] * C[m];
            bj += Xj[m] * C[m];
        }
        const double cli = i == 0 ? cl[0] : (i == 1 ? cl[1] : cl[2]), clj = j == 0 ? cl[0] : (j == 1 ? cl[1] : cl[2]);
        const double v = s - bi * clj - cli * bj + cli * clj * var;
        P[3 * i + j] = v;
        P[3 * j + i] = v;
    }
    if (lane == 0) *V = var;
}

// ---- pvio_b200_batch_window_trajectory: the state at any time inside the window, forward from the preceding frame
// through the part of its IMU factor's kept samples up to that time, and its covariance
struct BwTraj {
    int32_t slot, N, n_times, cov;    // cov: index among the records with a covariance (-1: none asked; -2: asked, but
                                      // no factor holds samples)
    int64_t t_off;                    // rows into the call's times, states and frames
    int64_t cov_off;                  // doubles into the covariance scratch: the joint block of the frames that own a
                                      // factor with samples (CovRec::cov_off)
    int64_t scov_off;                 // rows into the call's state covariances
    int32_t ns[kMaxFrames];           // samples of factor k (frames k, k + 1), 0: none
};
static_assert(sizeof(BwTraj) % sizeof(double) == 0, "records are staged as whole 8-byte words");
struct TrajArgs {
    const BwTraj *rec;                // [n]
    const double *times;              // [rows]
    double *states;                   // out: [rows][16]
    int32_t *frame;                   // out: [rows]
    double *scov;                     // out: [cov rows][225]
    const double *jcov;               // cov_kernel's joint blocks (scratch)
    const int32_t *status;            // [n_cov] cov_kernel's status
    int covs;                         // 1: the per-warp covariance scratch is laid out
};
// per warp of bw_trajectory_kernel: the chain, the emitted copy, then (with covariances) four 15 x 15 matrices
__host__ __device__ constexpr size_t traj_warp_bytes(bool covs) { return 2 * sizeof(ImuWarpSm) + (covs ? 4 * 225 * 8 : 0); }

// the first of the n sorted times t[i] that is >= x (upper: > x)
__device__ __forceinline__ int traj_bound(const double *t, int n, double x, bool upper) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (upper ? t[m] <= x : t[m] < x) lo = m + 1;
        else hi = m;
    }
    return lo;
}

// queries [q0, q1) of record r, which no factor takes: frame -1, a zero state, a NaN covariance.  One warp.
__device__ __forceinline__ void none_rows(const TrajArgs &T, const BwTraj &r, int lane, int q0, int q1, bool cov) {
    for (int q = q0; q < q1; ++q) {
        const size_t row = r.t_off + q;
        if (lane < 16) T.states[16 * row + lane] = 0.0;
        if (lane == 0) T.frame[row] = -1;
        if (cov)
            for (int e = lane; e < 225; e += 32) T.scov[225 * ((size_t)r.scov_off + q) + e] = CUDART_NAN;
    }
}

// One CTA per record, one warp per factor k with samples (warp k).  The warp's queries are the times t >= s_0.t of its
// factor and below s_0.t of the next factor with samples (so k is the largest such factor whose s_0.t <= t), found by
// binary search; it takes those at most its t_end, or all of them when factor k + 1 holds samples.  It walks its
// samples once, as imu_integrate_warp does (imu_step_warp), and emits each query as the walk passes it: the increment
// of the last sample at or before t, over t - s_j.t, goes onto a copy of the chain, which is what imu_integrate_warp
// gives for the samples at or before t with t_end = t.  Then PreIntegrator::predict from frame k's state, and with a
// covariance Phi Sigma_k Phi^T + Psi Sigma_delta Psi^T (imu_factor_propagate), Sigma_delta the partial increment's
// covariance itself.  Times no warp takes (before the first sample, past a factor's t_end, over a factor without
// samples) get frame -1, a zero state and a NaN covariance: warp 0 writes those before the earliest s_0.t, each warp
// those past its t_end.
__global__ void __launch_bounds__(32 * (kMaxFrames - 1)) bw_trajectory_kernel(BwArgs a, TrajArgs T) {
    extern __shared__ __align__(16) unsigned char traj_sm[];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const BwTraj &r = T.rec[blockIdx.x];
    const int nf = r.N - 1, nq = r.n_times;
    const double *tq = T.times + r.t_off;
    const size_t F0 = (size_t)r.slot * a.Ncap;
    auto s0 = [&](int k) { return a.imu_s[(F0 + k) * a.Scap * 7]; };
    const bool cov = r.cov != -1;                           // -2: covariances asked, no factor holds samples
    const bool cov_ok = r.cov >= 0 && T.status[r.cov] == PVIO_B200_OK;
    if (wv == 0) {
        double lo = CUDART_INF;
        for (int j = 0; j < nf; ++j)
            if (r.ns[j] > 0) lo = fmin(lo, s0(j));
        none_rows(T, r, lane, 0, traj_bound(tq, nq, lo, false), cov);
    }
    const int k = wv;
    if (k >= nf || r.ns[k] == 0) return;
    const size_t F = F0 + k;
    const double lo = s0(k);
    double hi = CUDART_INF;
    for (int j = k + 1; j < nf; ++j)
        if (r.ns[j] > 0) hi = fmin(hi, s0(j));
    const double *aux = a.imu_aux + F * kImuAux, t_end = aux[0];
    const int q0 = traj_bound(tq, nq, lo, false), q1 = max(q0, traj_bound(tq, nq, hi, false));
    const int q2 = (k + 1 < nf && r.ns[k + 1] > 0) ? q1 : min(q1, max(q0, traj_bound(tq, nq, t_end, true)));
    none_rows(T, r, lane, q2, q1, cov);
    if (q0 >= q2) return;
    unsigned char *base = traj_sm + (size_t)wv * traj_warp_bytes(T.covs);
    ImuWarpSm &S = *reinterpret_cast<ImuWarpSm *>(base), &E = *reinterpret_cast<ImuWarpSm *>(base + sizeof(ImuWarpSm));
    double *A = reinterpret_cast<double *>(base + 2 * sizeof(ImuWarpSm)), *B = A + 225, *C = B + 225, *D = C + 225;
    const double *x = a.frames + F * kFrameStride;
    const double bg[3] = {x[10], x[11], x[12]}, ba[3] = {x[13], x[14], x[15]};
    const double *smp = a.imu_s + F * a.Scap * 7, *noise = aux + 1;
    const int m = r.ns[k];
    // Sigma_k: frame k's diagonal block of the joint covariance of the frames that own a factor with samples
    unsigned has = 0;
    for (int j = 0; j < nf; ++j) has |= (r.ns[j] > 0 ? 1u : 0u) << j;
    const int K15 = 15 * __popc(has), p15 = 15 * __popc(has & ((1u << k) - 1u));
    const double *Sk = T.jcov + r.cov_off + (size_t)p15 * K15 + p15;
    imu_reset_warp(S, lane);
    int q = q0;
    for (int j = 0; j < m && q < q2; ++j) {
        const double *d = smp + (size_t)j * 7;
        const bool last = j + 1 == m;
        const double t_next = last ? t_end : smp[(size_t)(j + 1) * 7];
        for (; q < q2 && (last || tq[q] < t_next); ++q) {   // the queries whose last sample is s_j
            imu_copy_warp(S, E, lane);
            imu_step_warp(E, lane, d, tq[q] - d[0], bg, ba, noise);
            const size_t row = r.t_off + q;
            if (lane == 0) {
                bw_imu_predict(x, E.tsum, E.q, E.p, E.v, T.states + 16 * row);
                T.frame[row] = k;
            }
            if (!cov) continue;
            double *out = T.scov + 225 * (size_t)(r.scov_off + q);
            if (!cov_ok) {
                for (int e = lane; e < 225; e += 32) out[e] = CUDART_NAN;
                continue;
            }
            for (int e = lane; e < 225; e += 32) {
                const int i = e / 15, c = e % 15;
                A[e] = 0.5 * (Sk[(size_t)i * K15 + c] + Sk[(size_t)c * K15 + i]);
                D[e] = (i < 9 && c < 9) ? E.C[i * 9 + c]
                     : (i >= 9 && i < 12 && c >= 9 && c < 12) ? E.cbg[(i - 9) * 3 + c - 9]
                     : (i >= 12 && c >= 12) ? E.cba[(i - 12) * 3 + c - 12] : 0.0;
            }
            __syncwarp();
            double Rs[9], dR[9];
            quat_to_mat(x, Rs);
            quat_to_mat(E.q, dR);
            const ImuFactorJac f{E.tsum, E.p, E.v, E.dq_dbg, E.dp_dbg, E.dp_dba, E.dv_dbg, E.dv_dba};
            imu_factor_propagate(A, B, C, D, f, Rs, dR, lane);
            for (int e = lane; e < 225; e += 32) {
                const int i = e / 15, c = e % 15;
                out[e] = 0.5 * ((A[e] + D[e]) + (A[c * 15 + i] + D[c * 15 + i]));
            }
            __syncwarp();
        }
        if (!last && q < q2) imu_step_warp(S, lane, d, t_next - d[0], bg, ba, noise);
    }
}

}  // namespace pvio

using namespace pvio;

extern "C" {

int pvio_b200_batch_window_reset(pvio_b200_handle hh, int slot, const pvio_b200_window *w) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w) return PVIO_B200_EINVAL;
    if (slot < 0 || slot >= h->W) return fail(h, PVIO_B200_EINVAL, "batch_window_reset: slot out of range");
    if (w->n_planes > 0 || w->n_plane_tracks > 0) return fail(h, PVIO_B200_EINVAL, "batch_window_reset: resident windows carry no planes");
    TRY(ensure_bw(h));
    if (w->use_inertial) TRY(ensure_inertial(h));
    std::vector<WinSlot> next(1);             // nothing of a former pack or resident window survives
    next[0].resident = true; next[0].inertial = w->use_inertial ? 1 : 0;
    next[0].n_samples.assign(h->Ncap, 0);
    WinConst &C = h->cst.h[slot];
    C = win_const(w);
    CK(h, cudaMemcpyAsync(h->cst.dslot(slot), &C, sizeof(WinConst), cudaMemcpyHostToDevice, h->stream));
    Stage S(h->bw.stage, &h->bw.scratch);
    const Relayout lay(S, &slot, next);
    TRY(S.place(h, true));
    TRY(lay.launch(h, S, false));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, &slot, next);
    return 0;
}

int pvio_b200_batch_window_set_prior(pvio_b200_handle hh, int slot, int n_prior, const double *S, const double *e,
                                     const double *state0) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_slots(h, 1, &slot, "batch_window_set_prior: bad slot"));
    const WinSlot &s = h->slots[slot];
    if (n_prior < 0 || (n_prior > 0 && (!S || !e || !state0))) return fail(h, PVIO_B200_EINVAL, "batch_window_set_prior: null prior");
    if (!s.inertial && n_prior > 0) return fail(h, PVIO_B200_EINVAL, "batch_window_set_prior: the window carries no motion states");
    if (n_prior > s.N) return fail(h, PVIO_B200_EINVAL, "batch_window_set_prior: prior over more frames than the window holds");
    const size_t d = 15 * (size_t)n_prior;
    if (d > 0) {
        memcpy(h->prior_S.slot(slot), S, sizeof(double) * d * d);
        memcpy(h->prior_e.slot(slot), e, sizeof(double) * d);
        memcpy(h->prior_x0.slot(slot), state0, sizeof(double) * n_prior * kFrameStride);
        CK(h, cudaMemcpyAsync(h->prior_S.dslot(slot), h->prior_S.slot(slot), sizeof(double) * d * d, cudaMemcpyHostToDevice, h->stream));
        CK(h, cudaMemcpyAsync(h->prior_e.dslot(slot), h->prior_e.slot(slot), sizeof(double) * d, cudaMemcpyHostToDevice, h->stream));
        CK(h, cudaMemcpyAsync(h->prior_x0.dslot(slot), h->prior_x0.slot(slot), sizeof(double) * n_prior * kFrameStride,
                              cudaMemcpyHostToDevice, h->stream));
    }
    std::vector<WinSlot> next(1, s);
    next[0].n_prior = next[0].prior_resident = n_prior;
    Stage st(h->bw.stage, &h->bw.scratch);
    const Relayout lay(st, &slot, next);
    TRY(st.place(h, true));
    TRY(lay.launch(h, st, n_prior > 0));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, &slot, next);
    return 0;
}

int pvio_b200_batch_window_edit(pvio_b200_handle hh, int n, const pvio_b200_window_edit *edits) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !edits)) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: bad edit list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = edits[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_edit: bad slot list"));
    // every edit is applied to a copy of its slot's host mirror; nothing is staged before all of them passed
    std::vector<WinSlot> next(n);
    std::vector<BwEdit> recs(n);
    std::vector<int32_t> rm;
    std::vector<BwNew> nws;
    std::vector<BwObs> obs;
    std::vector<double> xs;
    int out_ints = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_edit &E = edits[i];
        WinSlot s = h->slots[E.slot];
        BwEdit &R = recs[i];
        R = BwEdit{};
        R.slot = E.slot; R.N_old = s.N; R.T_old = (int)s.ids.size(); R.frame = -1;
        if (E.n_new_tracks < 0 || E.n_obs < 0 || E.n_remove < 0 ||
            (E.n_new_tracks > 0 && (!E.new_frame || !E.new_z || !E.new_inv_depth)) ||
            (E.n_obs > 0 && (!E.obs_track || !E.obs_frame || !E.obs_z)) || (E.n_remove > 0 && !E.remove))
            return fail(h, PVIO_B200_EINVAL, "batch_window_edit: null array");
        if (E.replace_last || E.state || E.n_new_tracks > 0 || E.n_obs > 0) s.link = false;   // the newest frame changes
        if (E.replace_last) {                                         // map->erase_frame(frame_num - 1)
            if (s.N < 1) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: replace_last on an empty window");
            if (s.N - 1 < s.n_prior) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: the newest frame is covered by the prior");
            for (uint32_t &m : s.mask) m &= ~(1u << (s.N - 1));
            s.fixed &= ~(1 << (s.N - 1));
            if (s.N >= 2) s.n_samples[s.N - 2] = 0;                   // the replaced frame's samples leave
            --s.N;
            R.replace_last = 1;
        }
        // removals are looked up in the table as it stands before the call (they are applied after the observations,
        // which they make moot; a track cannot be new and removed in one edit)
        std::vector<int32_t> removed;
        R.rm_off = (int)rm.size();
        for (int k = 0; k < E.n_remove; ++k) {
            const int r = find_row(s, E.remove[k]);
            if (r < 0 || s.mask[r] == 0u) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: unknown or dead track removed");
            s.mask[r] = 0u;
            rm.push_back(r);
            removed.push_back(E.remove[k]);
        }
        R.n_rm = E.n_remove;
        std::sort(removed.begin(), removed.end());
        compact_rows(s, 0);
        if (E.state) {
            if (s.N >= h->Ncap) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: window of more than max_frames frames");
            const bool imu = s.inertial && s.N > 0;
            if (imu && !E.imu_record) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: an inertial window needs the IMU record to the previous frame");
            R.frame = s.N; R.has_imu = imu ? 1 : 0; R.x_off = (int)xs.size();
            xs.insert(xs.end(), E.state, E.state + kFrameStride);
            if (imu) xs.insert(xs.end(), E.imu_record, E.imu_record + kImuStride);
            if (E.fixed) s.fixed |= 1 << s.N;
            if (imu) s.n_samples[s.N - 1] = 0;                          // the new factor holds its edit record only
            ++s.N;
        }
        R.new_off = (int)nws.size(); R.n_new = E.n_new_tracks;
        for (int k = 0; k < E.n_new_tracks; ++k) {
            const int f = E.new_frame[k];
            if (f < 0 || f >= s.N) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: track starts outside the window");
            BwNew t{(int32_t)s.ids.size(), s.next_id, f, 0, E.new_z[2 * k], E.new_z[2 * k + 1], E.new_inv_depth[k]};
            s.ids.push_back(s.next_id++); s.mask.push_back(1u << f); s.role.push_back(-1);
            nws.push_back(t);
        }
        R.obs_off = (int)obs.size();
        for (int k = 0; k < E.n_obs; ++k) {
            const int32_t id = E.obs_track[k];
            const int f = E.obs_frame[k];
            if (f < 0 || f >= s.N) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: observation outside the window");
            if (std::binary_search(removed.begin(), removed.end(), id)) continue;
            const int r = find_row(s, id);
            if (r < 0) return fail(h, PVIO_B200_EINVAL, "batch_window_edit: observation of an unknown or dead track");
            if (f <= 31 - __builtin_clz(s.mask[r]))
                return fail(h, PVIO_B200_EINVAL, "batch_window_edit: observations of a track arrive in increasing frame order");
            s.mask[r] |= 1u << f;
            obs.push_back(BwObs{r, f, E.obs_z[2 * k], E.obs_z[2 * k + 1]});
        }
        R.n_obs = (int)obs.size() - R.obs_off;
        TRY(check_window(h, s));
        R.out_off = out_ints;
        out_ints += 1 + E.n_new_tracks;
        next[i] = std::move(s);
    }
    TRY(ensure_plane_tables(h, next));                 // observations of plane tracks may outgrow the plane tables
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto ed = S.up(recs);
    const auto nw = S.up(nws);
    const auto ob = S.up(obs);
    const auto x = S.up(xs);
    const auto rmv = S.up(rm), out = S.add<int32_t>(Stage::kDown, out_ints);
    const Relayout lay(S, slots.data(), next);
    TRY(S.place(h, true));
    bw_edit_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(ed), S.dev(rmv), S.dev(nw), S.dev(ob),
                                                    S.dev(x), S.dev(out));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(lay.launch(h, S, false));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    const int32_t *res = S.host(out);
    commit(h, slots.data(), next);
    for (int i = 0; i < n; ++i) {
        const int32_t *r = res + recs[i].out_off;
        if (r[0] != (int32_t)h->slots[slots[i]].ids.size())
            return fail(h, PVIO_B200_ECUDA, "batch_window_edit: the device track table disagrees with the host's");
        if (edits[i].new_ids) memcpy(edits[i].new_ids, r + 1, sizeof(int32_t) * edits[i].n_new_tracks);
    }
    return 0;
}

int pvio_b200_batch_window_set_planes(pvio_b200_handle hh, int n, const pvio_b200_window_planes *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_set_planes: bad slot list"));
    // every record is applied to a copy of its slot's host mirror; nothing is staged before all of them passed
    std::vector<WinSlot> next(n);
    std::vector<BwPlanes> recs(n);
    std::vector<BwRole> roles;
    std::vector<double> params;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_planes &R = records[i];
        WinSlot s = h->slots[R.slot];
        if (R.n_planes < -1 || R.n_planes > h->Pcap) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: plane count outside -1 (keep) .. 4");
        if (R.n_set < 0 || (R.n_set > 0 && (!R.track || !R.role)) || (R.n_planes > 0 && !R.plane_param))
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: null array");
        recs[i] = BwPlanes{R.slot, std::max(R.n_planes, 0), R.n_set, (int32_t)roles.size(), (int32_t)params.size(), 0};
        if (R.n_planes >= 0) {
            for (int k = 0; k < 4 * R.n_planes; ++k)
                if (!std::isfinite(R.plane_param[k])) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: non-finite plane parameters");
            params.insert(params.end(), R.plane_param, R.plane_param + 4 * R.n_planes);
            s.n_planes = R.n_planes;
        }
        std::vector<uint8_t> named(s.ids.size(), 0);
        for (int k = 0; k < R.n_set; ++k) {
            const int r = find_row(s, R.track[k]);
            if (r < 0) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: unknown or dead track");
            if (named[r]) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: a track named twice");
            named[r] = 1;
            const int role = R.role[k];
            if (role < -2 || role >= s.n_planes) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: role not -1, -2 or a plane of the slot");
            const double rho = R.inv_depth ? R.inv_depth[k] : NAN;
            if (std::isinf(rho)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: infinite inverse depth");
            s.role[r] = (int8_t)role;
            roles.push_back(BwRole{r, role, rho});
        }
        for (int8_t ro : s.role)
            if (ro >= s.n_planes) return fail(h, PVIO_B200_EINVAL, "batch_window_set_planes: a track keeps a plane the slot no longer has");
        TRY(check_window(h, s));
        next[i] = std::move(s);
    }
    TRY(ensure_plane_tables(h, next));
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto ro = S.up(roles);
    const auto pa = S.up(params);
    const Relayout lay(S, slots.data(), next);
    TRY(S.place(h, true));
    bw_planes_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rec), S.dev(ro), S.dev(pa));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(lay.launch(h, S, false));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, slots.data(), next);
    return 0;
}

int pvio_b200_batch_window_solve(pvio_b200_handle hh, int n, const int32_t *slots, const pvio_b200_options *opt,
                                 pvio_b200_summary *summaries) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return solve_slots(h, n, slots, opt, !opt || opt->run_postpass, summaries);
}

int pvio_b200_batch_window_drop_victim(pvio_b200_handle hh, int n, const int32_t *slots, double *S_out, int64_t S_stride,
                                       double *e_out, int64_t e_stride) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_slots(h, n, slots, "batch_window_drop_victim: bad slot list"));
    if (n == 0) return 0;
    std::vector<WinSlot> next(n);
    for (int i = 0; i < n; ++i) {
        WinSlot s = h->slots[slots[i]];
        if (!s.inertial) return fail(h, PVIO_B200_EINVAL, "batch_window_drop_victim: the window must carry motion states");
        if (s.N < 2) return fail(h, PVIO_B200_EINVAL, "batch_window_drop_victim: a window needs at least two frames");
        const int dk = 15 * (s.N - 1);
        if (!marg_eig_fits(dk))
            return fail(h, PVIO_B200_EINVAL, "batch_window_drop_victim: window too large for the shared-memory eigen-solver (15 (N - 1) <= 165)");
        if ((S_out && S_stride < (int64_t)dk * dk) || (e_out && e_stride < dk))
            return fail(h, PVIO_B200_EINVAL, "batch_window_drop_victim: output stride smaller than a window's prior");
        compact_rows(s, 1);                                            // map.cpp:76-88 on the host mirror
        --s.N; s.fixed >>= 1; s.n_prior = s.prior_resident = s.N;
        s.n_samples.erase(s.n_samples.begin());                        // factor 0 leaves, the others shift with their frames
        s.n_samples.push_back(0);
        TRY(check_window(h, s));
        next[i] = std::move(s);
    }
    std::vector<BwLayout> before(n);
    for (int i = 0; i < n; ++i) before[i] = layout_of(slots[i], h->slots[slots[i]]);
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto b = S.up(before);
    const Relayout lay(S, slots, next);
    TRY(S.place(h, true));
    TRY(run_marg(h, n, 0, true, true, slots, S.dev(lay.slots)));
    for (int i = 0; i < n; ++i) {
        const size_t dk = 15 * (size_t)(h->slots[slots[i]].N - 1);
        if (S_out) CK(h, cudaMemcpyAsync(S_out + i * S_stride, h->prior_S.dslot(slots[i]), sizeof(double) * dk * dk, cudaMemcpyDeviceToHost, h->stream));
        if (e_out) CK(h, cudaMemcpyAsync(e_out + i * e_stride, h->prior_e.dslot(slots[i]), sizeof(double) * dk, cudaMemcpyDeviceToHost, h->stream));
    }
    bw_drop_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(b));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(lay.launch(h, S, true));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, slots, next);
    return 0;
}

// the landmark index of every row of a slot in its packed window (rows of role < 0 with >= 2 observations, stably by
// anchor, as bw_layout_kernel orders them), -1 for the other rows
static std::vector<int32_t> landmark_of_rows(const WinSlot &s) {
    const int T = (int)s.ids.size();
    std::vector<int32_t> lm(T, -1);
    int k = 0;
    for (int a = 0; a < kMaxFrames; ++a)
        for (int r = 0; r < T; ++r)
            if (s.role[r] < 0 && __builtin_popcount(s.mask[r]) >= 2 && __builtin_ctz(s.mask[r]) == a) lm[r] = k++;
    return lm;
}

int pvio_b200_batch_window_covariance(pvio_b200_handle hh, int n, pvio_b200_window_covariance *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const char *what = "batch_window_covariance";
    auto bad = [&](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); };
    if (n < 0 || (n > 0 && !records)) return bad("bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n), frames;
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_covariance: bad slot list"));
    // every record checked against its slot's host mirror before anything is staged
    std::vector<CovRec> recs(n);
    std::vector<CovLm> lms;
    int64_t cov_n = 0, sig_n = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_covariance &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (s.N < 1) return bad("a window without frames");
        if (R.n_frames < 0 || R.n_frames > s.N || R.n_tracks < 0 || R.n_tracks > (int)s.ids.size())
            return bad("a frame or track count out of range");
        if (R.n_frames == 0 && R.n_tracks == 0) return bad("a record asking for nothing");
        if (R.n_frames > 0 && (!R.frames || !R.cov)) return bad("frames or cov missing");
        if (R.n_tracks > 0 && (!R.tracks || !R.inv_depth_var)) return bad("tracks or inv_depth_var missing");
        uint32_t seen = 0;
        for (int k = 0; k < R.n_frames; ++k) {
            const int f = R.frames[k];
            if (f < 0 || f >= s.N) return bad("a frame out of range");
            if ((seen >> f) & 1u) return bad("a frame named twice");
            seen |= 1u << f;
        }
        if (cov_smem_bytes(h->hdr.h[R.slot]) > 220 * 1024) return bad("reduced system too large for shared memory");
        const std::vector<int32_t> lm = R.n_tracks > 0 ? landmark_of_rows(s) : std::vector<int32_t>();
        std::vector<uint8_t> taken(s.ids.size(), 0);
        for (int k = 0; k < R.n_tracks; ++k) {
            const auto it = std::lower_bound(s.ids.begin(), s.ids.end(), R.tracks[k]);      // rows are in id order
            if (it == s.ids.end() || *it != R.tracks[k]) return bad("a track that is not live in its slot");
            const size_t r = it - s.ids.begin();
            if (taken[r]) return bad("a track named twice");
            taken[r] = 1;
            lms.push_back(CovLm{i, R.slot, lm[r], 0});
        }
        const int64_t D = (s.inertial ? 15 : 6) * (int64_t)s.N;
        recs[i] = CovRec{R.slot, R.n_frames, (int32_t)frames.size(), 0, cov_n, sig_n};
        frames.insert(frames.end(), R.frames, R.frames + R.n_frames);
        cov_n += 225 * (int64_t)R.n_frames * R.n_frames;
        sig_n += D * D;
    }
    const int n_lm = (int)lms.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto fr = S.up(frames);
    const auto lmv = S.up(lms);
    const auto sl = S.add(Stage::kUp, n, slots.data());
    const auto cov = S.add<double>(Stage::kDown, (size_t)cov_n), var = S.add<double>(Stage::kDown, (size_t)n_lm);
    const auto st = S.add<int32_t>(Stage::kDown, n);
    const auto sig = S.add<double>(Stage::kScratch, (size_t)sig_n);
    const auto sxi = S.add<double>(Stage::kScratch, (size_t)n * h->Ncap * h->Ncap * 36);
    TRY(S.place(h, true));
    TRY(run_covariance(h, n, slots.data(), S.dev(sl),
                       CovLaunch{S.dev(rec), S.dev(fr), S.dev(lmv), n_lm, S.dev(cov), S.dev(var), S.dev(st), S.dev(sig), S.dev(sxi)}));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0, t = 0; i < n; ++i) {
        pvio_b200_window_covariance &R = records[i];
        if (R.n_frames > 0) memcpy(R.cov, S.host(cov) + recs[i].cov_off, sizeof(double) * 225 * R.n_frames * R.n_frames);
        if (R.n_tracks > 0) memcpy(R.inv_depth_var, S.host(var) + t, sizeof(double) * R.n_tracks);
        t += R.n_tracks;
        R.status = S.host(st)[i];
    }
    return 0;
}

int pvio_b200_batch_window_landmarks(pvio_b200_handle hh, int n, pvio_b200_window_landmarks *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const char *what = "batch_window_landmarks";
    auto bad = [&](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); };
    if (n < 0 || (n > 0 && !records)) return bad("bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_landmarks: bad slot list"));
    // every record checked against its slot's host mirror before anything is staged; the all-tracks mode takes its rows
    // from the mirror's size, with no per-track work
    std::vector<BwLmk> recs(n);
    std::vector<int32_t> rows, cov_slots, cov_rec;
    std::vector<CovRec> crecs;
    int32_t n_pts = 0, n_cov_rows = 0, max_cov_rows = 0;
    int64_t sig_n = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_landmarks &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        const int T = (int)s.ids.size();
        if (s.N < 1) return bad("a window without frames");
        if (R.n_tracks < -1 || R.n_tracks > T) return bad("a track count out of range");
        const bool all = R.n_tracks == -1;
        const int nr = all ? T : R.n_tracks;
        if (all && R.capacity < T) return bad("capacity smaller than the slot's live tracks");
        if (!all && nr > 0 && !R.tracks) return bad("tracks missing");
        if (nr > 0 && !R.point) return bad("point missing");
        if (R.inv_depth_var && !R.point_cov) return bad("inv_depth_var without point_cov");
        const bool cov = R.point_cov != nullptr;
        if (cov && cov_smem_bytes(h->hdr.h[R.slot]) > 220 * 1024) return bad("reduced system too large for shared memory");
        BwLmk &L = recs[i];
        L = BwLmk{R.slot, nr, T, all ? -1 : (int32_t)rows.size(), n_pts, cov ? (int32_t)cov_slots.size() : -1, n_cov_rows, 0};
        if (!all) {
            std::vector<uint8_t> taken(T, 0);
            for (int k = 0; k < nr; ++k) {
                const int r = find_row(s, R.tracks[k]);
                if (r < 0) return bad("a track that is not live in its slot");
                if (taken[r]) return bad("a track named twice");
                taken[r] = 1;
                rows.push_back(r);
            }
        }
        n_pts += nr;
        if (cov) {
            const int64_t D = (s.inertial ? 15 : 6) * (int64_t)s.N;
            crecs.push_back(CovRec{R.slot, 0, 0, 0, 0, sig_n});
            cov_slots.push_back(R.slot);
            cov_rec.push_back(i);
            n_cov_rows += nr;
            max_cov_rows = std::max(max_cov_rows, nr);
            sig_n += D * D;
        }
    }
    const int n_cov = (int)cov_slots.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto rw = S.up(rows);
    const auto crc = S.up(cov_rec);
    const auto cr = S.up(crecs);
    const auto csl = S.up(cov_slots);
    const auto pts = S.add<double>(Stage::kDown, 3 * (size_t)n_pts);
    const auto rol = S.add<int32_t>(Stage::kDown, (size_t)n_pts);
    const auto pcov = S.add<double>(Stage::kDown, 9 * (size_t)n_cov_rows), var = S.add<double>(Stage::kDown, (size_t)n_cov_rows);
    const auto st = S.add<int32_t>(Stage::kDown, n_cov);
    const auto lmo = S.add<int32_t>(Stage::kScratch, (size_t)n_cov * h->Mcap);
    const auto sig = S.add<double>(Stage::kScratch, (size_t)sig_n);
    const auto sxi = S.add<double>(Stage::kScratch, (size_t)n_cov * h->Ncap * h->Ncap * 36);
    TRY(S.place(h, true));
    const LmkArgs L{S.dev(rec), S.dev(rw), S.dev(crc), S.dev(pts), S.dev(rol), S.dev(lmo), S.dev(st), S.dev(sxi), S.dev(pcov), S.dev(var)};
    const BwArgs a = launch_args<BwArgs>(h);
    bw_landmark_point_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L);
    ++h->launches;
    CK(h, cudaGetLastError());
    if (n_cov > 0) {
        TRY(run_cov_system(h, n_cov, cov_slots.data(), S.dev(csl),
                           CovLaunch{S.dev(cr), nullptr, nullptr, 0, nullptr, nullptr, S.dev(st), S.dev(sig), S.dev(sxi)}));
        const dim3 grid(n_cov, std::max(1, (max_cov_rows + kLmkWarps - 1) / kLmkWarps));
        if (h->hs_double) bw_landmark_cov_kernel<double><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        else bw_landmark_cov_kernel<float><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        ++h->launches;
        CK(h, cudaGetLastError());
    }
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_landmarks &R = records[i];
        const BwLmk &L = recs[i];
        const WinSlot &s = h->slots[R.slot];
        const size_t nr = L.n_rows;
        if (nr > 0) memcpy(R.point, S.host(pts) + 3 * (size_t)L.out_off, sizeof(double) * 3 * nr);
        if (R.role && nr > 0) memcpy(R.role, S.host(rol) + L.out_off, sizeof(int32_t) * nr);
        if (R.track_id && nr > 0) {
            if (L.rows_off < 0) memcpy(R.track_id, s.ids.data(), sizeof(int32_t) * nr);
            else memcpy(R.track_id, records[i].tracks, sizeof(int32_t) * nr);
        }
        R.status = PVIO_B200_OK;
        if (L.cov >= 0) {
            if (nr > 0) memcpy(R.point_cov, S.host(pcov) + 9 * (size_t)L.cov_off, sizeof(double) * 9 * nr);
            if (R.inv_depth_var && nr > 0) memcpy(R.inv_depth_var, S.host(var) + L.cov_off, sizeof(double) * nr);
            R.status = S.host(st)[L.cov];
        }
        R.n_rows = (int32_t)nr;
    }
    return 0;
}

int pvio_b200_batch_window_trajectory(pvio_b200_handle hh, int n, pvio_b200_window_trajectory *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const char *what = "batch_window_trajectory";
    auto bad = [&](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); };
    if (n < 0 || (n > 0 && !records)) return bad("bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_trajectory: bad slot list"));
    // every record checked before anything is staged
    std::vector<BwTraj> recs(n);
    std::vector<double> times;
    std::vector<int32_t> cov_slots, frames;
    std::vector<CovRec> crecs;
    int64_t rows = 0, cov_rows = 0, jcov_n = 0, sig_n = 0;
    int warps = 1;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_trajectory &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return bad("a visual-only slot");
        if (R.n_times < 0) return bad("a negative time count");
        if (R.n_times > 0 && (!R.times || !R.states || !R.frame)) return bad("times, states or frame missing");
        for (int q = 0; q < R.n_times; ++q) {
            if (!std::isfinite(R.times[q])) return bad("a time that is not finite");
            if (q > 0 && R.times[q] < R.times[q - 1]) return bad("times that decrease");
        }
        BwTraj &T = recs[i];
        T = BwTraj{};
        T.slot = R.slot; T.N = s.N; T.n_times = R.n_times; T.cov = -1; T.t_off = rows; T.scov_off = cov_rows;
        std::vector<int32_t> owners;
        for (int k = 0; k + 1 < s.N; ++k) {
            T.ns[k] = s.n_samples.empty() ? 0 : s.n_samples[k];
            if (T.ns[k] > 0) owners.push_back(k);
        }
        warps = std::max(warps, s.N - 1);
        if (R.state_cov && !owners.empty()) {        // Sigma_k of the frames that own a factor with samples
            if (cov_smem_bytes(h->hdr.h[R.slot]) > 220 * 1024) return bad("reduced system too large for shared memory");
            const int64_t K15 = 15 * (int64_t)owners.size(), D = 15 * (int64_t)s.N;
            T.cov = (int32_t)cov_slots.size(); T.cov_off = jcov_n;
            crecs.push_back(CovRec{R.slot, (int32_t)owners.size(), (int32_t)frames.size(), 0, jcov_n, sig_n});
            frames.insert(frames.end(), owners.begin(), owners.end());
            cov_slots.push_back(R.slot);
            jcov_n += K15 * K15;
            sig_n += D * D;
        }
        if (R.state_cov) {
            if (T.cov < 0) T.cov = -2;               // NaN rows only: no factor holds samples
            cov_rows += R.n_times;
        }
        times.insert(times.end(), R.times, R.times + R.n_times);
        rows += R.n_times;
    }
    const int n_cov = (int)cov_slots.size();
    const bool any_cov = cov_rows > 0;
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto tm = S.up(times);
    const auto cr = S.up(crecs);
    const auto fr = S.up(frames);
    const auto csl = S.up(cov_slots);
    const auto sto = S.add<double>(Stage::kDown, 16 * (size_t)rows);
    const auto fro = S.add<int32_t>(Stage::kDown, (size_t)rows);
    const auto sco = S.add<double>(Stage::kDown, 225 * (size_t)cov_rows);
    const auto st = S.add<int32_t>(Stage::kDown, n_cov);
    const auto jc = S.add<double>(Stage::kScratch, (size_t)jcov_n);
    const auto sig = S.add<double>(Stage::kScratch, (size_t)sig_n);
    const auto sxi = S.add<double>(Stage::kScratch, (size_t)n_cov * h->Ncap * h->Ncap * 36);
    TRY(S.place(h, true));
    if (n_cov > 0)
        TRY(run_cov_system(h, n_cov, cov_slots.data(), S.dev(csl),
                           CovLaunch{S.dev(cr), S.dev(fr), nullptr, 0, S.dev(jc), nullptr, S.dev(st), S.dev(sig), S.dev(sxi)}));
    const TrajArgs T{S.dev(rec), S.dev(tm), S.dev(sto), S.dev(fro), S.dev(sco), S.dev(jc), S.dev(st), any_cov ? 1 : 0};
    const size_t smem = warps * traj_warp_bytes(any_cov);
    if (smem > 48 * 1024)
        CK(h, cudaFuncSetAttribute(bw_trajectory_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bw_trajectory_kernel<<<n, 32 * warps, smem, h->stream>>>(launch_args<BwArgs>(h), T);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_trajectory &R = records[i];
        const BwTraj &T = recs[i];
        const size_t nq = R.n_times;
        if (nq > 0) {
            memcpy(R.states, S.host(sto) + 16 * (size_t)T.t_off, sizeof(double) * 16 * nq);
            memcpy(R.frame, S.host(fro) + T.t_off, sizeof(int32_t) * nq);
            if (R.state_cov) memcpy(R.state_cov, S.host(sco) + 225 * (size_t)T.scov_off, sizeof(double) * 225 * nq);
        }
        R.status = T.cov >= 0 ? S.host(st)[T.cov] : PVIO_B200_OK;
    }
    return 0;
}

int pvio_b200_batch_window_download(pvio_b200_handle hh, int n, const int32_t *slots, int32_t *n_frames, double *frames,
                                    int64_t frames_stride, int32_t *n_tracks, int64_t track_stride, int32_t *track_id,
                                    double *inv_depth, int32_t *anchor_frame, int32_t *n_observations, uint8_t *valid,
                                    double *quality) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_slots(h, n, slots, "batch_window_download: bad slot list"));
    if (n == 0) return 0;
    std::vector<BwDl> dls(n);
    int64_t off = 0;
    for (int i = 0; i < n; ++i) {
        const WinSlot &s = h->slots[slots[i]];
        const int T = (int)s.ids.size();
        if (frames && frames_stride < (int64_t)s.N * kFrameStride) return fail(h, PVIO_B200_EINVAL, "batch_window_download: frames_stride too small");
        if ((track_id || inv_depth || anchor_frame || n_observations || valid || quality) && track_stride < T)
            return fail(h, PVIO_B200_EINVAL, "batch_window_download: track_stride smaller than a slot's live tracks");
        dls[i] = BwDl{slots[i], s.N, T, 0, off};
        off += BwDlRec::bytes(s.N, T);
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto dl = S.up(dls);
    const auto out = S.add<uint8_t>(Stage::kDown, (size_t)off);
    TRY(S.place(h, true));
    bw_download_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(dl), S.dev(out));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        const int N = dls[i].N, T = dls[i].T;
        const BwDlRec o(S.host(out) + dls[i].off, N, T);
        const size_t t0 = (size_t)i * track_stride;
        if (n_frames) n_frames[i] = N;
        if (n_tracks) n_tracks[i] = T;
        if (frames) memcpy(frames + (size_t)i * frames_stride, o.fo, sizeof(double) * N * kFrameStride);
        if (track_id) memcpy(track_id + t0, o.io, sizeof(int32_t) * T);
        if (inv_depth) memcpy(inv_depth + t0, o.ro, sizeof(double) * T);
        if (anchor_frame) memcpy(anchor_frame + t0, o.ao, sizeof(int32_t) * T);
        if (n_observations) memcpy(n_observations + t0, o.no, sizeof(int32_t) * T);
        if (valid) memcpy(valid + t0, o.vo, T);
        if (quality) memcpy(quality + t0, o.qo, sizeof(double) * T);
    }
    return 0;
}

int pvio_b200_batch_window_localize(pvio_b200_handle hh, int n, pvio_b200_window_localize *records,
                                    const pvio_b200_options *opt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_localize: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_localize: bad slot list"));
    // every record is checked against its slot's host mirror before anything is staged
    LocPlan P;
    P.what = "batch_window_localize";
    for (int i = 0; i < n; ++i) TRY(loc_add(h, P, records[i], true));
    Stage S(h->bw.stage, &h->bw.scratch);
    const LocSecs s = loc_stage(S, P, true);
    TRY(S.place(h));
    const size_t w8 = sizeof(double);
    for (int i = 0; i < n; ++i) {
        memcpy(S.host(s.frames) + 16 * (size_t)i, records[i].state, w8 * 16);
        if (P.recs[i].inertial)
            memcpy(S.host(s.imu) + (size_t)P.recs[i].imu_off * kImuStride, records[i].imu_record, w8 * kImuStride);
    }
    TRY(S.upload(h));
    TRY(loc_launch(h, loc_args(S, s, opt), n));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev0, h->ev1);
    size_t k = 0;
    for (int i = 0; i < n; ++i) loc_results(S, s, P, i, k, records[i], ms);
    return 0;
}

int pvio_b200_batch_window_track_frame(pvio_b200_handle hh, int n, pvio_b200_window_track_frame *records,
                                       const pvio_b200_options *opt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_track_frame: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_track_frame: bad slot list"));
    // every record is checked before anything is staged: its localize half as localize checks it, then the rest
    LocPlan P;
    P.what = "batch_window_track_frame";
    std::vector<BwTrack> trs(n);
    std::vector<BwTrackJob> jobs;
    std::vector<int32_t> kf_row;
    std::vector<double> kf_z;
    size_t rows = 0, par = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_track_frame &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return loc_fail(h, P, "the window carries no motion states");
        TRY(loc_add(h, P, localize_view(R), false));
        if (!R.samples || !R.noise_cov || !R.imu_record || !R.keyframe || !R.skipped_frames) return loc_fail(h, P, "null array");
        if (R.n_samples < 1)
            return loc_fail(h, P, "a frame without IMU samples (integrate() returns false, preintegrator.cpp:86)");
        if (R.newest_is_keyframe != 0 && R.newest_is_keyframe != 1) return loc_fail(h, P, "newest_is_keyframe not 0 or 1");
        const bool merged = R.newest_is_keyframe == 0;
        if (merged && s.N < 2) return loc_fail(h, P, "a non-keyframe newest frame without a keyframe before it");
        if (merged && (R.n_merge < 1 || !R.merge_samples)) return loc_fail(h, P, "a non-keyframe newest frame without its samples");
        if (!merged && (R.n_merge != 0 || R.merge_samples)) return loc_fail(h, P, "a merge list with a keyframe newest frame");
        if (!all_finite(R.samples, 7 * (int64_t)R.n_samples) || (merged && !all_finite(R.merge_samples, 7 * (int64_t)R.n_merge)))
            return loc_fail(h, P, "non-finite sample");
        if (!std::isfinite(R.t_end) || !all_finite(R.noise_cov, 36) || !std::isfinite(R.cx) || !std::isfinite(R.cy))
            return loc_fail(h, P, "non-finite t_end, noise or principal point");
        if (*R.skipped_frames < 0) return loc_fail(h, P, "negative skipped_frames");
        BwTrack &t = trs[i];
        t = BwTrack{merged ? 1 : 0, merged ? s.N - 2 : s.N - 1, 0, (int32_t)kf_row.size(), merged ? 0 : 1, 0,
                    *R.skipped_frames, (int32_t)i * kImuAux, R.cx, R.cy};
        const uint32_t fi = 1u << t.frame_i;
        for (int k = 0; k < R.n_obs; ++k) {                    // loc_add found every track live and named once
            const int r = find_row(s, R.obs_track[k]);
            if (!(s.mask[r] & fi)) continue;
            kf_row.push_back(r);
            kf_z.insert(kf_z.end(), R.obs_z + 2 * k, R.obs_z + 2 * k + 2);
        }
        t.n_kf = (int32_t)kf_row.size() - t.kf_off;
        t.par_off = (int32_t)par;
        par += t.n_kf + (t.use_new ? R.n_new : 0);
        const size_t b = rows + (merged ? R.n_merge : 0), e = b + R.n_samples;
        if (e > (size_t)INT32_MAX || par > (size_t)INT32_MAX) return loc_fail(h, P, "too many samples or pairs in one call");
        jobs.push_back(BwTrackJob{i, (int32_t)b, (int32_t)e, 0});
        if (merged) jobs.push_back(BwTrackJob{i, (int32_t)rows, (int32_t)e, 1});
        rows = e;
    }
    // the localize sections without IMU records (the PnP reads the step-1 records, imu_off = record index); upload
    // track records | jobs | observed pairs' rows | their keypoints | merge_samples ++ samples | t_end and noise,
    // download the edit's IMU records | predicted states | keyframe words, scratch step-1 records | parallaxes
    const size_t w8 = sizeof(double), J = jobs.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    const LocSecs s = loc_stage(S, P, false);
    const auto tr = S.up(trs);
    const auto job = S.up(jobs);
    const auto kr = S.up(kf_row);
    const auto kz = S.up(kf_z), smp = S.add<double>(Stage::kUp, 7 * rows), aux = S.add<double>(Stage::kUp, (size_t)n * kImuAux);
    const auto rec_out = S.add<double>(Stage::kDown, (size_t)n * kImuStride), pred = S.add<double>(Stage::kDown, 16 * (size_t)n);
    const auto kfo = S.add<double>(Stage::kDown, 4 * (size_t)n);
    const auto rec1 = S.add<double>(Stage::kScratch, (size_t)n * kImuStride), pars = S.add<double>(Stage::kScratch, par);
    TRY(S.place(h));
    for (int i = 0; i < n; ++i) {
        double *a = S.host(aux) + (size_t)i * kImuAux;
        a[0] = records[i].t_end;
        memcpy(a + 1, records[i].noise_cov, w8 * 36);
    }
    for (const BwTrackJob &j : jobs) {                          // merge_samples ++ samples, back to back per record
        if (j.merged) continue;
        const pvio_b200_window_track_frame &R = records[j.rec];
        memcpy(S.host(smp) + 7 * (size_t)j.b, R.samples, w8 * 7 * R.n_samples);
        if (trs[j.rec].merged) memcpy(S.host(smp) + 7 * ((size_t)j.b - R.n_merge), R.merge_samples, w8 * 7 * R.n_merge);
    }
    TRY(S.upload(h));
    TrackArgs T;
    T.tr = S.dev(tr); T.job = S.dev(job); T.kf_row = S.dev(kr); T.kf_z = S.dev(kz); T.smp = S.dev(smp); T.aux = S.dev(aux);
    T.rec_out = S.dev(rec_out); T.pred = S.dev(pred); T.kfo = S.dev(kfo); T.rec1 = S.dev(rec1); T.par = S.dev(pars);
    T.n_jobs = (int)J;
    LocArgs L = loc_args(S, s, opt);
    L.imu = T.rec1;
    const BwArgs a = launch_args<BwArgs>(h);
    bw_track_integrate_kernel<<<(int)((J + kBwImuWarps - 1) / kBwImuWarps), 32 * kBwImuWarps, 0, h->stream>>>(a, L, T);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(loc_launch(h, L, n));
    bw_track_keyframe_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L, T);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, h->ev0, h->ev1);
    size_t k = 0;
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_track_frame &R = records[i];
        loc_results(S, s, P, i, k, localize_view(R), ms);
        memcpy(R.imu_record, S.host(rec_out) + (size_t)i * kImuStride, w8 * kImuStride);
        if (R.predicted) memcpy(R.predicted, S.host(pred) + 16 * (size_t)i, w8 * 16);
        const double *o = S.host(kfo) + 4 * (size_t)i;
        *R.keyframe = o[0] != 0.0 ? 1 : 0;
        if (R.parallax) *R.parallax = o[1];
        if (R.n_parallax) *R.n_parallax = (int32_t)o[2];
        *R.skipped_frames = (int32_t)o[3];
    }
    return 0;
}

int pvio_b200_batch_window_set_imu(pvio_b200_handle hh, int n, const pvio_b200_window_imu *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: bad record list");
    if (n == 0) return 0;
    // every record is checked before anything is staged
    std::vector<BwImu> recs(n);
    std::vector<std::pair<int32_t, int32_t>> pairs(n);
    size_t rows = 0;
    int smax = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_imu &R = records[i];
        if (R.slot < 0 || R.slot >= h->W || !h->slots[R.slot].resident)
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: slot out of range or not resident");
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: the window carries no motion states");
        if (R.frame < 1 || R.frame >= s.N) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: frame outside 1 .. N - 1");
        if (R.n_samples < 1)
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: a factor without IMU samples (integrate() returns false, preintegrator.cpp:86)");
        if (!R.samples || !R.noise_cov) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: null array");
        if (!all_finite(R.samples, 7 * (int64_t)R.n_samples)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: non-finite sample");
        if (!std::isfinite(R.t_end)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: non-finite t_end");
        if (!all_finite(R.noise_cov, 36)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: non-finite noise");
        recs[i] = BwImu{R.slot, R.frame - 1, R.n_samples, (int32_t)rows};
        pairs[i] = {R.slot, R.frame};
        rows += R.n_samples;
        smax = std::max(smax, R.n_samples);
    }
    std::sort(pairs.begin(), pairs.end());
    if (std::adjacent_find(pairs.begin(), pairs.end()) != pairs.end())
        return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: a (slot, frame) named twice");
    if (rows > (size_t)INT32_MAX) return fail(h, PVIO_B200_EINVAL, "batch_window_set_imu: too many samples in one call");
    TRY(ensure_imu_store(h, smax));
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto smp = S.add<double>(Stage::kUp, 7 * rows), aux = S.add<double>(Stage::kUp, (size_t)n * kImuAux);
    TRY(S.place(h));
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_imu &R = records[i];
        memcpy(S.host(smp) + 7 * (size_t)recs[i].off, R.samples, sizeof(double) * 7 * R.n_samples);
        double *a = S.host(aux) + (size_t)i * kImuAux;
        a[0] = R.t_end;
        memcpy(a + 1, R.noise_cov, sizeof(double) * 36);
    }
    TRY(S.upload(h));
    bw_set_imu_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rec), S.dev(smp), S.dev(aux));
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) h->slots[recs[i].slot].n_samples[recs[i].factor] = recs[i].n;
    return 0;
}

int pvio_b200_batch_window_imu_records(pvio_b200_handle hh, int n, const int32_t *slots, double *records,
                                       int64_t records_stride) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_slots(h, n, slots, "batch_window_imu_records: bad slot list"));
    if (n == 0) return 0;
    if (!records) return fail(h, PVIO_B200_EINVAL, "batch_window_imu_records: null array");
    std::vector<BwDl> dls(n);
    int64_t off = 0;
    for (int i = 0; i < n; ++i) {
        const WinSlot &s = h->slots[slots[i]];
        if (!s.inertial) return fail(h, PVIO_B200_EINVAL, "batch_window_imu_records: the window carries no motion states");
        const int64_t m = (int64_t)std::max(s.N - 1, 0) * kImuStride;
        if (records_stride < m) return fail(h, PVIO_B200_EINVAL, "batch_window_imu_records: records_stride smaller than a slot's records");
        dls[i] = BwDl{slots[i], std::max(s.N, 1), 0, 0, off};
        off += m * (int64_t)sizeof(double);
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto dl = S.up(dls);
    const auto out = S.add<uint8_t>(Stage::kDown, (size_t)off);
    TRY(S.place(h, true));
    bw_imu_records_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(dl), S.dev(out));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i)
        memcpy(records + i * records_stride, S.host(out) + dls[i].off, sizeof(double) * (size_t)(dls[i].N - 1) * kImuStride);
    return 0;
}

int pvio_b200_batch_window_set_keypoints(pvio_b200_handle hh, int n, const pvio_b200_window_keypoints *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_set_keypoints: bad slot list"));
    std::vector<BwKeys> ks(n);
    std::vector<int2> pairs;
    std::vector<int> kmax(n, -1);
    std::vector<uint32_t> gens(n, 0);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_keypoints &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (s.N < 1) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: a window without frames");
        if (R.tracker_slot < 0 || R.tracker_slot > kMaxBatchSlot)
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: tracker slot out of range");
        if (!R.frame_id) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: frame id 0");
        const KltBatchState &B = h->kltb;
        const SlotKeypoints *K = (size_t)R.tracker_slot < B.kps.size() ? &B.kps[R.tracker_slot] : nullptr;
        if (!K || !K->live || (R.frame_id != K->frame_id && R.frame_id != K->prev_frame_id))
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: the frame is not one of the tracker slot's two newest");
        gens[i] = K->gen;
        if (R.n < 0 || (R.n > 0 && (!R.track || !R.keypoint))) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: null array");
        if (R.newest_is_keyframe != 0 && R.newest_is_keyframe != 1)
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: newest_is_keyframe not 0 or 1");
        if (R.skipped_frames < 0) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: negative skipped_frames");
        ks[i] = BwKeys{R.slot, (int32_t)s.ids.size(), R.n, (int32_t)pairs.size()};
        const uint32_t newest = 1u << (s.N - 1);
        std::vector<uint8_t> named(s.ids.size(), 0);
        std::vector<int32_t> kps(R.keypoint, R.keypoint + R.n);
        for (int k = 0; k < R.n; ++k) {
            const int r = find_row(s, R.track[k]);
            if (r < 0) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: unknown or dead track");
            if (!(s.mask[r] & newest)) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: a track not observed in the newest frame");
            if (named[r]) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: a track named twice");
            named[r] = 1;
            if (R.keypoint[k] < 0) return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: negative keypoint index");
            pairs.push_back(make_int2(r, R.keypoint[k]));
            kmax[i] = std::max(kmax[i], (int)R.keypoint[k]);
        }
        std::sort(kps.begin(), kps.end());
        if (std::adjacent_find(kps.begin(), kps.end()) != kps.end())
            return fail(h, PVIO_B200_EINVAL, "batch_window_set_keypoints: a keypoint named twice");
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto k = S.up(ks);
    const auto p = S.up(pairs);
    TRY(S.place(h, true));
    bw_set_keypoints_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(k), S.dev(p));
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_keypoints &R = records[i];
        WinSlot &s = h->slots[R.slot];
        s.link = true; s.link_tracker = R.tracker_slot; s.link_frame = R.frame_id; s.link_kmax = kmax[i]; s.link_gen = gens[i];
        s.newest_kf = R.newest_is_keyframe; s.skipped = R.skipped_frames;
    }
    return 0;
}

// ------------------------------------------------------------------------ mirror_frame's stages
// A record's tracker slot as the mirror reads it: frame i (the slot's newest) and the new frame j with its prev_index.
// n_j bounds the new frame's keypoints when the staging is laid out (track_camera lays it out before they exist) and
// is their count when the mirror runs.
struct MirView { const double2 *zi, *zj; const int32_t *prev; int n_i, n_j; };

// One call of pvio_b200_batch_window_mirror_frame, or the mirror half of pvio_b200_batch_window_track_camera: the
// checked records, their staging and the device views of track_frame's kernels.  Both calls run add for every record,
// stage, then front, launch or their own split of it, check, append and commit.
struct MirCall {
    const char *what;
    std::vector<int32_t> slots;
    std::vector<BwMirror> mir;
    std::vector<BwLoc> locs;
    std::vector<BwTrack> trs;
    std::vector<BwEdit> eds;
    std::vector<BwTrackJob> jobs;             // per record its step-1 job, then its merged job (split: all step-1 first)
    std::vector<BwImu> kimu;                  // the factors that keep their samples, as set_imu stages them
    std::vector<double> kaux, gpt;
    std::vector<int32_t> grow;
    std::vector<WinSlot> next;                // the slots' windows after the call, but for their row counts
    std::vector<uint8_t> taken;
    size_t kp = 0, tab = 0, rm = 0, rows = 0;
    int smax = 0, n1 = 0;                     // n1: the step-1 jobs (split)
    bool cam = false;                         // staged for track_camera (stage)

    Stage S;
    Stage::Sec<BwMirror> mr;
    Stage::Sec<BwLoc> lo;
    Stage::Sec<BwTrack> tr;
    Stage::Sec<BwTrackJob> job;
    Stage::Sec<double> pq, smp, aux, gp, kax, frames, out, rec_out, pred, kfo, z, pts, nz, kf_z, rho, rho_next, par, rec1, xs;
    Stage::Sec<int32_t> gr, cnt, live, kpt, eout, tabs, rmap, lrow, cand, row, kf_row;
    Stage::Sec<BwEdit> ed;
    Stage::Sec<BwImu> kim;
    Stage::Sec<int2> cont;
    Stage::Sec<uint8_t> valid;
    Stage::Sec<PnpArgs> args;
    Stage::Sec<BwNew> nw;
    Stage::Sec<BwObs> ob;
    std::optional<Relayout> lay;
    LocArgs L;
    TrackArgs T;
    MirArgs M;

    MirCall(Handle *h, const char *w, int n)
        : what(w), mir(n), locs(n), trs(n), eds(n), next(n), S(h->bw.stage, &h->bw.scratch) {}
    int bad(Handle *h, const char *why) const { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); }

    // Record i checked against its slot's host mirror; tracker_why: the caller's verdict on the tracker slot (null:
    // usable), checked after the link.  Returns null or why the record is rejected.
    const char *add(Handle *h, int i, const pvio_b200_window_mirror &R, const MirView &v, const char *tracker_why,
                    bool split) {
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return "the window carries no motion states";
        if (s.N < 1) return "a window without frames";
        if (!s.link) return "the slot has no link to a tracker slot (set_keypoints)";
        if (R.tracker_slot != s.link_tracker) return "not the tracker slot of the slot's link";
        if (const char *why = take_slot(taken, R.tracker_slot, "a tracker slot named twice")) return why;
        if (tracker_why) return tracker_why;
        if (!R.samples || !R.noise_cov || !R.kp_track || !R.state || !R.keyframe) return "null array";
        if (R.max_keypoints < v.n_j) return "max_keypoints below the tracker's keypoint count";
        if (R.n_samples < 1) return "a frame without IMU samples (integrate() returns false, preintegrator.cpp:86)";
        if (R.keep_samples != 0 && R.keep_samples != 1) return "keep_samples not 0 or 1";
        if (!all_finite(R.samples, 7 * (int64_t)R.n_samples)) return "non-finite sample";
        if (!std::isfinite(R.t_end) || !all_finite(R.noise_cov, 36) || !std::isfinite(R.cx) || !std::isfinite(R.cy))
            return "non-finite t_end, noise or principal point";
        const bool merged = !s.newest_kf;
        if (merged && s.N < 2) return "a non-keyframe newest frame without a keyframe before it";
        if (merged && s.N - 1 < s.n_prior) return "the newest frame is covered by the prior";
        const int n_merge = merged ? s.n_samples[s.N - 2] : 0;
        if (merged && n_merge < 1) return "a non-keyframe newest frame whose factor holds no samples";
        if (!merged && s.N >= h->Ncap) return "window of more than max_frames frames";
        if (R.n_given < 0 || (R.n_given > 0 && (!R.given_track || !R.given_point))) return "null array";
        std::vector<std::pair<int, int>> given;
        std::vector<uint8_t> named(s.ids.size(), 0);
        for (int k = 0; k < R.n_given; ++k) {
            const int r = find_row(s, R.given_track[k]);
            if (r < 0) return "unknown or dead track";
            if (named[r]) return "a track named twice";
            named[r] = 1;
            if (!all_finite(R.given_point + 3 * k, 3)) return "non-finite given point";
            given.push_back({r, k});
        }
        std::sort(given.begin(), given.end());
        const int T = (int)s.ids.size(), fnew = merged ? s.N - 1 : s.N;
        const size_t first = rows;            // the call's sample rows: merge list ++ own samples per record
        slots.push_back(R.slot);
        mir[i] = BwMirror{v.zi, v.zj, v.prev, R.slot, T, v.n_i, v.n_j, (int32_t)tab, (int32_t)kp, (int32_t)grow.size(),
                          R.n_given, (int32_t)rm, (int32_t)first, n_merge, merged ? 1 : 0, s.N, s.next_id, 0, 0};
        for (const auto &g : given) {
            grow.push_back(g.first);
            gpt.insert(gpt.end(), R.given_point + 3 * g.second, R.given_point + 3 * g.second + 3);
        }
        locs[i] = BwLoc{R.slot, s.N - 1, 1, 0, (int32_t)kp, i, 0, (int32_t)kp};
        trs[i] = BwTrack{merged ? 1 : 0, merged ? s.N - 2 : s.N - 1, 0, (int32_t)kp, merged ? 0 : 1, (int32_t)kp,
                         s.skipped, (int32_t)i * kImuAux, R.cx, R.cy};
        eds[i] = BwEdit{R.slot, s.N, T, merged ? 1 : 0, 0, 0, fnew, 1, i * kMirX, 0, (int32_t)kp, 0, (int32_t)kp,
                        (int32_t)(kp + i)};
        const size_t b = first + n_merge, e = b + R.n_samples;
        if (split) {
            jobs.insert(jobs.begin() + n1++, BwTrackJob{i, (int32_t)b, (int32_t)e, 0});
        } else {
            jobs.push_back(BwTrackJob{i, (int32_t)b, (int32_t)e, 0});
        }
        if (merged) jobs.push_back(BwTrackJob{i, (int32_t)first, (int32_t)e, 1});
        rows = e;
        const int n_list = n_merge + R.n_samples;
        if (R.keep_samples) {
            kimu.push_back(BwImu{R.slot, fnew - 1, n_list, (int32_t)first});
            kaux.push_back(R.t_end);
            kaux.insert(kaux.end(), R.noise_cov, R.noise_cov + 36);
            smax = std::max(smax, n_list);
        }
        next[i] = mirror_next(s, {}, 0, R.keep_samples ? n_list : 0);
        kp += v.n_j; tab += 2 * (size_t)v.n_i; rm += T;
        if (rows > (size_t)INT32_MAX || kp + mir.size() > (size_t)INT32_MAX || tab > (size_t)INT32_MAX)
            return "too many samples or keypoints in one call";
        return nullptr;
    }

    // staging: upload records | track_frame's records, jobs, samples, t_end and noise | given points | edit records |
    // kept factors | re-layout; download counts | continued rows (the capacity check), then the results; device only
    // the mirror's tables and lists, the localize sections, the edit's lists.  camera (track_camera): the continued rows
    // are the section right after the counts, so that one copy brings both back (they then come back with the results
    // too), and the delta_key_q of every record comes back; otherwise they are the last section, after the results'
    // range, downloaded on their own (mirror_frame).  Uploads everything.
    int stage(Handle *h, const pvio_b200_window_mirror *records, const pvio_b200_options *opt, bool camera) {
        const int n = (int)mir.size();
        if (!kimu.empty()) TRY(ensure_imu_store(h, smax));   // the kept lists' room, before anything is staged
        const size_t w8 = sizeof(double);
        mr = S.up(mir);
        lo = S.up(locs);
        tr = S.up(trs);
        job = S.up(jobs);
        smp = S.add<double>(Stage::kUp, 7 * rows); aux = S.add<double>(Stage::kUp, (size_t)n * kImuAux);
        gr = S.up(grow);
        gp = S.up(gpt);
        ed = S.up(eds);
        kim = S.up(kimu);
        kax = S.up(kaux);
        lay.emplace(S, slots.data(), next);
        cam = camera;
        cnt = S.add<int32_t>(Stage::kDown, 4 * (size_t)n);
        if (camera) cont = S.add<int2>(Stage::kDown, kp);
        live = S.add<int32_t>(Stage::kDown, n);
        frames = S.add<double>(Stage::kDown, 16 * (size_t)n); out = S.add<double>(Stage::kDown, 8 * (size_t)n);
        rec_out = S.add<double>(Stage::kDown, (size_t)n * kImuStride); pred = S.add<double>(Stage::kDown, 16 * (size_t)n);
        kfo = S.add<double>(Stage::kDown, 4 * (size_t)n);
        kpt = S.add<int32_t>(Stage::kDown, kp);
        if (camera) pq = S.add<double>(Stage::kDown, 4 * (size_t)n);
        else cont = S.add<int2>(Stage::kDown, kp);
        eout = S.add<int32_t>(Stage::kScratch, kp + n);
        tabs = S.add<int32_t>(Stage::kScratch, tab); rmap = S.add<int32_t>(Stage::kScratch, rm);
        lrow = S.add<int32_t>(Stage::kScratch, kp); cand = S.add<int32_t>(Stage::kScratch, kp);
        row = S.add<int32_t>(Stage::kScratch, kp); kf_row = S.add<int32_t>(Stage::kScratch, kp);
        z = S.add<double>(Stage::kScratch, 2 * kp); pts = S.add<double>(Stage::kScratch, 3 * kp);
        nz = S.add<double>(Stage::kScratch, 4 * kp); kf_z = S.add<double>(Stage::kScratch, 2 * kp);
        rho = S.add<double>(Stage::kScratch, kp); rho_next = S.add<double>(Stage::kScratch, kp);
        valid = S.add<uint8_t>(Stage::kScratch, kp);
        par = S.add<double>(Stage::kScratch, kp); rec1 = S.add<double>(Stage::kScratch, (size_t)n * kImuStride);
        args = S.add<PnpArgs>(Stage::kScratch, n);
        nw = S.add<BwNew>(Stage::kScratch, kp);
        ob = S.add<BwObs>(Stage::kScratch, kp);
        xs = S.add<double>(Stage::kScratch, (size_t)n * kMirX);
        S.pow2 = camera;                      // laid out for output bounds that change from frame to frame
        TRY(S.place(h));
        for (int i = 0; i < n; ++i) {
            const pvio_b200_window_mirror &R = records[i];
            memcpy(S.host(smp) + 7 * ((size_t)mir[i].merge_row + mir[i].n_merge), R.samples, w8 * 7 * R.n_samples);
            double *a = S.host(aux) + (size_t)i * kImuAux;
            a[0] = R.t_end;
            memcpy(a + 1, R.noise_cov, w8 * 36);
        }
        TRY(S.upload(h));
        const SolveOptions so = solve_options(opt);
        L.rec = S.dev(lo); L.row = S.dev(row); L.z = S.dev(z); L.imu = S.dev(rec1); L.nz = S.dev(nz);
        L.frames = S.dev(frames); L.pts = S.dev(pts); L.out = S.dev(out); L.rho = S.dev(rho); L.rho_next = S.dev(rho_next);
        L.valid = S.dev(valid); L.args = S.dev(args); L.max_iter = so.max_iter; L.radius0 = so.radius0;
        T.tr = S.dev(tr); T.job = S.dev(job); T.kf_row = S.dev(kf_row); T.kf_z = S.dev(kf_z); T.smp = S.dev(smp);
        T.aux = S.dev(aux); T.rec_out = S.dev(rec_out); T.pred = S.dev(pred); T.kfo = S.dev(kfo); T.rec1 = S.dev(rec1);
        T.par = S.dev(par); T.n_jobs = (int)jobs.size();
        M.rec = S.dev(mr); M.loc = S.dev(lo); M.tr = S.dev(tr); M.tab = S.dev(tabs); M.grow = S.dev(gr); M.gpt = S.dev(gp);
        M.row = S.dev(row); M.z = S.dev(z); M.pts = S.dev(pts); M.nz = S.dev(nz); M.kf_row = S.dev(kf_row);
        M.kf_z = S.dev(kf_z); M.smp = S.dev(smp); M.cont = S.dev(cont); M.cand = S.dev(cand); M.rmap = S.dev(rmap);
        M.lrow = S.dev(lrow); M.kp = S.dev(kpt); M.cnt = S.dev(cnt); M.ed = S.dev(ed); M.nw = S.dev(nw); M.ob = S.dev(ob);
        M.x = S.dev(xs); M.lay = S.dev(lay->lay); M.eout = S.dev(eout); M.live = S.dev(live);
        return 0;
    }

    // bw_track_integrate_kernel on jobs [j0, j0 + nj); at least one CTA, so that the launches do not depend on the jobs
    int integrate(Handle *h, int j0, int nj) {
        TrackArgs t = T;
        t.job = T.job + j0;
        t.n_jobs = nj;
        bw_track_integrate_kernel<<<std::max((nj + kBwImuWarps - 1) / kBwImuWarps, 1), 32 * kBwImuWarps, 0, h->stream>>>(
            launch_args<BwArgs>(h), L, t);
        ++h->launches;
        CK(h, cudaGetLastError());
        return 0;
    }

    // mirror, then track_frame's kernels on its lists; integrate_jobs: the integrate launch's jobs from j0
    int launch(Handle *h, int j0) {
        const int n = (int)mir.size();
        const BwArgs a = launch_args<BwArgs>(h);
        bw_mirror_kernel<<<n, kBwThreads, 0, h->stream>>>(a, M);
        ++h->launches;
        CK(h, cudaGetLastError());
        TRY(integrate(h, j0, (int)jobs.size() - j0));
        TRY(loc_launch(h, L, n));
        bw_track_keyframe_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L, T);
        ++h->launches;
        CK(h, cudaGetLastError());
        return 0;
    }

    // the counts and continued rows down, a synchronisation, and the capacity: the windows as they would be if every
    // candidate turned out valid
    int check(Handle *h, bool camera) {
        const int n = (int)mir.size();
        if (camera) {
            TRY(S.download(h, cnt, cont));
        } else {
            TRY(S.download(h, cnt, cnt));
            TRY(S.download(h, cont, cont));
        }
        CK(h, cudaStreamSynchronize(h->stream));
        std::vector<WinSlot> most(n);
        for (int i = 0; i < n; ++i) {
            const int32_t *c = S.host(cnt) + 4 * (size_t)i;
            const int2 *cr = S.host(cont) + mir[i].kp_off;
            std::vector<int> rws(c[0]);
            for (int k = 0; k < c[0]; ++k) rws[k] = cr[k].x;
            most[i] = mirror_next(h->slots[slots[i]], rws, c[2], 0);
            TRY(check_window(h, most[i]));
        }
        return ensure_plane_tables(h, most);  // observations of plane tracks may outgrow the plane tables
    }

    // append: the edit, the re-layout, the kept samples, the link; the results down and a synchronisation
    int append(Handle *h) {
        const int n = (int)mir.size();
        const BwArgs a = launch_args<BwArgs>(h);
        bw_mirror_append_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L, T, M);
        ++h->launches;
        CK(h, cudaGetLastError());
        bw_edit_kernel<<<n, kBwThreads, 0, h->stream>>>(a, S.dev(ed), nullptr, S.dev(nw), S.dev(ob), S.dev(xs), S.dev(eout));
        ++h->launches;
        CK(h, cudaGetLastError());
        TRY(lay->launch(h, S, false));
        if (!kimu.empty()) {
            bw_set_imu_kernel<<<(int)kimu.size(), kBwThreads, 0, h->stream>>>(a, S.dev(kim), S.dev(smp), S.dev(kax));
            ++h->launches;
            CK(h, cudaGetLastError());
        }
        bw_mirror_link_kernel<<<n, kBwThreads, 0, h->stream>>>(a, M);
        ++h->launches;
        CK(h, cudaGetLastError());
        TRY(cam ? S.download(h) : S.download(h, cnt, kpt));
        CK(h, cudaStreamSynchronize(h->stream));
        return 0;
    }

    // the host mirrors from kp_track (continued tracks hold ids below the slot's next id, new tracks the next ids) with
    // the link to each tracker slot's new frame, committed; then the outputs
    int commit_out(Handle *h, pvio_b200_window_mirror *records, const uint64_t *frame_id, const uint32_t *gen) {
        const int n = (int)mir.size();
        const size_t w8 = sizeof(double);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, h->ev0, h->ev1);
        for (int i = 0; i < n; ++i) {
            const pvio_b200_window_mirror &R = records[i];
            const WinSlot &s = h->slots[slots[i]];
            const int32_t *k = S.host(kpt) + mir[i].kp_off;
            std::vector<int> rws;
            int n_new = 0, kmax = -1;
            for (int j = 0; j < mir[i].n_j; ++j) {
                if (k[j] < 0) continue;
                kmax = j;
                if (k[j] < s.next_id) rws.push_back(find_row(s, k[j])); else ++n_new;
            }
            const double *o = S.host(kfo) + 4 * (size_t)i;
            next[i] = mirror_next(s, rws, n_new, R.keep_samples ? mir[i].n_merge + R.n_samples : 0);
            next[i].link_frame = frame_id[i]; next[i].link_kmax = kmax; next[i].link_gen = gen[i];
            next[i].newest_kf = o[0] != 0.0 ? 1 : 0; next[i].skipped = (int)o[3];
        }
        commit(h, slots.data(), next);
        for (int i = 0; i < n; ++i) {
            const pvio_b200_window_mirror &R = records[i];
            if (S.host(live)[i] != (int32_t)h->slots[slots[i]].ids.size())
                return fail(h, PVIO_B200_ECUDA, (std::string(what) + ": the device track table disagrees with the host's").c_str());
            memcpy(R.kp_track, S.host(kpt) + mir[i].kp_off, sizeof(int32_t) * mir[i].n_j);
            if (R.counts) memcpy(R.counts, S.host(cnt) + 4 * (size_t)i, sizeof(int32_t) * 4);
            memcpy(R.state, S.host(frames) + 16 * (size_t)i, w8 * 16);
            if (R.predicted) memcpy(R.predicted, S.host(pred) + 16 * (size_t)i, w8 * 16);
            if (R.imu_record) memcpy(R.imu_record, S.host(rec_out) + (size_t)i * kImuStride, w8 * kImuStride);
            const double *o = S.host(kfo) + 4 * (size_t)i;
            *R.keyframe = o[0] != 0.0 ? 1 : 0;
            if (R.parallax) *R.parallax = o[1];
            if (R.n_parallax) *R.n_parallax = (int32_t)o[2];
            if (R.skipped_frames) *R.skipped_frames = (int32_t)o[3];
            if (R.summary) {
                const double *b = S.host(out) + 8 * (size_t)i;
                pvio_b200_summary &sm = *R.summary;
                memset(&sm, 0, sizeof(sm));
                sm.iterations = (int)b[0]; sm.accepted_steps = (int)b[1]; sm.termination = (int)b[2]; sm.usable = (int)b[3];
                sm.initial_cost = b[4]; sm.final_cost = b[5]; sm.final_radius = b[6]; sm.final_mu = b[7];
                sm.solve_seconds = ms * 1e-3;
            }
        }
        return 0;
    }
};

int pvio_b200_batch_window_mirror_frame(pvio_b200_handle hh, int n, pvio_b200_window_mirror *records,
                                        const pvio_b200_options *opt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_mirror_frame: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_mirror_frame: bad slot list"));
    // every record is checked against its slot's host mirror and its tracker slot before anything is staged
    const KltBatchState &B = h->kltb;
    MirCall C(h, "batch_window_mirror_frame", n);
    std::vector<uint64_t> fid(n);
    std::vector<uint32_t> gen(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_mirror &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        const SlotKeypoints *K = R.tracker_slot >= 0 && (size_t)R.tracker_slot < B.kps.size() ? &B.kps[R.tracker_slot] : nullptr;
        const bool ok = K && K->live && K->gen == s.link_gen && K->prev_frame_id != 0 && K->prev_frame_id == s.link_frame &&
                        s.link_kmax < K->prev_n;
        MirView v{};
        if (ok) v = MirView{K->z(1 - K->cur), K->z(K->cur), K->prev(K->cur), K->prev_n, K->n};
        if (const char *why = C.add(h, i, R, v, ok ? nullptr : "the tracker slot's previous frame is not the slot's newest frame",
                                    false))
            return C.bad(h, why);
        fid[i] = K->frame_id; gen[i] = K->gen;
    }
    TRY(C.stage(h, records, opt, false));
    TRY(C.launch(h, 0));
    TRY(C.check(h, false));
    TRY(C.append(h));
    return C.commit_out(h, records, fid.data(), gen.data());
}

int pvio_b200_batch_window_track_camera(pvio_b200_handle hh, int n, pvio_b200_window_camera *records, int max_level,
                                        int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                                        int border, double ransac_threshold, double ransac_confidence,
                                        double keypoint_distance, const pvio_b200_options *opt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_track_camera: bad record list");
    if (n == 0) return 0;
    std::vector<int32_t> slots(n);
    for (int i = 0; i < n; ++i) slots[i] = records[i].slot;
    TRY(check_slots(h, n, slots.data(), "batch_window_track_camera: bad slot list"));
    // every record is checked, as feature_track and as mirror_frame (against the tracker slot before it advances), before
    // anything is staged
    const KltBatchOptions ko{max_level, max_iter, eps, clahe_clip, tiles_x, tiles_y, border, ransac_threshold,
                             ransac_confidence};
    std::vector<pvio_b200_feature_frame> ff(n);
    std::vector<pvio_b200_window_mirror> mr(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_camera &R = records[i];
        ff[i] = pvio_b200_feature_frame{R.tracker_slot, R.width, R.height, R.stride, R.frame_id, R.image, R.fx, R.fy,
                                        R.cx, R.cy, R.map_frames, R.max_keypoints, nullptr, R.keypoints, R.prev_index,
                                        R.n_keypoints, R.feature_counts, R.info};
        mr[i] = pvio_b200_window_mirror{R.slot, R.tracker_slot, R.n_samples, R.keep_samples, R.samples, R.t_end,
                                        R.noise_cov, R.cx, R.cy, R.n_given, R.given_track, R.given_point,
                                        R.max_keypoints, R.kp_track, R.counts, R.state, R.predicted, R.imu_record,
                                        R.keyframe, R.parallax, R.n_parallax, R.skipped_frames, R.summary};
    }
    MirCall C(h, "batch_window_track_camera", n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_camera &R = records[i];
        if (!h->slots[R.slot].inertial) return C.bad(h, "the window carries no motion states");
        if (R.map_frames == 0) return C.bad(h, "map_frames 0 (a sequence start goes through batch_feature_track)");
        if (!R.n_keypoints) return C.bad(h, "null array");
        if (R.fx != h->cst.h[R.slot].fx || R.fy != h->cst.h[R.slot].fy) return C.bad(h, "fx, fy not the slot's");
    }
    FtRun run;
    run.staged = true;
    TRY(ft_check(h, n, ff.data(), ko, keypoint_distance, false, run));
    const KltBatchState &B = h->kltb;
    std::vector<uint64_t> fid(n);
    std::vector<uint32_t> gen(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_camera &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        const SlotKeypoints &K = B.kps[R.tracker_slot];     // ft_check found it live with its newest frame cached
        const bool ok = K.gen == s.link_gen && K.frame_id == s.link_frame && s.link_kmax < K.n;
        const MirView v{K.z(K.cur), nullptr, nullptr, K.n, run.out_cap[i]};
        if (const char *why = C.add(h, i, mr[i], v, ok ? nullptr : "the tracker slot's newest frame is not the slot's newest frame",
                                    true))
            return C.bad(h, why);
        fid[i] = R.frame_id; gen[i] = K.gen;
    }

    // the mirror's staging, laid out for every new frame's output bound and uploaded; the step-1 integration and
    // prediction from each slot's newest frame; the feature stages with delta_key_q composed from it on the device
    TRY(C.stage(h, mr.data(), opt, true));
    TRY(C.integrate(h, 0, C.n1));
    static_assert(offsetof(BwLoc, slot) == 0 && sizeof(BwLoc) % sizeof(int32_t) == 0,
                  "ft_predict_kernel reads each record's window slot from the staged BwLoc records");
    const FtPredict pred{C.S.dev(C.rec1), launch_args<BwArgs>(h).cst, &C.S.dev(C.lo)->slot,
                         (int)(sizeof(BwLoc) / sizeof(int32_t)), C.S.dev(C.pq)};
    TRY(ft_run(h, n, ff.data(), ko, keypoint_distance, &pred, run));
    for (int i = 0; i < n; ++i)
        if (run.count[i] > run.out_cap[i]) return C.bad(h, "more keypoints than the stated bound");

    // the new frames into the mirror's records; mirror, track_frame's kernels, the capacity check, the append; then the
    // tracker slots and the window slots commit
    for (int i = 0; i < n; ++i) {
        const SlotKeypoints &K = B.kps[records[i].tracker_slot];
        BwMirror &m = C.S.host(C.mr)[i];
        m.zj = K.z(2); m.prev = K.prev(2); m.n_j = run.count[i];
        C.mir[i] = m;
    }
    TRY(C.S.upload(h, C.mr));
    TRY(C.launch(h, C.n1));
    TRY(C.check(h, true));
    TRY(C.append(h));
    TRY(ft_finish(h, n, ff.data(), run));
    for (int i = 0; i < n; ++i)
        if (records[i].predict_q) memcpy(records[i].predict_q, C.S.host(C.pq) + 4 * (size_t)i, sizeof(double) * 4);
    return C.commit_out(h, mr.data(), fid.data(), gen.data());
}

int pvio_b200_batch_window_save(pvio_b200_handle hh, int n, pvio_b200_window_snapshot *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_save: bad record list");
    if (n == 0) return 0;
    auto bad = [h](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string("batch_window_save: ") + why).c_str()); };
    // every record is checked and sized from the host mirrors before anything is staged
    const KltBatchState &B = h->kltb;
    std::vector<SnapHead> heads(n);
    std::vector<SnapOff> offs(n);
    std::vector<SnapRec> recs;
    std::vector<SnapFac> facs;
    std::vector<int> packed;                  // the records with data, in call order
    std::vector<uint8_t> wseen(h->W, 0), tseen;
    int64_t area = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        if (R.slot < -1 || R.slot >= h->W || R.tracker_slot < -1 || R.tracker_slot > kMaxBatchSlot)
            return bad("slot or tracker slot out of range");
        if (R.slot < 0 && R.tracker_slot < 0) return bad("a record names neither a slot nor a tracker slot");
        const SlotKeypoints *K = nullptr;
        if (R.slot >= 0) {
            if (!h->slots[R.slot].resident) return bad("slot not resident");
            if (wseen[R.slot]) return bad("a slot named twice");
            wseen[R.slot] = 1;
        }
        if (R.tracker_slot >= 0) {
            K = (size_t)R.tracker_slot < B.kps.size() ? &B.kps[R.tracker_slot] : nullptr;
            if (!K || !K->live) return bad("tracker slot not live");
            if ((size_t)R.tracker_slot >= tseen.size()) tseen.resize(R.tracker_slot + 1, 0);
            if (tseen[R.tracker_slot]) return bad("a tracker slot named twice");
            tseen[R.tracker_slot] = 1;
        }
        if (R.capacity < 0) return bad("negative capacity");
        SnapHead &H = heads[i];
        memset(&H, 0, sizeof(H));
        H.magic = PVIO_B200_SNAPSHOT_MAGIC; H.version = PVIO_B200_SNAPSHOT_VERSION;
        H.parts = (R.slot >= 0 ? kSnapWindow : 0) | (K ? kSnapTracker : 0);
        int n_fac = 0, rows = 0;
        if (R.slot >= 0) {
            const WinSlot &s = h->slots[R.slot];
            H.N = s.N; H.T = (int32_t)s.ids.size(); H.fixed = s.fixed; H.next_id = s.next_id; H.n_prior = s.n_prior;
            H.inertial = s.inertial; H.n_planes = s.n_planes; H.newest_kf = s.newest_kf; H.skipped = s.skipped;
            // the link, when it names the record's tracker slot, its current sequence and one of its two held
            // frames, with every row's keypoint index inside that frame's keypoints (otherwise: saved unlinked)
            const int held = !K || !s.link_frame ? -1 : s.link_frame == K->frame_id ? K->n
                                                     : s.link_frame == K->prev_frame_id ? K->prev_n : -1;
            H.linked = K && s.link && s.link_tracker == R.tracker_slot && s.link_gen == K->gen && s.link_kmax < held ? 1 : 0;
            H.link_frame = H.linked ? s.link_frame : 0;
            for (int k = 0; k < snap_factors(H); ++k)
                if (s.n_samples[k] > 0) { ++n_fac; rows += s.n_samples[k]; }
        }
        int pk = -1;
        if (K) {
            H.n[0] = K->n; H.n[1] = K->prev_n; H.frame_no = K->frame_no;
            H.frame_id = K->frame_id; H.prev_frame_id = K->prev_frame_id;
            H.K[0] = K->fx; H.K[1] = K->fy; H.K[2] = K->cx; H.K[3] = K->cy;
            pk = snap_pyramid(B, R.tracker_slot);
            if (pk >= 0) {
                const KltPyramids &c = B.slots[R.tracker_slot];
                H.w = c.w; H.h = c.h; H.levels = c.levels; H.clahe = c.pyr_clahe[pk];
            }
        }
        offs[i] = snap_layout(H, n_fac, rows);
        H.size = offs[i].size;
        if (!R.data) continue;
        if (R.capacity < H.size) return bad("capacity below the record's size");
        SnapRec r = snap_rec(H, offs[i], R.slot, area - offs[i].dev0, (int)facs.size(), n_fac, rows);
        r.link = H.linked;
        if (R.slot >= 0) {
            const WinSlot &s = h->slots[R.slot];
            int64_t at = offs[i].smp;
            for (int k = 0; k < snap_factors(H); ++k)
                if (s.n_samples[k] > 0) { facs.push_back(SnapFac{k, s.n_samples[k], at}); at += 56 * (int64_t)s.n_samples[k]; }
        }
        if (K) snap_tracker(r, *K, pk >= 0 ? &B.slots[R.tracker_slot] : nullptr, pk);
        recs.push_back(r);
        packed.push_back(i);
        area += H.size - offs[i].dev0;
    }
    if (!recs.empty()) {
        Stage S(h->bw.stage, &h->bw.scratch);
        const auto rc = S.up(recs);
        const auto fc = S.up(facs);
        const auto out = S.add<uint8_t>(Stage::kDown, (size_t)area);
        TRY(S.place(h, true));
        bw_save_kernel<<<(int)recs.size(), kSnapThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(fc), S.dev(out));
        ++h->launches;
        CK(h, cudaGetLastError());
        TRY(S.download(h));
        CK(h, cudaStreamSynchronize(h->stream));
        for (size_t j = 0; j < packed.size(); ++j) {
            const int i = packed[j];
            const pvio_b200_window_snapshot &R = records[i];
            const SnapHead &H = heads[i];
            const SnapOff &o = offs[i];
            memset(R.data, 0, o.dev0);
            memcpy(R.data, &H, sizeof(H));
            if (R.slot >= 0) {
                const WinSlot &s = h->slots[R.slot];
                memcpy(R.data + o.ids, s.ids.data(), 4 * (size_t)H.T);
                memcpy(R.data + o.mask, s.mask.data(), 4 * (size_t)H.T);
                memcpy(R.data + o.role, s.role.data(), H.T);
                memcpy(R.data + o.nsmp, s.n_samples.data(), 4 * (size_t)snap_factors(H));
            }
            memcpy(R.data + o.dev0, S.host(out) + recs[j].base + o.dev0, H.size - o.dev0);
        }
    }
    for (int i = 0; i < n; ++i) records[i].size = heads[i].size;
    return 0;
}

int pvio_b200_batch_window_restore(pvio_b200_handle hh, int n, const pvio_b200_window_snapshot *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 0 || (n > 0 && !records)) return fail(h, PVIO_B200_EINVAL, "batch_window_restore: bad record list");
    if (n == 0) return 0;
    auto bad = [h](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string("batch_window_restore: ") + why).c_str()); };
    // every blob is checked completely before anything is staged
    std::vector<SnapHead> heads(n);
    std::vector<SnapOff> offs(n);
    std::vector<std::vector<int32_t>> nsmp(n);
    std::vector<int32_t> wslots;              // the window records' slots and their windows after the call
    std::vector<WinSlot> next;
    std::vector<uint8_t> wseen(h->W, 0), tseen;
    int smax = 0;
    bool inertial = false;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        if (R.slot < -1 || R.slot >= h->W || R.tracker_slot < -1 || R.tracker_slot > kMaxBatchSlot)
            return bad("slot or tracker slot out of range");
        if (R.slot < 0 && R.tracker_slot < 0) return bad("a record names neither a slot nor a tracker slot");
        if (R.slot >= 0) {
            if (wseen[R.slot]) return bad("a slot named twice");
            wseen[R.slot] = 1;
        }
        if (R.tracker_slot >= 0) {
            if ((size_t)R.tracker_slot >= tseen.size()) tseen.resize(R.tracker_slot + 1, 0);
            if (tseen[R.tracker_slot]) return bad("a tracker slot named twice");
            tseen[R.tracker_slot] = 1;
        }
        if (!R.data || R.capacity < (int64_t)sizeof(SnapHead)) return bad("a blob shorter than its head");
        SnapHead &H = heads[i];
        memcpy(&H, R.data, sizeof(H));
        if (H.magic != PVIO_B200_SNAPSHOT_MAGIC || H.version != PVIO_B200_SNAPSHOT_VERSION) return bad("not a blob of this version");
        if (H.size != R.capacity) return bad("the declared size is not the byte count");
        if (H.parts < 1 || H.parts > 3) return bad("bad parts");
        const bool win = H.parts & kSnapWindow, trk = H.parts & kSnapTracker;
        if ((R.slot >= 0 && !win) || (R.tracker_slot >= 0 && !trk)) return bad("the record names a part the blob lacks");
        // counts, before the layout is computed from them
        if (win) {
            if (H.N < 0 || H.N > kMaxFrames || H.T < 0 || H.T > 65536 || H.n_planes < 0 || H.n_planes > h->Pcap ||
                H.n_prior < 0 || H.n_prior > H.N)
                return bad("window counts out of range");
            if ((H.inertial != 0 && H.inertial != 1) || (H.n_prior > 0 && !H.inertial)) return bad("a prior on a visual-only window");
            if ((H.newest_kf != 0 && H.newest_kf != 1) || H.skipped < 0 || H.next_id < 0 || (H.linked != 0 && H.linked != 1))
                return bad("bad keyframe flag, skipped-frame counter, next id or link flag");
            if (H.fixed < 0 || (H.fixed >> H.N) != 0) return bad("a fixed frame outside the window");
        }
        if (trk) {
            if (H.n[0] < 0 || H.n[1] < 0 || !H.frame_id || (!H.prev_frame_id && H.n[1] > 0))
                return bad("bad tracker counts or frame ids");
            if (!(H.K[0] != 0.0 && H.K[1] != 0.0) || !all_finite(H.K, 4)) return bad("bad K");
            if (H.levels != 0 &&
                (H.levels < 1 || H.levels > kMaxLevels || H.w < kKltMinFrame || H.h < kKltMinFrame || H.w > 32768 ||
                 H.h > 32768 || klt_levels(H.w, H.h, H.levels - 1) != H.levels || !std::isfinite(H.clahe) || H.clahe < 0.0))
                return bad("a pyramid shape the tracker does not build");
        }
        if (win && H.linked && (!trk || !H.link_frame || (H.link_frame != H.frame_id && H.link_frame != H.prev_frame_id)))
            return bad("a link to a frame the blob's tracker part does not hold");
        const int F = snap_factors(H);
        SnapOff o = snap_layout(H, 0, 0);
        if (R.capacity < o.dev0) return bad("the declared size is not the byte count");
        nsmp[i].resize(F);
        memcpy(nsmp[i].data(), R.data + o.nsmp, 4 * (size_t)F);
        int64_t rows = 0;
        int n_fac = 0, fmax = 0;
        for (int32_t c : nsmp[i]) {
            if (c < 0) return bad("a negative sample count");
            rows += c; n_fac += c > 0; fmax = std::max(fmax, (int)c);
        }
        if (rows > INT32_MAX) return bad("too many samples");
        offs[i] = o = snap_layout(H, n_fac, rows);
        if (o.size != H.size) return bad("the declared size is not the byte count");
        // contents
        auto rd = [&R](int64_t off, size_t k, auto *dst) { memcpy(dst, R.data + off, sizeof(*dst) * k); };
        std::vector<int32_t> kpn;                 // the tracker part's keypoints' prev_index, newest frame first
        if (trk) {
            kpn.resize((size_t)H.n[0] + H.n[1]);
            rd(o.kp, kpn.size(), kpn.data());
            for (size_t k = 0; k < kpn.size(); ++k)
                if (kpn[k] < -1 || (k < (size_t)H.n[0] && kpn[k] >= H.n[1])) return bad("a prev_index outside its keypoint count");
        }
        WinSlot s;
        if (win) {
            s.resident = true; s.N = H.N; s.n_prior = s.prior_resident = H.n_prior; s.fixed = H.fixed;
            s.inertial = H.inertial; s.n_planes = H.n_planes; s.next_id = H.next_id;
            s.ids.resize(H.T); s.mask.resize(H.T); s.role.resize(H.T);
            rd(o.ids, H.T, s.ids.data()); rd(o.mask, H.T, s.mask.data()); rd(o.role, H.T, s.role.data());
            for (int r = 0; r < H.T; ++r) {
                if (s.ids[r] < 0 || s.ids[r] >= H.next_id || (r > 0 && s.ids[r] <= s.ids[r - 1]))
                    return bad("track ids not increasing or not below the next id");
                if (s.mask[r] == 0u || (s.mask[r] >> H.N) != 0u) return bad("a frame mask 0 or outside the window");
                if (s.role[r] < -2 || s.role[r] >= H.n_planes) return bad("a role not -1, -2 or a plane of the blob");
            }
            std::vector<int32_t> tkp(H.T);
            rd(o.tkp, H.T, tkp.data());
            const int cnt = !H.linked ? 0 : H.link_frame == H.frame_id ? H.n[0] : H.n[1];
            for (int r = 0; r < H.T; ++r) {
                if (tkp[r] < -1 || tkp[r] >= cnt) return bad("a keypoint index outside its keypoint count");
                s.link_kmax = std::max(s.link_kmax, (int)tkp[r]);
            }
            s.newest_kf = H.newest_kf; s.skipped = H.skipped;
        }
        if (R.slot < 0) continue;
        // the target's capacities
        if (H.N > h->Ncap) return bad("more frames than max_frames");
        TRY(check_window(h, s));
        s.n_samples.assign(h->Ncap, 0);
        std::copy(nsmp[i].begin(), nsmp[i].end(), s.n_samples.begin());
        if (R.tracker_slot >= 0 && H.linked) {
            const KltBatchState &B = h->kltb;
            s.link = true; s.link_tracker = R.tracker_slot; s.link_frame = H.link_frame;
            s.link_gen = ((size_t)R.tracker_slot < B.kps.size() ? B.kps[R.tracker_slot].gen : 0u) + 1u;
        } else {
            s.link_kmax = -1;
        }
        smax = std::max(smax, fmax);
        inertial |= H.inertial != 0;
        wslots.push_back(R.slot);
        next.push_back(std::move(s));
    }

    // buffers, grown as the other calls grow them
    KltBatchState &B = h->kltb;
    if (!wslots.empty()) {
        TRY(ensure_bw(h));
        if (inertial) TRY(ensure_inertial(h));
        if (smax > 0) TRY(ensure_imu_store(h, smax));
        TRY(ensure_plane_tables(h, next));
    }
    if (tseen.size() > B.kps.size()) B.kps.resize(tseen.size());
    if (tseen.size() > B.slots.size()) B.slots.resize(tseen.size());
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        if (R.tracker_slot < 0) continue;
        SlotKeypoints &K = B.kps[R.tracker_slot];
        for (int b = 0; b < 2; ++b)
            if (K.cap[b] < (size_t)H.n[b]) {
                const size_t need = std::max<size_t>(H.n[b], 1024);
                TRY(alloc(h, K.buf[b], SlotKeypoints::bytes(need), kDevice));
                K.cap[b] = need;
            }
        K.cur = 0;
        KltPyramids &c = B.slots[R.tracker_slot];
        if (H.levels > 0) {
            if (c.w != H.w || c.h != H.h || c.levels != H.levels) {
                c = KltPyramids{};
                klt_layout(c, H.w, H.h, H.levels);
            }
            for (auto &p : c.pyr) TRY(reserve(h, p, c.off[c.levels], kDevice));
        }
    }

    // staging: upload the blobs (16-byte aligned, first) | records | factors | re-layout
    std::vector<SnapRec> recs(n);
    std::vector<SnapFac> facs;
    int64_t area = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        const SnapOff &o = offs[i];
        int n_fac = 0, rows = 0;
        if (R.slot >= 0) {
            int64_t at = o.smp;
            for (int k = 0; k < (int)nsmp[i].size(); ++k)
                if (nsmp[i][k] > 0) {
                    facs.push_back(SnapFac{k, nsmp[i][k], at});
                    at += 56 * (int64_t)nsmp[i][k]; ++n_fac; rows += nsmp[i][k];
                }
        }
        SnapRec &r = recs[i];
        r = snap_rec(H, o, R.slot, area, (int)facs.size() - n_fac, n_fac, rows);
        r.link = R.slot >= 0 && R.tracker_slot >= 0 && H.linked;
        if (R.tracker_slot >= 0)
            snap_tracker(r, B.kps[R.tracker_slot], H.levels > 0 ? &B.slots[R.tracker_slot] : nullptr, 0);
        r.n[0] = R.tracker_slot >= 0 ? H.n[0] : 0; r.n[1] = R.tracker_slot >= 0 ? H.n[1] : 0;
        area += H.size;
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto blob = S.add<uint8_t>(Stage::kUp, (size_t)area);
    const auto rc = S.up(recs);
    const auto fc = S.up(facs);
    std::unique_ptr<Relayout> lay;
    if (!wslots.empty()) lay.reset(new Relayout(S, wslots.data(), next));
    TRY(S.place(h));
    for (int i = 0; i < n; ++i) memcpy(S.host(blob) + recs[i].base, records[i].data, heads[i].size);
    TRY(S.upload(h));
    bw_restore_kernel<<<n, kSnapThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(fc), S.dev(blob));
    ++h->launches;
    CK(h, cudaGetLastError());
    if (lay) {
        TRY(lay->launch(h, S, true));
        bw_restore_origin_kernel<<<n, 32, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(blob));
        ++h->launches;
        CK(h, cudaGetLastError());
    }
    CK(h, cudaStreamSynchronize(h->stream));

    // the host mirrors
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        if (R.slot >= 0) memcpy(&h->cst.h[R.slot], R.data + offs[i].cst, sizeof(WinConst));
        if (R.tracker_slot < 0) continue;
        SlotKeypoints &K = B.kps[R.tracker_slot];
        K.n = H.n[0]; K.prev_n = H.n[1]; K.live = true; K.frame_no = H.frame_no;
        K.frame_id = H.frame_id; K.prev_frame_id = H.prev_frame_id; ++K.gen;
        K.fx = H.K[0]; K.fy = H.K[1]; K.cx = H.K[2]; K.cy = H.K[3];
        KltPyramids &c = B.slots[R.tracker_slot];
        c.pyr_id[0] = H.levels > 0 ? H.frame_id : 0; c.pyr_clahe[0] = H.clahe;
        c.pyr_id[1] = 0; c.pyr_clahe[1] = 0.0;
    }
    commit(h, wslots.data(), next);
    return 0;
}

// ------------------------------------------------------------------------ the single resident window: slot 0
int pvio_b200_window_reset(pvio_b200_handle hh, const pvio_b200_window *constants) {
    if (!constants) return PVIO_B200_EINVAL;
    pvio_b200_window c = *constants;          // the arrays of `constants` are ignored, its plane counts with them
    c.n_planes = 0; c.n_plane_tracks = 0;
    return pvio_b200_batch_window_reset(hh, 0, &c);
}

int pvio_b200_window_set_prior(pvio_b200_handle hh, int n_prior, const double *S, const double *e, const double *state0) {
    return pvio_b200_batch_window_set_prior(hh, 0, n_prior, S, e, state0);
}

int pvio_b200_window_append_frame(pvio_b200_handle hh, const double *state, int fixed, const double *imu_record) {
    if (!state) return PVIO_B200_EINVAL;
    pvio_b200_window_edit e{};
    e.state = state; e.fixed = fixed; e.imu_record = imu_record;
    return pvio_b200_batch_window_edit(hh, 1, &e);
}

int pvio_b200_window_add_tracks(pvio_b200_handle hh, int n, const int32_t *frame, const double *z, const double *inv_depth, int32_t *ids_out) {
    pvio_b200_window_edit e{};
    e.n_new_tracks = n; e.new_frame = frame; e.new_z = z; e.new_inv_depth = inv_depth; e.new_ids = ids_out;
    return pvio_b200_batch_window_edit(hh, 1, &e);
}

int pvio_b200_window_add_observations(pvio_b200_handle hh, int n, const int32_t *track, const int32_t *frame, const double *z) {
    pvio_b200_window_edit e{};
    e.n_obs = n; e.obs_track = track; e.obs_frame = frame; e.obs_z = z;
    return pvio_b200_batch_window_edit(hh, 1, &e);
}

int pvio_b200_window_remove_track(pvio_b200_handle hh, int32_t track) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const WinSlot *s = window0(h);
    if (!s) return PVIO_B200_EINVAL;
    if (track < 0 || track >= s->next_id) return fail(h, PVIO_B200_EINVAL, "window_remove_track: unknown track");
    if (find_row(*s, track) < 0) return 0;    // already gone
    pvio_b200_window_edit e{};
    e.n_remove = 1; e.remove = &track;
    return pvio_b200_batch_window_edit(hh, 1, &e);
}

int pvio_b200_window_solve(pvio_b200_handle hh, const pvio_b200_options *opt, pvio_b200_summary *summary) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const int32_t slot = 0;
    return solve_slots(h, 1, &slot, opt, false, summary);
}

int pvio_b200_window_drop_victim(pvio_b200_handle hh) {
    const int32_t slot = 0;
    return pvio_b200_batch_window_drop_victim(hh, 1, &slot, nullptr, 0, nullptr, 0);
}

int pvio_b200_window_get(pvio_b200_handle hh, int32_t *n_frames, double *frames, int n_tracks, const int32_t *tracks,
                         double *inv_depth, int32_t *anchor_frame, int32_t *n_observations) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const WinSlot *s = window0(h);
    if (!s) return PVIO_B200_EINVAL;
    if (n_tracks > 0 && !tracks) return fail(h, PVIO_B200_EINVAL, "window_get: null track list");
    for (int i = 0; i < n_tracks; ++i)
        if (tracks[i] < 0 || tracks[i] >= s->next_id) return fail(h, PVIO_B200_EINVAL, "window_get: unknown track");
    if (n_frames) *n_frames = s->N;
    if (!frames && n_tracks <= 0) return 0;   // the frame count is the host's
    const int T = (int)s->ids.size();
    std::vector<double> rho(T);
    std::vector<int32_t> anchor(T), count(T);
    const int32_t slot = 0;
    TRY(pvio_b200_batch_window_download(hh, 1, &slot, nullptr, frames, (int64_t)s->N * kFrameStride, nullptr, T, nullptr,
                                        rho.data(), anchor.data(), count.data(), nullptr, nullptr));
    for (int i = 0; i < n_tracks; ++i) {
        const int r = find_row(*s, tracks[i]);   // a gone track: anchor -1, no observations, its inverse depth not written
        if (r >= 0 && inv_depth) inv_depth[i] = rho[r];
        if (anchor_frame) anchor_frame[i] = r >= 0 ? anchor[r] : -1;
        if (n_observations) n_observations[i] = r >= 0 ? count[r] : 0;
    }
    return 0;
}

}  // extern "C"
