// A new camera frame on the resident slots: localize (PnP on the slot's landmarks and triangulation of the new
// tracks), track_frame (IMU integration, prediction and the keyframe check), the tracker link (set_keypoints,
// mirror_frame), and track_camera, which runs feature_track and the mirror in one call.
#include <climits>
#include <cmath>
#include <cstddef>
#include <optional>
#include <vector>

#include "batch_window.cuh"
#include "imu.cuh"
#include "tri.cuh"

namespace pvio {

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

// The localize half of a batch of records (pvio_b200_batch_window_localize, pvio_b200_batch_window_track_frame): every
// record checked against its slot's host mirror, the observations that take part kept with the index they came from,
// the new tracks' keypoint pairs
struct LocPlan {
    std::vector<BwLoc> recs;
    std::vector<int32_t> rows, from;
    std::vector<double> zs, pts, nzs;
    int n_imu = 0;
};

// checks record R (imu_given: it must carry its IMU record when inertial) and appends it to the plan; null, or why the
// record is rejected
static const char *loc_add(const Handle *h, LocPlan &P, const pvio_b200_window_localize &R, bool imu_given) {
    const WinSlot &s = h->slots[R.slot];
    if (s.N < 1) return "a window without frames";
    if (!R.state || R.n_obs < 0 || R.n_new < 0 || (R.n_obs > 0 && (!R.obs_track || !R.obs_z)) ||
        (R.n_new > 0 && (!R.new_z_last || !R.new_z || !R.new_valid || !R.new_inv_depth)))
        return "null array";
    if (imu_given && R.use_inertial && !R.imu_record)
        return "an inertial record needs the IMU record from the newest frame";
    P.recs.push_back(BwLoc{R.slot, s.N - 1, R.use_inertial ? 1 : 0, 0, (int32_t)P.rows.size(), R.use_inertial ? P.n_imu++ : -1,
                           R.n_new, (int32_t)(P.nzs.size() / 4)});
    BwLoc &L = P.recs.back();
    const uint32_t newest = 1u << (s.N - 1);
    std::vector<uint8_t> named(s.ids.size(), 0);
    for (int k = 0; k < R.n_obs; ++k) {
        const int r = find_row(s, R.obs_track[k]);
        if (r < 0) return "unknown or dead track";
        if (named[r]) return "a track named twice";
        named[r] = 1;
        const double *z = R.obs_z + 2 * k;
        if (!std::isfinite(z[0]) || !std::isfinite(z[1])) return "non-finite keypoint";
        const double *x = R.obs_point ? R.obs_point + 3 * k : nullptr;
        const bool given = x && std::isfinite(x[0]) && std::isfinite(x[1]) && std::isfinite(x[2]);
        if (x && !given && !(std::isnan(x[0]) && std::isnan(x[1]) && std::isnan(x[2])))
            return "a point row neither finite nor NaN";
        if (!(s.mask[r] & newest)) continue;                              // pnp.cpp:58
        if (!given && s.role[r] != -1) return "a plane track without its plane-cast point";
        P.rows.push_back(r);
        P.from.push_back(k);
        P.zs.insert(P.zs.end(), z, z + 2);
        for (int j = 0; j < 3; ++j) P.pts.push_back(given ? x[j] : NAN);
    }
    L.n_obs = (int32_t)P.rows.size() - L.obs_off;
    for (int k = 0; k < R.n_new; ++k) {
        const double *a = R.new_z_last + 2 * k, *b = R.new_z + 2 * k;
        if (!std::isfinite(a[0]) || !std::isfinite(a[1]) || !std::isfinite(b[0]) || !std::isfinite(b[1]))
            return "non-finite keypoint";
        P.nzs.insert(P.nzs.end(), {a[0], a[1], b[0], b[1]});
    }
    return nullptr;
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
    TRY(launched(h, "bw_localize_gather_kernel"));
    TRY(launch_pnp(h, n, L.args));
    CK(h, cudaGetLastError());
    bw_localize_triangulate_kernel<<<n, kLocTriThreads, 0, h->stream>>>(a, L);
    return launched(h, "bw_localize_triangulate_kernel");
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
        return launched(h, "bw_track_integrate_kernel");
    }

    // mirror, then track_frame's kernels on its lists; integrate_jobs: the integrate launch's jobs from j0
    int launch(Handle *h, int j0) {
        const int n = (int)mir.size();
        const BwArgs a = launch_args<BwArgs>(h);
        bw_mirror_kernel<<<n, kBwThreads, 0, h->stream>>>(a, M);
        TRY(launched(h, "bw_mirror_kernel"));
        TRY(integrate(h, j0, (int)jobs.size() - j0));
        TRY(loc_launch(h, L, n));
        bw_track_keyframe_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L, T);
        return launched(h, "bw_track_keyframe_kernel");
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
        TRY(launched(h, "bw_mirror_append_kernel"));
        bw_edit_kernel<<<n, kBwThreads, 0, h->stream>>>(a, S.dev(ed), nullptr, S.dev(nw), S.dev(ob), S.dev(xs), S.dev(eout));
        TRY(launched(h, "bw_edit_kernel"));
        TRY(lay->launch(h, S, false));
        if (!kimu.empty()) {
            bw_set_imu_kernel<<<(int)kimu.size(), kBwThreads, 0, h->stream>>>(a, S.dev(kim), S.dev(smp), S.dev(kax));
            TRY(launched(h, "bw_set_imu_kernel"));
        }
        bw_mirror_link_kernel<<<n, kBwThreads, 0, h->stream>>>(a, M);
        TRY(launched(h, "bw_mirror_link_kernel"));
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

}  // namespace pvio

using namespace pvio;

extern "C" {

int pvio_b200_batch_window_localize(pvio_b200_handle hh, int n, pvio_b200_window_localize *records,
                                    const pvio_b200_options *opt) {
    BwCall C(hh, "batch_window_localize");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record is checked against its slot's host mirror before anything is staged
    LocPlan P;
    for (int i = 0; i < n; ++i)
        if (const char *why = loc_add(h, P, records[i], true)) return C.bad(why);
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
    BwCall C(hh, "batch_window_track_frame");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record is checked before anything is staged: its localize half as localize checks it, then the rest
    LocPlan P;
    std::vector<BwTrack> trs(n);
    std::vector<BwTrackJob> jobs;
    std::vector<int32_t> kf_row;
    std::vector<double> kf_z;
    size_t rows = 0, par = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_track_frame &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return C.bad("the window carries no motion states");
        if (const char *why = loc_add(h, P, localize_view(R), false)) return C.bad(why);
        if (!R.samples || !R.noise_cov || !R.imu_record || !R.keyframe || !R.skipped_frames) return C.bad("null array");
        if (R.n_samples < 1) return C.bad("a frame without IMU samples (integrate() returns false, preintegrator.cpp:86)");
        if (R.newest_is_keyframe != 0 && R.newest_is_keyframe != 1) return C.bad("newest_is_keyframe not 0 or 1");
        const bool merged = R.newest_is_keyframe == 0;
        if (merged && s.N < 2) return C.bad("a non-keyframe newest frame without a keyframe before it");
        if (merged && (R.n_merge < 1 || !R.merge_samples)) return C.bad("a non-keyframe newest frame without its samples");
        if (!merged && (R.n_merge != 0 || R.merge_samples)) return C.bad("a merge list with a keyframe newest frame");
        if (!all_finite(R.samples, 7 * (int64_t)R.n_samples) || (merged && !all_finite(R.merge_samples, 7 * (int64_t)R.n_merge)))
            return C.bad("non-finite sample");
        if (!std::isfinite(R.t_end) || !all_finite(R.noise_cov, 36) || !std::isfinite(R.cx) || !std::isfinite(R.cy))
            return C.bad("non-finite t_end, noise or principal point");
        if (*R.skipped_frames < 0) return C.bad("negative skipped_frames");
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
        if (e > (size_t)INT32_MAX || par > (size_t)INT32_MAX) return C.bad("too many samples or pairs in one call");
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
    TRY(launched(h, "bw_track_integrate_kernel"));
    TRY(loc_launch(h, L, n));
    bw_track_keyframe_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L, T);
    TRY(launched(h, "bw_track_keyframe_kernel"));
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

int pvio_b200_batch_window_set_keypoints(pvio_b200_handle hh, int n, const pvio_b200_window_keypoints *records) {
    BwCall C(hh, "batch_window_set_keypoints");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    std::vector<BwKeys> ks(n);
    std::vector<int2> pairs;
    std::vector<int> kmax(n, -1);
    std::vector<uint32_t> gens(n, 0);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_keypoints &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (s.N < 1) return C.bad("a window without frames");
        if (R.tracker_slot < 0 || R.tracker_slot > kMaxBatchSlot) return C.bad("tracker slot out of range");
        if (!R.frame_id) return C.bad("frame id 0");
        const KltBatchState &B = h->kltb;
        const SlotKeypoints *K = (size_t)R.tracker_slot < B.kps.size() ? &B.kps[R.tracker_slot] : nullptr;
        if (!K || !K->live || (R.frame_id != K->frame_id && R.frame_id != K->prev_frame_id))
            return C.bad("the frame is not one of the tracker slot's two newest");
        gens[i] = K->gen;
        if (R.n < 0 || (R.n > 0 && (!R.track || !R.keypoint))) return C.bad("null array");
        if (R.newest_is_keyframe != 0 && R.newest_is_keyframe != 1) return C.bad("newest_is_keyframe not 0 or 1");
        if (R.skipped_frames < 0) return C.bad("negative skipped_frames");
        ks[i] = BwKeys{R.slot, (int32_t)s.ids.size(), R.n, (int32_t)pairs.size()};
        const uint32_t newest = 1u << (s.N - 1);
        std::vector<uint8_t> named(s.ids.size(), 0);
        std::vector<int32_t> kps(R.keypoint, R.keypoint + R.n);
        for (int k = 0; k < R.n; ++k) {
            const int r = find_row(s, R.track[k]);
            if (r < 0) return C.bad("unknown or dead track");
            if (!(s.mask[r] & newest)) return C.bad("a track not observed in the newest frame");
            if (named[r]) return C.bad("a track named twice");
            named[r] = 1;
            if (R.keypoint[k] < 0) return C.bad("negative keypoint index");
            pairs.push_back(make_int2(r, R.keypoint[k]));
            kmax[i] = std::max(kmax[i], (int)R.keypoint[k]);
        }
        std::sort(kps.begin(), kps.end());
        if (std::adjacent_find(kps.begin(), kps.end()) != kps.end()) return C.bad("a keypoint named twice");
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto k = S.up(ks);
    const auto p = S.up(pairs);
    TRY(S.place(h, true));
    bw_set_keypoints_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(k), S.dev(p));
    TRY(launched(h, "bw_set_keypoints_kernel"));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_keypoints &R = records[i];
        WinSlot &s = h->slots[R.slot];
        s.link = true; s.link_tracker = R.tracker_slot; s.link_frame = R.frame_id; s.link_kmax = kmax[i]; s.link_gen = gens[i];
        s.newest_kf = R.newest_is_keyframe; s.skipped = R.skipped_frames;
    }
    return 0;
}

int pvio_b200_batch_window_mirror_frame(pvio_b200_handle hh, int n, pvio_b200_window_mirror *records,
                                        const pvio_b200_options *opt) {
    BwCall C(hh, "batch_window_mirror_frame");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record is checked against its slot's host mirror and its tracker slot before anything is staged
    const KltBatchState &B = h->kltb;
    MirCall M(h, C.what, n);
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
        if (const char *why = M.add(h, i, R, v, ok ? nullptr : "the tracker slot's previous frame is not the slot's newest frame",
                                    false))
            return C.bad(why);
        fid[i] = K->frame_id; gen[i] = K->gen;
    }
    TRY(M.stage(h, records, opt, false));
    TRY(M.launch(h, 0));
    TRY(M.check(h, false));
    TRY(M.append(h));
    return M.commit_out(h, records, fid.data(), gen.data());
}

int pvio_b200_batch_window_track_camera(pvio_b200_handle hh, int n, pvio_b200_window_camera *records, int max_level,
                                        int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                                        int border, double ransac_threshold, double ransac_confidence,
                                        double keypoint_distance, const pvio_b200_options *opt) {
    BwCall C(hh, "batch_window_track_camera");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
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
    MirCall M(h, C.what, n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_camera &R = records[i];
        if (!h->slots[R.slot].inertial) return C.bad("the window carries no motion states");
        if (R.map_frames == 0) return C.bad("map_frames 0 (a sequence start goes through batch_feature_track)");
        if (!R.n_keypoints) return C.bad("null array");
        if (R.fx != h->cst.h[R.slot].fx || R.fy != h->cst.h[R.slot].fy) return C.bad("fx, fy not the slot's");
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
        if (const char *why = M.add(h, i, mr[i], v, ok ? nullptr : "the tracker slot's newest frame is not the slot's newest frame",
                                    true))
            return C.bad(why);
        fid[i] = R.frame_id; gen[i] = K.gen;
    }

    // the mirror's staging, laid out for every new frame's output bound and uploaded; the step-1 integration and
    // prediction from each slot's newest frame; the feature stages with delta_key_q composed from it on the device
    TRY(M.stage(h, mr.data(), opt, true));
    TRY(M.integrate(h, 0, M.n1));
    static_assert(offsetof(BwLoc, slot) == 0 && sizeof(BwLoc) % sizeof(int32_t) == 0,
                  "ft_predict_kernel reads each record's window slot from the staged BwLoc records");
    const FtPredict pred{M.S.dev(M.rec1), launch_args<BwArgs>(h).cst, &M.S.dev(M.lo)->slot,
                         (int)(sizeof(BwLoc) / sizeof(int32_t)), M.S.dev(M.pq)};
    TRY(ft_run(h, n, ff.data(), ko, keypoint_distance, &pred, run));
    for (int i = 0; i < n; ++i)
        if (run.count[i] > run.out_cap[i]) return C.bad("more keypoints than the stated bound");

    // the new frames into the mirror's records; mirror, track_frame's kernels, the capacity check, the append; then the
    // tracker slots and the window slots commit
    for (int i = 0; i < n; ++i) {
        const SlotKeypoints &K = B.kps[records[i].tracker_slot];
        BwMirror &m = M.S.host(M.mr)[i];
        m.zj = K.z(2); m.prev = K.prev(2); m.n_j = run.count[i];
        M.mir[i] = m;
    }
    TRY(M.S.upload(h, M.mr));
    TRY(M.launch(h, M.n1));
    TRY(M.check(h, true));
    TRY(M.append(h));
    TRY(ft_finish(h, n, ff.data(), run));
    for (int i = 0; i < n; ++i)
        if (records[i].predict_q) memcpy(records[i].predict_q, M.S.host(M.pq) + 4 * (size_t)i, sizeof(double) * 4);
    return M.commit_out(h, mr.data(), fid.data(), gen.data());
}

}  // extern "C"
