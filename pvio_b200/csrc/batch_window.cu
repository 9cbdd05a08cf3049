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
#include <climits>
#include <cmath>
#include <vector>

#include "batch_window.cuh"
#include "imu.cuh"

namespace pvio {

// ------------------------------------------------------------------------ staged records (host -> device)
struct BwDl { int32_t slot, N, T, pad; int64_t off; };                  // download: bytes into the result area
struct BwPlanes { int32_t slot, n_planes, n_set, set_off, param_off, pad; };   // one set_planes record (n_planes < 0: keep)
struct BwRole { int32_t row, role; double rho; };                       // rho NaN: keep the row's inverse depth

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

__global__ void __launch_bounds__(kBwThreads) bw_set_imu_kernel(BwArgs a, const BwImu *recs, const double *smp,
                                                                const double *aux) {
    const BwImu r = recs[blockIdx.x];
    const size_t F = (size_t)r.slot * a.Ncap + r.factor;
    double *dst = a.imu_s + F * a.Scap * 7;
    const double *src = smp + (size_t)r.off * 7;
    for (int i = threadIdx.x; i < 7 * r.n; i += kBwThreads) dst[i] = src[i];
    for (int i = threadIdx.x; i < kImuAux; i += kBwThreads) a.imu_aux[F * kImuAux + i] = aux[(size_t)blockIdx.x * kImuAux + i];
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

int ensure_bw(Handle *h) {
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

int ensure_imu_store(Handle *h, int S) {
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

int check_window(Handle *h, const WinSlot &s) {
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

void compact_rows(WinSlot &s, int shift) {
    size_t o = 0;
    for (size_t r = 0; r < s.ids.size(); ++r) {
        const uint32_t m = s.mask[r] >> shift;
        if (m) { s.ids[o] = s.ids[r]; s.mask[o] = m; s.role[o] = s.role[r]; ++o; }
    }
    s.ids.resize(o); s.mask.resize(o); s.role.resize(o);
}

Relayout::Relayout(Stage &S, const int32_t *sl, const std::vector<WinSlot> &next) : lays(next.size()) {
    for (size_t i = 0; i < next.size(); ++i) lays[i] = layout_of(sl[i], next[i]);
    lay = S.up(lays);
    slots = S.add(Stage::kUp, next.size(), sl);
}

int Relayout::launch(Handle *h, const Stage &S, bool prior) const {
    const int n = (int)lays.size();
    bw_layout_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(lay));
    TRY(launched(h, "bw_layout_kernel"));
    return launch_layout_tail(h, S.dev(slots), n, prior);
}

void commit(Handle *h, const int32_t *slots, std::vector<WinSlot> &next) {
    for (size_t i = 0; i < next.size(); ++i) {
        h->slots[slots[i]] = std::move(next[i]);
        host_header(h, slots[i]);
    }
}

int ensure_plane_tables(Handle *h, const std::vector<WinSlot> &next) {
    int T = 0, O = 0;
    for (const WinSlot &s : next) { const BwShape sh = shape_of(s); T = std::max(T, sh.T); O = std::max(O, sh.O); }
    return T > 0 ? ensure_planes(h, T, O) : 0;
}

int check_slots(Handle *h, int n, const int32_t *slots, const char *what) {
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
        TRY(launched(h, "bw_reintegrate_kernel"));
    }
    CK(h, cudaEventRecord(h->ev0, h->stream));
    TRY(run_named_solve(h, opt, range, S.dev(nm), named.data()));
    CK(h, cudaEventRecord(h->ev1, h->stream));
    if (post) TRY(run_postpass_slots(h, n, S.dev(sl)));
    bw_writeback_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(lay), post ? 1 : 0);
    TRY(launched(h, "bw_writeback_kernel"));
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

// slot 0 as the single resident window (pvio_b200_window_*); null, with the error set, before pvio_b200_window_reset
static const WinSlot *window0(Handle *h) {
    if (!h->slots[0].resident) {
        fail(h, PVIO_B200_EINVAL, "window: no resident window: call pvio_b200_window_reset first");
        return nullptr;
    }
    return &h->slots[0];
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
    TRY(launched(h, "bw_edit_kernel"));
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
    BwCall C(hh, "batch_window_set_planes");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record is applied to a copy of its slot's host mirror; nothing is staged before all of them passed
    std::vector<WinSlot> next(n);
    std::vector<BwPlanes> recs(n);
    std::vector<BwRole> roles;
    std::vector<double> params;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_planes &R = records[i];
        WinSlot s = h->slots[R.slot];
        if (R.n_planes < -1 || R.n_planes > h->Pcap) return C.bad("plane count outside -1 (keep) .. 4");
        if (R.n_set < 0 || (R.n_set > 0 && (!R.track || !R.role)) || (R.n_planes > 0 && !R.plane_param))
            return C.bad("null array");
        recs[i] = BwPlanes{R.slot, std::max(R.n_planes, 0), R.n_set, (int32_t)roles.size(), (int32_t)params.size(), 0};
        if (R.n_planes >= 0) {
            for (int k = 0; k < 4 * R.n_planes; ++k)
                if (!std::isfinite(R.plane_param[k])) return C.bad("non-finite plane parameters");
            params.insert(params.end(), R.plane_param, R.plane_param + 4 * R.n_planes);
            s.n_planes = R.n_planes;
        }
        std::vector<uint8_t> named(s.ids.size(), 0);
        for (int k = 0; k < R.n_set; ++k) {
            const int r = find_row(s, R.track[k]);
            if (r < 0) return C.bad("unknown or dead track");
            if (named[r]) return C.bad("a track named twice");
            named[r] = 1;
            const int role = R.role[k];
            if (role < -2 || role >= s.n_planes) return C.bad("role not -1, -2 or a plane of the slot");
            const double rho = R.inv_depth ? R.inv_depth[k] : NAN;
            if (std::isinf(rho)) return C.bad("infinite inverse depth");
            s.role[r] = (int8_t)role;
            roles.push_back(BwRole{r, role, rho});
        }
        for (int8_t ro : s.role)
            if (ro >= s.n_planes) return C.bad("a track keeps a plane the slot no longer has");
        TRY(check_window(h, s));
        next[i] = std::move(s);
    }
    TRY(ensure_plane_tables(h, next));
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto ro = S.up(roles);
    const auto pa = S.up(params);
    const Relayout lay(S, C.slots.data(), next);
    TRY(S.place(h, true));
    bw_planes_kernel<<<n, kBwThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rec), S.dev(ro), S.dev(pa));
    TRY(launched(h, "bw_planes_kernel"));
    TRY(lay.launch(h, S, false));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, C.slots.data(), next);
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
    TRY(launched(h, "bw_drop_kernel"));
    TRY(lay.launch(h, S, true));
    CK(h, cudaStreamSynchronize(h->stream));
    commit(h, slots, next);
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
    TRY(launched(h, "bw_download_kernel"));
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

int pvio_b200_batch_window_set_imu(pvio_b200_handle hh, int n, const pvio_b200_window_imu *records) {
    BwCall C(hh, "batch_window_set_imu");
    if (!C.open(n, records, false)) return C.rc;
    Handle *h = C.h;
    // every record is checked before anything is staged
    std::vector<BwImu> recs(n);
    std::vector<std::pair<int32_t, int32_t>> pairs(n);
    size_t rows = 0;
    int smax = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_imu &R = records[i];
        if (R.slot < 0 || R.slot >= h->W || !h->slots[R.slot].resident) return C.bad("slot out of range or not resident");
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return C.bad("the window carries no motion states");
        if (R.frame < 1 || R.frame >= s.N) return C.bad("frame outside 1 .. N - 1");
        if (R.n_samples < 1) return C.bad("a factor without IMU samples (integrate() returns false, preintegrator.cpp:86)");
        if (!R.samples || !R.noise_cov) return C.bad("null array");
        if (!all_finite(R.samples, 7 * (int64_t)R.n_samples)) return C.bad("non-finite sample");
        if (!std::isfinite(R.t_end)) return C.bad("non-finite t_end");
        if (!all_finite(R.noise_cov, 36)) return C.bad("non-finite noise");
        recs[i] = BwImu{R.slot, R.frame - 1, R.n_samples, (int32_t)rows};
        pairs[i] = {R.slot, R.frame};
        rows += R.n_samples;
        smax = std::max(smax, R.n_samples);
    }
    std::sort(pairs.begin(), pairs.end());
    if (std::adjacent_find(pairs.begin(), pairs.end()) != pairs.end()) return C.bad("a (slot, frame) named twice");
    if (rows > (size_t)INT32_MAX) return C.bad("too many samples in one call");
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
    TRY(launched(h, "bw_set_imu_kernel"));
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
    TRY(launched(h, "bw_imu_records_kernel"));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i)
        memcpy(records + i * records_stride, S.host(out) + dls[i].off, sizeof(double) * (size_t)(dls[i].N - 1) * kImuStride);
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
