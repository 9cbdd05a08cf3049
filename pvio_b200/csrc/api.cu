// libpvio_b200: C-ABI entry points (include/pvio_b200.h), host-side packing and launch
// orchestration of the bundle-adjustment kernels.  No torch types, no CPU fallback, no environment switches:
// one pipeline (frame-major table -> linearise -> Schur -> solve -> back-substitution / candidate), in fp32
// Jacobians for visual-only windows and fp64 for windows with motion states.
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include "api_internal.h"
#include "ba_fobs.cuh"
#include "ba_linearize.cuh"
#include "ba_schur.cuh"
#include "ba_solve.cuh"
#include "ba_cov.cuh"
#include "ba_tr.cuh"
#include "ba_update.cuh"

namespace pvio {

int fail(Handle *h, int code, const char *what, cudaError_t e) {
    if (h) {
        h->err = what ? what : "";
        if (e != cudaSuccess) { h->err += ": "; h->err += cudaGetErrorString(e); }
    }
    return code;
}

void drop_graphs(Handle *h) {
    for (auto &kv : h->graphs) cudaGraphExecDestroy(kv.second.first);
    h->graphs.clear();
}

static LinBufs lin_bufs(Handle *h) {
    const size_t W = h->W, N = h->Ncap, M = h->Mcap, es = h->hs_double ? sizeof(double) : sizeof(float);
    LinBufs b;
    b.hs = W * N * M * 6 * es; b.jr = W * N * M * 2 * es; b.lm_w = W * M * 2 * es;
    b.lm_msk = W * M; b.lm_aux = W * M;
    b.Hred = h->sys_set; b.Hdd = h->sys_set; b.g = h->sys_set; b.cost = h->sys_set;
    return b;
}

// pinned staging: slot j of src -> slot i of dst (a slot of the shorter stride; the arrays may differ in stride only)
template <typename T>
static void copy_slot(DevBuf<T> &dst, size_t i, const DevBuf<T> &src, size_t j) {
    memcpy(dst.slot(i), src.slot(j), sizeof(T) * std::min(dst.per, src.per));
}

// f(t.table...) for each table of the plane-table sets t (ensure_planes pairs the grown tables with the old ones)
template <typename F, typename... P>
static void for_each_plane_table(F f, P &...t) {
    f(t.plane_param...); f(t.pt_plane...); f(t.pt_begin...); f(t.pt_frame...); f(t.pt_z...);
}

// Every per-slot array the host stages in pinned memory and copies to the device slot by slot: f(array, prior) for the
// vision arrays, then the inertial arrays and the prior (prior: its S, e and x0) when allocated, then the plane tables
// when allocated.  Stops at the first f that returns non-zero and returns that code.  A new per-slot array needs its
// alloc and one entry here.
template <typename F>
static int for_each_staged(Handle *h, F f) {
    int rc = 0;
    auto v = [&](auto &b, bool prior) { if (rc == 0) rc = f(b, prior); };
    v(h->hdr, false); v(h->cst, false); v(h->obs, false); v(h->lms, false); v(h->rho, false); v(h->frames, false);
    if (h->have_inertial) {
        v(h->imu_idx, false); v(h->imu_data, false); v(h->prior_frames, false);
        v(h->prior_S, true); v(h->prior_e, true); v(h->prior_x0, true);
    }
    if (h->have_planes) for_each_plane_table([&](auto &b) { v(b, false); }, h->planes);
    return rc;
}

// The handle's arrays as the kernels see them (BatchArrays).  Called after every (re)allocation, which also drops the
// cached graphs: their launches carry the old view.
static void refresh_arrays(Handle *h) {
    BatchArrays &a = h->arrays;
    const size_t W = h->W, N = h->Ncap, npc = N * (N + 1) / 2;
    a.hdr = h->hdr.d; a.cst = h->cst.d; a.obs = h->obs.d; a.fz = h->fz.d; a.flm = h->flm.d; a.seg = h->seg.d; a.lms = h->lms.d;
    a.rho = h->rho.d; a.frames = h->frames.d; a.ctrl = h->ctrl.d; a.rho_cand = h->rho_cand.d; a.frames_cand = h->frames_cand.d;
    a.lm_scale = h->lm_scale.d; a.lm_aux = h->lm_aux.d; a.lm_w = h->lm_w.d; a.lm_msk = h->lm_msk.d; a.jr = h->jr.d; a.hs = h->hs.d;
    // the reduced-system outputs of set 0 lie back to back in Hred, set 1 sys_set elements behind them (LinBufs)
    a.Hred = h->Hred.d; a.Hdd = a.Hred + W * npc * 36; a.gdir = a.Hdd + W * N * 36; a.gred = a.gdir + W * N * 6;
    a.cost_vis = a.gred + W * N * 6;
    a.dx_pose = h->dx_pose.d; a.dx_lm = h->dx_lm.d; a.v_pose = h->v_pose.d; a.lm_v = h->lm_v.d; a.pose_scale = h->pose_scale.d;
    a.acc = h->acc.d; a.aux_cost = h->aux_cost.d;
    a.imu_idx = h->imu_idx.d; a.imu_data = h->imu_data.d; a.prior_frames = h->prior_frames.d; a.prior_S = h->prior_S.d;
    a.prior_L = h->prior_L.d; a.prior_e = h->prior_e.d; a.prior_x0 = h->prior_x0.d;
    const PlaneTables &p = h->planes;
    a.plane_param = p.plane_param.d; a.pt_plane = p.pt_plane.d; a.pt_begin = p.pt_begin.d; a.pt_frame = p.pt_frame.d;
    a.pt_z = p.pt_z.d; a.pt_J = h->pt_J.d;
    a.Ncap = h->Ncap; a.Mcap = h->Mcap; a.Kcap = h->Kcap; a.Pcap = h->Pcap; a.Tcap = h->Tcap; a.Ocap = h->Ocap;
    a.bufs = lin_bufs(h);
}

int ensure_inertial(Handle *h) {
    if (h->have_inertial) return 0;
    const size_t W = h->W, N = h->Ncap, M = h->Mcap, dcap = 15 * N;
    cudaStreamSynchronize(h->stream);
    drop_graphs(h);                                 // the record array is reallocated below: pointers in cached graphs go stale
    TRY(alloc(h, h->imu_idx, W * N * 2, kBoth, N * 2));
    TRY(alloc(h, h->imu_data, W * N * kImuStride, kBoth, N * kImuStride));
    TRY(alloc(h, h->prior_frames, W * N, kBoth, N));
    TRY(alloc(h, h->prior_S, W * dcap * dcap, kBoth, dcap * dcap));
    TRY(alloc(h, h->prior_L, W * dcap * dcap, kDevice, dcap * dcap));
    TRY(alloc(h, h->prior_e, W * dcap, kBoth, dcap));
    TRY(alloc(h, h->prior_x0, W * N * kFrameStride, kBoth, N * kFrameStride));
    // windows with motion states run the fp64 pipeline: h records of 8-byte elements, two buffer sets (LinBufs)
    TRY(alloc(h, h->hs, 2 * W * N * M * 6 * sizeof(double), kDevice));
    TRY(alloc(h, h->jr, 2 * W * N * M * 2 * sizeof(double), kDevice));
    TRY(alloc(h, h->lm_w, 2 * W * M * 2 * sizeof(double), kDevice));
    h->hs_double = true;
    h->have_inertial = true;
    refresh_arrays(h);
    return 0;
}

// device array src -> device array dst slot by slot, the arrays differing in slot stride only (on the handle's stream)
template <typename T>
static int copy_slots_d2d(Handle *h, DevBuf<T> &dst, const DevBuf<T> &src) {
    CK(h, cudaMemcpy2DAsync(dst.d, sizeof(T) * dst.per, src.d, sizeof(T) * src.per, sizeof(T) * std::min(dst.per, src.per),
                            (size_t)h->W, cudaMemcpyDeviceToDevice, h->stream));
    return 0;
}

// Plane buffers grow on demand WITHOUT losing any slot's tables: the slots packed into the pinned staging area, and the
// device copies, which the resident windows (batch_window.cu) build on the device and never upload.
int ensure_planes(Handle *h, int T, int O) {
    if (h->have_planes && T <= h->Tcap && O <= h->Ocap) return 0;
    const int Tn = std::max({T, h->Tcap, 256}), On = std::max({O, h->Ocap, 256 * 8});
    const size_t W = h->W;
    cudaStreamSynchronize(h->stream);
    drop_graphs(h);
    const size_t P4 = (size_t)h->Pcap * 4;
    PlaneTables next;
    TRY(alloc(h, next.plane_param, W * P4, kBoth, P4));
    TRY(alloc(h, next.pt_plane, W * Tn, kBoth, Tn));
    TRY(alloc(h, next.pt_begin, W * (Tn + 1), kBoth, Tn + 1));
    TRY(alloc(h, next.pt_frame, W * On, kBoth, On));
    TRY(alloc(h, next.pt_z, W * On * 2, kBoth, On * 2));
    if (h->have_planes) {
        int rc = 0;
        for_each_plane_table([&](auto &dst, auto &src) {
            for (size_t i = 0; i < W; ++i) copy_slot(dst, i, src, i);
            if (rc == 0) rc = copy_slots_d2d(h, dst, src);
        }, next, h->planes);
        TRY(rc);
        CK(h, cudaStreamSynchronize(h->stream));      // the old arrays are freed below
    }
    h->planes = std::move(next);
    TRY(alloc(h, h->pt_J, W * Tn * (6 * (size_t)h->Ncap + 2), kDevice));      // device scratch of solve_kernel's plane block
    h->Tcap = Tn; h->Ocap = On;
    h->have_planes = true;
    refresh_arrays(h);
    return 0;
}

// ------------------------------------------------------------------------ small kernels
// Lambda = S^T S of the marginalisation prior (once per upload; constant across iterations)
// slots (may be NULL): CTA row b works on window slots[b] instead of w0 + b
__global__ void prior_lambda_kernel(const WinHdr *hdr, const double *S, double *L, int Ncap, int w0, const int32_t *slots) {
    const int w = slots ? slots[blockIdx.x] : blockIdx.x + w0;
    const int d = 15 * hdr[w].n_prior, dcap = 15 * Ncap;
    const double *Sw = S + (size_t)w * dcap * dcap;
    double *Lw = L + (size_t)w * dcap * dcap;
    // gridDim.y CTAs share a window (a single window would otherwise leave all SMs but one idle)
    for (int e = blockIdx.y * blockDim.x + threadIdx.x; e < d * d; e += blockDim.x * gridDim.y) {
        const int i = e / d, j = e - i * d;
        double s = 0.0;
        for (int k = 0; k < d; ++k) s += Sw[(size_t)k * d + i] * Sw[(size_t)k * d + j];
        Lw[e] = s;
    }
}

// Landmark post-pass (bundle_adjustor.cpp:277-296): depth test in every observing camera
// (anchor included) and mean pixel reprojection error.  One group of 16 lanes per landmark.
__global__ void postpass_kernel(const WinHdr *hdr, const WinConst *cst, const ObsRec *obs, const LmRec *lms,
                                const double *rho, const double *frames, uint8_t *valid, double *quality,
                                double *err_acc, int Ncap, int Mcap, int Kcap, int w0, const int32_t *slots) {
    const int w = slots ? slots[blockIdx.y] : blockIdx.y + w0;
    const WinHdr &H = hdr[w];
    const WinConst &wc = cst[w];
    __shared__ FrameSm F[kMaxFrames];
    if (threadIdx.x < H.N) make_frame(frames + ((size_t)w * Ncap + threadIdx.x) * kFrameStride, wc, F[threadIdx.x]);
    __syncthreads();
    const int lane = threadIdx.x & (kGroup - 1);
    const int gid = (blockIdx.x * blockDim.x + threadIdx.x) / kGroup;
    const int ngrp = gridDim.x * blockDim.x / kGroup;
    for (int l0 = 0; l0 < H.M; l0 += ngrp) {
        const int l = l0 + gid;
        const bool ok = l < H.M;
        const LmRec lr = lms[(size_t)w * Mcap + (ok ? l : 0)];
        const int n_obs = ok ? lm_nobs(lr.meta) : 0;
        const int anchor = lm_anchor(lr.meta);
        const unsigned fmask = ok ? lm_mask(lr.meta) : 0u;
        double x[3];
        float xf[3], cl[3];
        world_point(F[anchor], lr.zrx, lr.zry, ok ? rho[(size_t)w * Mcap + l] : 1.0, x, xf, cl);
        // lane = frame: its observation is record popc(mask below the lane); the anchor lane uses z_ref
        int frame = -1;
        float zx = 0.f, zy = 0.f;
        if ((fmask >> lane) & 1u) {
            const ObsRec o = obs[(size_t)w * Kcap + lr.obs_begin + __popc(fmask & ((1u << lane) - 1u))];
            frame = lane; zx = o.zx; zy = o.zy;
        } else if (lane == anchor && ok) {
            frame = anchor; zx = lr.zrx; zy = lr.zry;
        }
        double e = 0.0;
        int bad = 0;
        if (frame >= 0) {
            const FrameSm &Ft = F[frame];
            const double d0 = x[0] - Ft.c[0], d1 = x[1] - Ft.c[1], d2 = x[2] - Ft.c[2];
            const double y0 = Ft.Rwc[0] * d0 + Ft.Rwc[3] * d1 + Ft.Rwc[6] * d2;
            const double y1 = Ft.Rwc[1] * d0 + Ft.Rwc[4] * d1 + Ft.Rwc[7] * d2;
            const double y2 = Ft.Rwc[2] * d0 + Ft.Rwc[5] * d1 + Ft.Rwc[8] * d2;
            if (y2 <= 1.0e-3 || y2 > 50.0) bad = 1;                        // :286
            const double ex = (y0 / y2 - (double)zx) * wc.fx, ey = (y1 / y2 - (double)zy) * wc.fy;
            e = sqrt(ex * ex + ey * ey);                                   // :291
        }
        const unsigned badm = __ballot_sync(0xffffffffu, bad);
        const int grp_bad = (badm >> (threadIdx.x & 16)) & 0xffff;
#pragma unroll
        for (int off = kGroup / 2; off > 0; off >>= 1) e += __shfl_xor_sync(0xffffffffu, e, off, kGroup);
        if (ok && lane == 0) {
            const bool v = grp_bad == 0;
            if (valid) valid[(size_t)w * Mcap + l] = v ? 1 : 0;
            if (quality) quality[(size_t)w * Mcap + l] = v ? e / fmax((double)(n_obs + 1), 1.0) : 0.0;
            if (err_acc) { atomicAdd(&err_acc[2 * w], e); atomicAdd(&err_acc[2 * w + 1], (double)(n_obs + 1)); }
        }
    }
}

// ------------------------------------------------------------------------ packing
WinConst win_const(const pvio_b200_window *w) {
    WinConst C;
    memset(&C, 0, sizeof(C));
    memcpy(C.cam_q, w->cam_q_cs, 32); memcpy(C.cam_p, w->cam_p_cs, 24);
    memcpy(C.imu_q, w->imu_q_cs, 32); memcpy(C.imu_p, w->imu_p_cs, 24);
    memcpy(C.sic, w->sqrt_inv_cov, 32);
    C.fx = w->fx; C.fy = w->fy; C.cauchy_a = w->cauchy_a > 0 ? w->cauchy_a : 1.0; C.plane_sic = w->plane_sqrt_inv_cov;
    return C;
}

static int pack_window(Handle *h, int slot, const pvio_b200_window *w, const pvio_b200_state *s) {
    const int N = w->n_frames, M = w->n_landmarks, K = w->n_obs;
    if (slot < 0 || slot >= h->W) return fail(h, PVIO_B200_EINVAL, "slot out of range");
    if (N < 1 || N > h->Ncap || N > kMaxFrames || M > h->Mcap || K > h->Kcap || M < 0 || K < 0)
        return fail(h, PVIO_B200_EINVAL, "window exceeds the handle's capacity");
    if (!s->frames || (M > 0 && (!s->inv_depth || !w->lm_anchor || !w->lm_z_ref || !w->lm_obs_begin)) ||
        (K > 0 && (!w->obs_frame || !w->obs_z)))
        return fail(h, PVIO_B200_EINVAL, "null array in window / state");
    // every index array of the caller is range-checked here: bad indices would become device-side out-of-bounds accesses
    if (M > 0 && (w->lm_obs_begin[0] != 0 || w->lm_obs_begin[M] != K))
        return fail(h, PVIO_B200_EINVAL, "lm_obs_begin must start at 0 and end at n_obs");
    const bool inertial = w->use_inertial != 0;
    const int n_imu = inertial ? w->n_imu : 0, n_prior = inertial ? w->n_prior : 0;
    if (n_imu < 0 || n_prior < 0 || n_imu > h->Ncap || n_prior > h->Ncap || n_prior > N)
        return fail(h, PVIO_B200_EINVAL, "too many IMU / prior frames");
    for (int n = 0; n < n_imu; ++n) {
        const int i = w->imu_frame_i[n], j = w->imu_frame_j[n];
        if (i < 0 || i >= N || j < 0 || j >= N || i == j) return fail(h, PVIO_B200_EINVAL, "IMU factor with bad frame indices");
    }
    {
        unsigned seen = 0;
        for (int n = 0; n < n_prior; ++n) {
            const int f = w->prior_frames[n];
            if (f < 0 || f >= N || ((seen >> f) & 1u)) return fail(h, PVIO_B200_EINVAL, "prior_frames must be distinct window indices");
            seen |= 1u << f;
        }
    }
    // prior_S == NULL names the prior the marginaliser left in this slot's device arrays (pvio_b200_batch_marginalize,
    // pvio_b200_window_drop_victim); checked before anything of the slot is overwritten
    WinSlot &ws = h->slots[slot];
    if (n_prior > 0 && !w->prior_S && ws.prior_resident != n_prior)
        return fail(h, PVIO_B200_EINVAL, "prior_S == NULL: no device-resident prior of that size in this slot");
    if (w->n_plane_tracks < 0 || w->n_planes < 0 || w->n_planes > h->Pcap) return fail(h, PVIO_B200_EINVAL, "too many planes");
    if (w->n_plane_tracks > 0) {
        if (!w->pt_obs_begin || !w->pt_plane || !w->pt_obs_frame || !w->pt_obs_z || !w->plane_param || w->pt_obs_begin[0] != 0)
            return fail(h, PVIO_B200_EINVAL, "null / malformed plane-track arrays");
        for (int t = 0; t < w->n_plane_tracks; ++t) {
            const int len = w->pt_obs_begin[t + 1] - w->pt_obs_begin[t];
            if (len < 0 || len > kMaxFrames) return fail(h, PVIO_B200_EINVAL, "plane track too long / CSR offsets not monotone");
            if (w->pt_plane[t] < 0 || w->pt_plane[t] >= w->n_planes) return fail(h, PVIO_B200_EINVAL, "pt_plane out of range");
        }
        const int O = w->pt_obs_begin[w->n_plane_tracks];
        for (int i = 0; i < O; ++i)
            if (w->pt_obs_frame[i] < 0 || w->pt_obs_frame[i] >= N) return fail(h, PVIO_B200_EINVAL, "pt_obs_frame out of range");
    }
    if (n_imu > 0 || n_prior > 0 || inertial) TRY(ensure_inertial(h));
    // the slot's header and bookkeeping are replaced only once the whole window is accepted: batch_shape sizes the
    // launches and scatter_dx the downloads of the windows already uploaded by them, so a rejected window (e.g. one
    // that needs a 97th chunk) must leave them as they were
    WinHdr H;
    WinConst C;
    memset(&H, 0, sizeof(H));
    H.N = N; H.M = M; H.K = K; H.use_inertial = inertial ? 1 : 0;
    for (int f = 0; f < N; ++f) if (w->frame_fixed && w->frame_fixed[f]) H.fixed_mask |= 1 << f;
    C = win_const(w);
    // frames + origin (mean frame position keeps |x_l| ~ depth in the fp32 Jacobian arithmetic)
    double *fr = h->frames.slot(slot);
    memcpy(fr, s->frames, sizeof(double) * N * kFrameStride);
    double o[3] = {0, 0, 0};
    for (int f = 0; f < N; ++f) for (int k = 0; k < 3; ++k) o[k] += fr[f * kFrameStride + 4 + k];
    for (int k = 0; k < 3; ++k) C.origin[k] = o[k] / N;
    // landmarks sorted by anchor (the reference's first-visit order already is, bundle_adjustor.cpp:92-103)
    std::vector<int32_t> perm;
    bool sorted = true;
    for (int l = 0; l < M; ++l) {
        const int a = w->lm_anchor[l];
        if (a < 0 || a >= N) return fail(h, PVIO_B200_EINVAL, "landmark with bad anchor");
        if (l > 0 && a < w->lm_anchor[l - 1]) sorted = false;
    }
    if (!sorted) {
        perm.resize(M);
        std::iota(perm.begin(), perm.end(), 0);
        std::stable_sort(perm.begin(), perm.end(), [&](int a, int b) { return w->lm_anchor[a] < w->lm_anchor[b]; });
    }
    ObsRec *ob = h->obs.slot(slot);
    LmRec *lm = h->lms.slot(slot);
    double *rh = h->rho.slot(slot);
    int k_out = 0, nch = 0;
    for (int lp = 0; lp < M; ++lp) {
        const int l = sorted ? lp : perm[lp];
        const int a = w->lm_anchor[l];
        const int b0 = w->lm_obs_begin[l], b1 = w->lm_obs_begin[l + 1];
        const int n = b1 - b0;
        if (b0 < 0 || b1 > K || n < 0 || n >= kGroup) return fail(h, PVIO_B200_EINVAL, "landmark with bad observation range / too many observations");
        lm[lp].zrx = (float)w->lm_z_ref[2 * l];
        lm[lp].zry = (float)w->lm_z_ref[2 * l + 1];
        lm[lp].obs_begin = k_out;
        rh[lp] = s->inv_depth[l];
        // records in increasing frame order: the frame index lives in the landmark's mask, not in the record
        unsigned seen = 0;
        for (int k = b0; k < b1; ++k) {
            const int f = w->obs_frame[k];
            if (f <= a || f >= N || (seen >> f) & 1)
                return fail(h, PVIO_B200_EINVAL, "observation frames must be distinct and later than the anchor (Track::first_frame is the lowest id)");
            seen |= 1u << f;
        }
        if (k_out + n > h->Kcap) return fail(h, PVIO_B200_EINVAL, "observation table overflow");
        for (int k = b0; k < b1; ++k) {
            const int f = w->obs_frame[k];
            const int pos = k_out + __builtin_popcount(seen & ((1u << f) - 1u));
            ob[pos].zx = (float)w->obs_z[2 * k];
            ob[pos].zy = (float)w->obs_z[2 * k + 1];
        }
        k_out += n;
        lm[lp].meta = lm_meta(a, (w->lm_in_victim && w->lm_in_victim[l]) ? 1 : 0, n, seen);
        // chunks: <= kChunk landmarks of one anchor
        if (nch == 0 || (H.chunk_meta[nch - 1] >> 8) != a || (H.chunk_meta[nch - 1] & 0xff) == kChunk) {
            if (nch == kMaxChunks) return fail(h, PVIO_B200_EINVAL, "too many landmark chunks");
            H.chunk_begin[nch] = lp;
            H.chunk_meta[nch] = (a << 8);
            ++nch;
        }
        H.chunk_meta[nch - 1] += 1;
    }
    H.n_chunks = nch;
    H.K = k_out;
    // inertial part
    H.n_imu = n_imu;
    H.n_prior = n_prior;
    if (n_imu > 0 || n_prior > 0) {
        int32_t *ii = h->imu_idx.slot(slot);
        for (int n = 0; n < n_imu; ++n) { ii[2 * n] = w->imu_frame_i[n]; ii[2 * n + 1] = w->imu_frame_j[n]; }
        if (n_imu > 0) memcpy(h->imu_data.slot(slot), w->imu_data, sizeof(double) * n_imu * kImuStride);
        const size_t d = 15 * (size_t)n_prior;
        for (int n = 0; n < n_prior; ++n) h->prior_frames.slot(slot)[n] = w->prior_frames[n];
        if (d > 0 && w->prior_S) {          // a host prior replaces a device-resident one
            ws.prior_resident = 0;
            memcpy(h->prior_S.slot(slot), w->prior_S, sizeof(double) * d * d);   // dense d x d, row-major
            memcpy(h->prior_e.slot(slot), w->prior_e, sizeof(double) * d);
            memcpy(h->prior_x0.slot(slot), w->prior_state0, sizeof(double) * n_prior * kFrameStride);
        }
    }
    // planes
    H.n_planes = w->n_planes; H.n_ptracks = w->n_plane_tracks;
    if (H.n_ptracks > 0) {
        const int O = w->pt_obs_begin[H.n_ptracks];
        TRY(ensure_planes(h, H.n_ptracks, O));
        PlaneTables &p = h->planes;
        memcpy(p.plane_param.slot(slot), w->plane_param, sizeof(double) * 4 * H.n_planes);
        memcpy(p.pt_plane.slot(slot), w->pt_plane, sizeof(int32_t) * H.n_ptracks);
        memcpy(p.pt_begin.slot(slot), w->pt_obs_begin, sizeof(int32_t) * (H.n_ptracks + 1));
        memcpy(p.pt_frame.slot(slot), w->pt_obs_frame, sizeof(int32_t) * O);
        float *z = p.pt_z.slot(slot);
        for (int i = 0; i < 2 * O; ++i) z[i] = (float)w->pt_obs_z[i];
    }
    h->hdr.h[slot] = H;
    h->cst.h[slot] = C;
    ws.resident = false;                  // a packed slot is no longer a resident window
    ws.n_samples.clear();                 // and its IMU factors hold no samples
    ws.perm = std::move(perm);
    return 0;
}

// pinned staging -> device of window slots [w0, w0 + n)
template <typename T>
static int h2d(Handle *h, DevBuf<T> &b, int w0, int n, cudaStream_t st) {
    if (!b.d || !b.h || b.per == 0) return 0;
    CK(h, cudaMemcpyAsync(b.dslot(w0), b.slot(w0), b.per * n * sizeof(T), cudaMemcpyHostToDevice, st));
    return 0;
}

// Host -> device copy of windows [w0, w0 + n) on stream st, then the device-side preparation that is constant
// across the iterations of a solve: the frame-major table and Lambda = S^T S of the priors.
static int upload_range(Handle *h, int w0, int n, cudaStream_t st) {
    if (n < 1 || w0 < 0 || w0 + n > h->W) return fail(h, PVIO_B200_EINVAL, "bad window range");
    TRY(for_each_staged(h, [&](auto &b, bool prior) {
        if (!prior) return h2d(h, b, w0, n, st);
        for (int i = w0; i < w0 + n;) {      // a device-resident prior is never re-uploaded: copy the runs of the other slots
            if (h->slots[i].prior_resident) { ++i; continue; }
            int j = i;
            while (j < w0 + n && !h->slots[j].prior_resident) ++j;
            TRY(h2d(h, b, i, j - i, st));
            i = j;
        }
        return 0;
    }));
    bool any_prior = false;
    if (h->have_inertial) {
        for (int i = w0; i < w0 + n; ++i) any_prior |= h->hdr.h[i].n_prior > 0;
        if (any_prior) {
            prior_lambda_kernel<<<dim3(n, n < 64 ? 32 : 1), 256, 0, st>>>(h->hdr.d, h->prior_S.d, h->prior_L.d, h->Ncap, w0, nullptr);
            ++h->launches;
        }
    }
    FobsArgs fa = launch_args<FobsArgs>(h);
    fa.w0 = w0;
    fobs_build_kernel<<<n, 256, 0, st>>>(fa);
    ++h->launches;
    CK(h, cudaGetLastError());
    return 0;
}

static int upload(Handle *h, int n) {
    TRY(upload_range(h, 0, n, h->stream));
    h->n_uploaded = n;
    return 0;
}

int pack_and_upload(Handle *h, const pvio_b200_window *w, const pvio_b200_state *s) {
    TRY(pack_window(h, 0, w, s));
    return upload(h, 1);
}

// ------------------------------------------------------------------------ launches
struct StepCfg {
    double mu = -1.0;              // < 0: per-window WinCtrl::mu
    double beta = 1.0;             // truncated Gauss-Newton step: step = beta * dx_gn
    int apply = 0;                 // plain GN step: the candidate becomes the state
    int compute_scale = 1;
    int alias_bias = 0;
    int dump = 0;
    int loop = 0;                  // kernels obey the per-window trust-region flags
    int w0 = 0;                    // first window (sub-batch pipelining)
    int fork_aux = 0;              // latency path: the non-vision candidate cost runs beside the candidate's linearisation sweep
    cudaStream_t stream = nullptr; // nullptr: the handle's stream
    const int32_t *slots = nullptr;// device list of the windows of the sweeps (PipeArgs::slots); nullptr: [w0, w0 + n)
    int one_cta = 0;               // sweeps: one CTA per window whatever n (sweep_grid_x otherwise)
};

// what the windows [w0, w0 + n) need from the launch: worst case over the batch
struct BatchShape {
    int N = 1, M = 1, nfree = 1, D = 0;
    int N_inertial = 0;               // the largest window with motion states (0: none)
    bool inertial = false, planes = false;
    size_t solve_smem_full = 0, solve_smem_lean = 0;
};

static size_t solve_smem_one(const WinHdr &H, bool lean) {
    size_t D = (H.use_inertial ? 15 : 6) * (size_t)H.N;
    if (lean) {                       // the lean kernel drops constant frames from the system
        const int nfree = H.N - __builtin_popcount((unsigned)H.fixed_mask & ((1u << H.N) - 1u));
        if (nfree > 0) D = 6 * (size_t)nfree;
    }
    const size_t nb = (D + 3) / 4, Dp = nb * 4;
    const size_t np_ = (size_t)H.N * (H.N + 1) / 2;
    size_t scr = lean ? Dp + 10 * 36 + 36 : std::max<size_t>(Dp, 2 * np_ * 36 + (size_t)H.N * 36 + (size_t)H.N * 12);   // X blocks, X T_g, diagonal, gradients
    if (H.use_inertial) scr = std::max<size_t>(scr, 8 * 450 + 8 * 16 + 8 * 480 + 8 * 225);      // kImuRound factors: raw J, r; whitened [J | r]; their W
    if (H.n_prior > 0) scr = std::max<size_t>(scr, 3 * 15 * (size_t)H.n_prior + 9 * (size_t)H.n_prior + 8 * 225);   // + one 15 x 15 block per warp
    return sizeof(double) * ((nb + 1) * (nb + 2) / 2 * 18 + 4 * Dp + (size_t)H.N * 36 + scr);   // tiles of kTP = 18 doubles (ba_solve.cuh)
}

// named: windows k with named[k] == 0 are skipped (a solve of named resident slots: the others take no part in it)
static BatchShape batch_shape(Handle *h, int w0, int n, bool by_capacity, const int32_t *h_slots = nullptr,
                              const uint8_t *named = nullptr) {
    BatchShape b;
    for (int k = w0; k < w0 + n; ++k) {
        if (named && !named[k]) continue;
        const WinHdr &H = h->hdr.h[h_slots ? h_slots[k - w0] : k];
        b.N = std::max(b.N, H.N); b.M = std::max(b.M, H.M);
        const unsigned allm = (1u << H.N) - 1u, freem = ~(unsigned)H.fixed_mask & allm;
        b.nfree = std::max(b.nfree, __builtin_popcount(freem));
        b.inertial |= H.use_inertial != 0;
        if (H.use_inertial) b.N_inertial = std::max(b.N_inertial, H.N);
        b.planes |= H.n_ptracks > 0;
        b.solve_smem_full = std::max(b.solve_smem_full, solve_smem_one(H, false));
        b.solve_smem_lean = std::max(b.solve_smem_lean, solve_smem_one(H, true));
    }
    if (by_capacity) {                 // graph-cached launches: shapes depend on the frame counts (part of the graph key) only
        // sized for the most landmarks any window can hold (pack_window, batch_window: kMaxChunks chunks), not for the
        // capacity: a max_landmarks above that would ask the linearise and update sweeps for more shared memory than the
        // device has, although no window can use it
        b.M = std::min(h->Mcap, kMaxChunks * kChunk); b.nfree = b.N;
        WinHdr H;
        memset(&H, 0, sizeof(H));
        H.N = b.N;                     // a visual window of the largest size, an inertial one of the largest inertial size
        b.solve_smem_full = solve_smem_one(H, false);
        if (b.inertial) {
            H.N = b.N_inertial; H.use_inertial = 1; H.n_prior = b.N_inertial;
            b.solve_smem_full = std::max(b.solve_smem_full, solve_smem_one(H, false));
        }
    }
    return b;
}

static PipeArgs pipe_args(Handle *h, const StepCfg &c) {
    PipeArgs a = launch_args<PipeArgs>(h);
    a.compute_scale = c.compute_scale; a.mu_override = c.mu; a.w0 = c.w0; a.loop = c.loop; a.slots = c.slots;
    return a;
}

// CTAs per window of the sweeps: one once the batch fills the machine, otherwise a window is cut into row ranges
static int sweep_grid_x(Handle *h, int n) { return n * 2 < h->sm_count ? 16 : 1; }

// CTA shapes of the sweeps (fp32 pipeline): warps per CTA and resident CTAs per SM the register allocation targets,
// chosen by measurement on an H100 (cfg2, 4096 windows): 5 CTAs / SM for the linearise or the Schur sweep is 15-50 %
// slower per step, 3 for either is within the run-to-run spread; the results do not depend on them.  The update sweep at
// 8 CTAs / SM (64 registers) takes 0.352 ms per step, at 6 (80 registers) 0.361 ms (H100 SXM, 700 W power limit).
constexpr int kLinWarps = 4, kLinBlocks = 4;
// the linearise sweep may drop to 3 CTAs / SM for its fp64 shared-memory sums (lin_part_fits; 72 KB at cfg2, where 4 do
// not fit).  That instantiation is compiled for the 3 CTAs it gets (168 registers instead of 128) and spends the room on
// two rows in flight per lane (kLinPartRows); the one without the shared sums keeps one row at 4 CTAs / SM
constexpr int kLinPartMinBlocks = 3, kLinPartRows = 2;
constexpr int kSchurThreads = 128, kSchurBlocks = 4;
constexpr int kUpdWarps = 4, kUpdBlocks = 8;

template <typename real>
static size_t schur_launch_smem(int N, int nfree) { return schur_smem_bytes<real>(N, kSchurThreads, nfree); }

#define LAUNCH_CK(h, what)                                                                        \
    do {                                                                                          \
        cudaError_t e__ = cudaGetLastError();                                                     \
        if (e__ != cudaSuccess) return fail((h), PVIO_B200_ECUDA, "launch of " what, e__);        \
    } while (0)

// linearise + Schur stage of windows [w0, w0 + n)
// zeroes the direct / reduced system of the buffer set a sweep is about to accumulate into with atomics (several CTAs
// per window: the latency path)
static __global__ void zero_system_kernel(PipeArgs a_in, int npairs_cap) {
    PipeArgs a = a_in;
    const int w = a.slots ? a.slots[blockIdx.x] : blockIdx.x + a.w0;
    const int bsel = pipe_buffer(a, w);
    if (bsel < 0) return;
    pipe_select(a, bsel);
    double *Hred = a.Hred + (size_t)w * npairs_cap * 36, *Hdd = a.Hdd + (size_t)w * a.Ncap * 36;
    double *gdir = a.gdir + (size_t)w * a.Ncap * 6, *gred = a.gred + (size_t)w * a.Ncap * 6;
    for (int i = threadIdx.x; i < npairs_cap * 36; i += blockDim.x) Hred[i] = 0.0;
    for (int i = threadIdx.x; i < a.Ncap * 36; i += blockDim.x) Hdd[i] = 0.0;
    for (int i = threadIdx.x; i < a.Ncap * 6; i += blockDim.x) { gdir[i] = 0.0; gred[i] = 0.0; }
    if (threadIdx.x == 0) a.cost_vis[w] = 0.0;
}

// Whether a linearise CTA that owns its window keeps the per-landmark (j.j, j.r) sums in shared memory (PipeArgs::lm_part)
// at this shape: only when the larger layout fits and leaves at least min(kLinPartMinBlocks, the CTAs / SM without it)
// resident (occupancy API: registers and shared memory), so that e.g. a large max_landmarks falls back to the jr records
// instead of failing or losing more occupancy.  k_part / k_plain: the instantiations launched with and without the
// shared sums (the same kernel in fp64), each asked about with its own layout.
template <typename real>
static bool lin_part_fits(Handle *h, const void *k_part, const void *k_plain, int N, int Mp) {
    const auto key = std::make_tuple((int)sizeof(real), N, Mp);
    auto it = h->lin_part.find(key);
    if (it != h->lin_part.end()) return it->second;
    const size_t with = lin_smem_bytes<real>(N, Mp, kLinWarps, true), without = lin_smem_bytes<real>(N, Mp, kLinWarps, false);
    int nb_with = 0, nb_without = 0;
    bool ok = false;
    if ((int)with <= h->smem_lim) {
        const cudaError_t e1 = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_with, k_part, kLinWarps * 32, with);
        const cudaError_t e2 = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb_without, k_plain, kLinWarps * 32, without);
        if (e1 != cudaSuccess || e2 != cudaSuccess) cudaGetLastError();      // a failed query only means: keep jr
        else ok = nb_with >= 1 && nb_with >= std::min(nb_without, kLinPartMinBlocks);
    }
    h->lin_part[key] = ok;
    return ok;
}

// linearise sweep (+ per-landmark completion as its own launch when several CTAs share a window).  spec: the
// speculative sweep of the trust-region loop over the CANDIDATE, into the window's other buffer set (ba_tr.cuh).
static int launch_lin(Handle *h, int n, const StepCfg &c, const BatchShape &b, bool loss, bool victim_only, bool spec) {
    cudaStream_t st = c.stream ? c.stream : h->stream;
    const int gx = c.one_cta ? 1 : sweep_grid_x(h, n);
    PipeArgs a = pipe_args(h, c);
    a.victim_only = victim_only ? 1 : 0;
    a.spec = spec ? 1 : 0;
    if (gx > 1) {
        zero_system_kernel<<<n, 256, 0, st>>>(a, h->Ncap * (h->Ncap + 1) / 2);
        ++h->launches;
        LAUNCH_CK(h, "zero_system_kernel");
    }
    const int Mp = (b.M + 31) & ~31;
    if (!h->hs_double) {
        if (!loss) return fail(h, PVIO_B200_EINVAL, "the loss-free sweep runs in fp64");
        auto k_part = lin_obs_kernel<true, float, kLinWarps, kLinPartMinBlocks, kLinPartRows>;
        auto k_plain = lin_obs_kernel<true, float, kLinWarps, kLinBlocks>;
        a.lm_part = gx == 1 && lin_part_fits<float>(h, (const void *)k_part, (const void *)k_plain, b.N, Mp) ? 1 : 0;
        auto k = a.lm_part ? k_part : k_plain;
        k<<<dim3(gx, n), kLinWarps * 32, lin_smem_bytes<float>(b.N, Mp, kLinWarps, a.lm_part), st>>>(a);
        LAUNCH_CK(h, "lin_obs_kernel<float>");
        if (gx > 1) { lm_finish_kernel<float><<<dim3((b.M + 127) / 128, n), 128, 0, st>>>(a); ++h->launches; LAUNCH_CK(h, "lm_finish_kernel<float>"); }
    } else {
        auto k = loss ? lin_obs_kernel<true, double, kLinWarps, 2> : lin_obs_kernel<false, double, kLinWarps, 2>;
        a.lm_part = gx == 1 && lin_part_fits<double>(h, (const void *)k, (const void *)k, b.N, Mp) ? 1 : 0;
        k<<<dim3(gx, n), kLinWarps * 32, lin_smem_bytes<double>(b.N, Mp, kLinWarps, a.lm_part), st>>>(a);
        LAUNCH_CK(h, "lin_obs_kernel<double>");
        if (gx > 1) { lm_finish_kernel<double><<<dim3((b.M + 127) / 128, n), 128, 0, st>>>(a); ++h->launches; LAUNCH_CK(h, "lm_finish_kernel<double>"); }
    }
    ++h->launches;
    return 0;
}

static int launch_schur(Handle *h, int n, const StepCfg &c, const BatchShape &b, bool victim_only) {
    cudaStream_t st = c.stream ? c.stream : h->stream;
    const int gx = c.one_cta ? 1 : sweep_grid_x(h, n);
    PipeArgs a = pipe_args(h, c);
    a.victim_only = victim_only ? 1 : 0;
    const int sgx = std::min(gx, std::max(1, (b.M + kSlab - 1) / kSlab));
    if (!h->hs_double) {
        schur_kernel<float, kSchurThreads, kSchurBlocks><<<dim3(sgx, n), kSchurThreads, schur_launch_smem<float>(b.N, b.nfree), st>>>(a);
        LAUNCH_CK(h, "schur_kernel<float>");
    } else {
        schur_kernel<double, kSchurThreads, 1><<<dim3(sgx, n), kSchurThreads, schur_launch_smem<double>(b.N, b.nfree), st>>>(a);
        LAUNCH_CK(h, "schur_kernel<double>");
    }
    ++h->launches;
    return 0;
}

// the linearise + Schur stage at the state; its two halves are timed by events when it is the plain batched step
static int run_linearize(Handle *h, int n, const StepCfg &c, const BatchShape &b, bool loss = true, bool victim_only = false) {
    cudaStream_t st = c.stream ? c.stream : h->stream;
    if (h->kev.empty()) {
        h->kev.resize(3 * 256);
        for (auto &e : h->kev) CK(h, cudaEventCreate(&e));
    }
    const int slot = (h->kev_count % 256) * 3;
    const bool timed = !h->capturing && !c.loop && !c.stream;   // stage times are a property of the plain batched step
    if (timed) CK(h, cudaEventRecord(h->kev[slot], st));
    TRY(launch_lin(h, n, c, b, loss, victim_only, false));
    if (timed) CK(h, cudaEventRecord(h->kev[slot + 1], st));
    TRY(launch_schur(h, n, c, b, victim_only));
    if (timed) { CK(h, cudaEventRecord(h->kev[slot + 2], st)); ++h->kev_count; }
    return 0;
}

int run_marg_vision(Handle *h, int n, const int32_t *h_slots, const int32_t *d_slots) {
    StepCfg c;
    c.mu = 0.0; c.compute_scale = 1; c.slots = d_slots;
    const BatchShape b = batch_shape(h, 0, n, false, h_slots);
    return run_linearize(h, n, c, b, false, true);
}

size_t cov_smem_bytes(const WinHdr &H) { return solve_smem_one(H, false); }

static CovArgs cov_args(Handle *h, const CovLaunch &L) {
    CovArgs a;
    static_cast<SolveArgs &>(a) = launch_args<SolveArgs>(h);
    a.alias_bias = 0; a.Hfull = nullptr; a.gfull = nullptr; a.compute_scale = 1; a.w0 = 0; a.mu_override = 0.0; a.loop = 0;
    a.recs = L.recs; a.frames = L.frames; a.lms = L.lms; a.n_lm = L.n_lm;
    a.cov = L.cov; a.var = L.var; a.status = L.status; a.sig = L.sig; a.sig_xi = L.sig_xi;
    return a;
}

int run_cov_system(Handle *h, int n, const int32_t *h_slots, const int32_t *d_slots, const CovLaunch &L) {
    // the solve's linearisation at the state (with the loss, either pipeline), mu = 0 in the landmark pivots; one CTA
    // per window so that the launch count does not depend on n
    StepCfg c;
    c.mu = 0.0; c.compute_scale = 1; c.slots = d_slots; c.one_cta = 1;
    const BatchShape b = batch_shape(h, 0, n, false, h_slots);
    TRY(launch_lin(h, n, c, b, true, false, false));
    TRY(launch_schur(h, n, c, b, false));
    const CovArgs a = cov_args(h, L);
    size_t smem = 0;
    for (int i = 0; i < n; ++i) smem = std::max(smem, cov_smem_bytes(h->hdr.h[h_slots[i]]));
    cov_kernel<<<n, 256, smem, h->stream>>>(a);
    LAUNCH_CK(h, "cov_kernel");
    ++h->launches;
    return 0;
}

int run_covariance(Handle *h, int n, const int32_t *h_slots, const int32_t *d_slots, const CovLaunch &L) {
    TRY(run_cov_system(h, n, h_slots, d_slots, L));
    const CovArgs a = cov_args(h, L);
    const int blocks = std::max(1, (L.n_lm + kCovLmWarps - 1) / kCovLmWarps);
    if (h->hs_double) cov_lm_kernel<double><<<blocks, 32 * kCovLmWarps, 0, h->stream>>>(a);
    else cov_lm_kernel<float><<<blocks, 32 * kCovLmWarps, 0, h->stream>>>(a);
    LAUNCH_CK(h, "cov_lm_kernel");
    ++h->launches;
    return 0;
}

static int run_solve(Handle *h, int n, const StepCfg &c, const BatchShape &b) {
    SolveArgs a = launch_args<SolveArgs>(h);
    a.alias_bias = c.alias_bias;
    a.Hfull = c.dump ? h->Hfull.d : nullptr; a.gfull = c.dump ? h->gfull.d : nullptr;
    a.compute_scale = c.compute_scale; a.mu_override = c.mu; a.w0 = c.w0; a.loop = c.loop;
    cudaStream_t st = c.stream ? c.stream : h->stream;
    // visual-only batches: the lean kernel (no IMU / prior / plane code, no full staging), a narrow CTA
    // per window so that many windows are resident per SM; otherwise the full kernel with a wide CTA
    const bool visual = n >= 64 && !b.inertial && !b.planes && b.solve_smem_lean <= 48 * 1024;
    const size_t smem = visual ? b.solve_smem_lean : b.solve_smem_full;
    if (smem > 220 * 1024) return fail(h, PVIO_B200_EINVAL, "reduced system too large for shared memory");
    if (visual) solve_kernel_visual<<<n, 64, smem, st>>>(a);
    else solve_kernel<<<n, 256, smem, st>>>(a);
    ++h->launches;
    LAUNCH_CK(h, "solve_kernel");
    return 0;
}

static CostArgs cost_args(Handle *h, const StepCfg &c) {
    CostArgs k = launch_args<CostArgs>(h);
    k.alias_bias = c.alias_bias; k.w0 = c.w0; k.loop = c.loop; k.apply = c.apply; k.beta = c.beta;
    return k;
}

static UpdArgs upd_args(Handle *h, const StepCfg &c) {
    UpdArgs u = launch_args<UpdArgs>(h);
    u.mu_override = c.mu; u.w0 = c.w0; u.step_a = 0.0; u.step_b = c.beta; u.loop = c.loop;
    return u;
}

template <int kMode>
static int launch_update(Handle *h, int n, const StepCfg &c, const BatchShape &b, int gx) {
    cudaStream_t st = c.stream ? c.stream : h->stream;
    const UpdArgs u = upd_args(h, c);
    const int Mp = (b.M + 31) & ~31;
    constexpr int kW = kUpdWarps;
    constexpr int kB = 4, kBf = kUpdBlocks;
    if (kMode == 1 && n * 2 < h->sm_count) {        // latency path: one wide CTA per window for the back-substitution
        if (!h->hs_double) update_obs_kernel<float, 8, 2, 1><<<dim3(gx, n), 256, upd_smem_bytes<float>(b.N, Mp, 8), st>>>(u);
        else update_obs_kernel<double, 8, 2, 1><<<dim3(gx, n), 256, upd_smem_bytes<double>(b.N, Mp, 8), st>>>(u);
    }
    else if (!h->hs_double) update_obs_kernel<float, kW, kBf, kMode><<<dim3(gx, n), kW * 32, upd_smem_bytes<float>(b.N, Mp, kW), st>>>(u);
    else update_obs_kernel<double, kW, kB, kMode><<<dim3(gx, n), kW * 32, upd_smem_bytes<double>(b.N, Mp, kW), st>>>(u);
    ++h->launches;
    LAUNCH_CK(h, "update_obs_kernel");
    return 0;
}

// part 0: cost + decision in one launch; 1: cost only, on stream `on`; 2: decision only (aux_cost_kernel)
static int launch_aux_cost(Handle *h, int n, const StepCfg &c, const BatchShape &b, int part = 0, cudaStream_t on = nullptr) {
    cudaStream_t st = on ? on : (c.stream ? c.stream : h->stream);
    const CostArgs k = cost_args(h, c);
    // inertial windows: 8 warps share the prior's S r0 product; reprojection-only batches only need the acceptance copy
    const int threads = (b.inertial && part != 2) ? 256 : 64;
    const size_t smem = sizeof(double) * 2 * 15 * kMaxFrames;
    if (part == 1) aux_cost_kernel<1><<<n, threads, smem, st>>>(k);
    else if (part == 2) aux_cost_kernel<2><<<n, threads, smem, st>>>(k);
    else aux_cost_kernel<0><<<n, threads, smem, st>>>(k);
    ++h->launches;
    LAUNCH_CK(h, "aux_cost_kernel");
    return 0;
}

// One plain Gauss-Newton iteration (fixed mu, step beta * dx_gn): linearise, Schur, solve (which also clears the
// window's step scalars), back-substitution + candidate in one sweep, non-vision cost + optional acceptance.  5 launches.
static int run_gn_step(Handle *h, int n, const StepCfg &c, const BatchShape &b) {
    TRY(run_linearize(h, n, c, b));
    TRY(run_solve(h, n, c, b));
    TRY(launch_update<0>(h, n, c, b, sweep_grid_x(h, n)));
    TRY(launch_aux_cost(h, n, c, b));
    return 0;
}

// The second stream of the split step shares the handle's aux stream (the latency path only captures through it)
static int aux_stream(Handle *h) {
    if (h->stream_aux) return 0;
    CK(h, cudaStreamCreateWithFlags(&h->stream_aux, cudaStreamNonBlocking));
    CK(h, cudaEventCreateWithFlags(&h->ev_aux_fork, cudaEventDisableTiming));
    CK(h, cudaEventCreateWithFlags(&h->ev_aux_join, cudaEventDisableTiming));
    return 0;
}

// Sub-batches of the plain batched step (run_gn_step_split).  Each sweep launch drains the whole grid before the next
// sweep of the same windows may start: a sweep's last wave and the next sweep's first CTAs leave most SMs idle.  Cutting
// the batch into contiguous sub-batches on two streams lets one sub-batch's CTAs fill what the other's tail leaves.
// Measured on an H100 SXM (700 W, cfg2, DESIGN §9): 2 parts take 1.253 instead of 1.345 ms per step at 4096 windows,
// 0.653 instead of 0.732 at 2048 and 0.372 instead of 0.386 at 1024; 4 parts are no faster at 4096 and slower below;
// 3 parts are slower everywhere (two of them share a stream, so that stream's sweeps wait for each other).
constexpr int kStepParts = 2, kStepPartsMax = 4, kStepSplitMinPerSm = 7;

static int gn_step_parts(Handle *h, int n) {
    // every part keeps the launch shapes of the whole batch: one CTA per window in the sweeps (sweep_grid_x) and the
    // lean solve kernel (run_solve) -- at least max(SMs, 64) windows
    const int most = std::min(kStepPartsMax, n / std::max(h->sm_count, 64));
    const int want = h->step_parts > 0 ? h->step_parts : (n >= kStepSplitMinPerSm * h->sm_count ? kStepParts : 1);
    return std::max(1, std::min(want, most));
}

// run_gn_step over `parts` contiguous sub-batches of equal size (+-1), on the handle's stream (even parts) and the aux
// stream (odd parts), issued breadth first: lin(0), lin(1), ..., Schur(0), Schur(1), ...  Every window runs the same
// kernels with the same arguments as in the unsplit step (b is the whole batch's shape), so the results are bit-identical.  The aux stream
// joins the handle's stream before the call returns.  The stage times (last_kernel_ms) stay those of the whole batch:
// from before the first linearise launch to the end of the last linearise (Schur) sweep of any sub-batch, taken on a
// third stream that waits for both compute streams, so that no compute launch waits for a timing event.
static int run_gn_step_split(Handle *h, int n, const StepCfg &c0, const BatchShape &b, int parts) {
    TRY(aux_stream(h));
    if (!h->stream_mark) {
        CK(h, cudaStreamCreateWithFlags(&h->stream_mark, cudaStreamNonBlocking));
        for (auto &e : h->ev_stage) CK(h, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    if (h->kev.empty()) {
        h->kev.resize(3 * 256);
        for (auto &e : h->kev) CK(h, cudaEventCreate(&e));
    }
    const int slot = (h->kev_count % 256) * 3;
    cudaStream_t st[2] = {h->stream, h->stream_aux};
    int w0[kStepPartsMax + 1];
    for (int k = 0; k <= parts; ++k) w0[k] = (int)((int64_t)n * k / parts);
    StepCfg c[kStepPartsMax];
    for (int k = 0; k < parts; ++k) { c[k] = c0; c[k].w0 = w0[k]; c[k].stream = st[k & 1]; }
    auto m = [&](int k) { return w0[k + 1] - w0[k]; };
    auto mark = [&](cudaEvent_t e) {         // e: once every launch so far on both streams has finished
        for (int s = 0; s < 2; ++s) {
            CK(h, cudaEventRecord(h->ev_stage[s], st[s]));
            CK(h, cudaStreamWaitEvent(h->stream_mark, h->ev_stage[s], 0));
        }
        CK(h, cudaEventRecord(e, h->stream_mark));
        return 0;
    };
    CK(h, cudaEventRecord(h->kev[slot], h->stream));
    CK(h, cudaEventRecord(h->ev_aux_fork, h->stream));
    CK(h, cudaStreamWaitEvent(h->stream_aux, h->ev_aux_fork, 0));
    for (int k = 0; k < parts; ++k) TRY(launch_lin(h, m(k), c[k], b, true, false, false));
    TRY(mark(h->kev[slot + 1]));
    for (int k = 0; k < parts; ++k) TRY(launch_schur(h, m(k), c[k], b, false));
    TRY(mark(h->kev[slot + 2]));
    ++h->kev_count;
    for (int k = 0; k < parts; ++k) TRY(run_solve(h, m(k), c[k], b));
    for (int k = 0; k < parts; ++k) TRY(launch_update<0>(h, m(k), c[k], b, 1));
    for (int k = 0; k < parts; ++k) TRY(launch_aux_cost(h, m(k), c[k], b));
    CK(h, cudaEventRecord(h->ev_aux_join, h->stream_aux));
    CK(h, cudaStreamWaitEvent(h->stream, h->ev_aux_join, 0));
    CK(h, cudaStreamWaitEvent(h->stream, h->kev[slot + 2], 0));   // last_kernel_ms synchronises the handle's stream only
    return 0;
}

// One iteration of the device-side trust-region loop (ba_tr.cuh): 8 launches (9 in the first body), no host decision.
// The linearisation of the STATE is launched in the first body only: afterwards the state's linearisation is either the
// accepted candidate's (buffer swap) or still valid (rejected step), and the one case that invalidates it -- a failed
// linear solve, retried with mu * 10 -- is relinearised by the candidate sweep of the same body (pipe_buffer).
static int iteration_body(Handle *h, int n, const StepCfg &c, const BatchShape &b, bool first) {
    cudaStream_t st = c.stream ? c.stream : h->stream;
    if (first) TRY(launch_lin(h, n, c, b, true, false, false));
    TRY(launch_schur(h, n, c, b, false));
    TRY(run_solve(h, n, c, b));
    TRY(launch_update<1>(h, n, c, b, 1));
    jv_vision_kernel<<<dim3(sweep_grid_x(h, n), n), kLinThreads, 0, st>>>(upd_args(h, c));
    LAUNCH_CK(h, "jv_vision_kernel");
    jv_aux_kernel<<<n, 64, sizeof(double) * 15 * kMaxFrames, st>>>(cost_args(h, c));
    LAUNCH_CK(h, "jv_aux_kernel");
    h->launches += 2;
    TRY(launch_update<2>(h, n, c, b, 1));
    const bool fork = c.fork_aux && (b.inertial || b.planes);   // the candidate's IMU / prior / plane cost on a parallel branch
    if (fork) {
        CK(h, cudaEventRecord(h->ev_aux_fork, st));
        CK(h, cudaStreamWaitEvent(h->stream_aux, h->ev_aux_fork, 0));
        TRY(launch_aux_cost(h, n, c, b, 1, h->stream_aux));
        CK(h, cudaEventRecord(h->ev_aux_join, h->stream_aux));
    }
    TRY(launch_lin(h, n, c, b, true, false, true));      // the candidate's linearisation: its cost decides, its Jacobians stay
    if (fork) {
        CK(h, cudaStreamWaitEvent(st, h->ev_aux_join, 0));
        TRY(launch_aux_cost(h, n, c, b, 2));
    } else {
        TRY(launch_aux_cost(h, n, c, b));
    }
    return 0;
}

// The whole trust-region solve of the uploaded windows [w0, w0 + n) on stream st: init + max_iter (+ spare) identical
// bodies.  For the latency path (a few windows from window 0) the sequence is captured once into a CUDA graph keyed by
// (n, max_iter, flags) with capacity-sized launch shapes, and replayed: ONE launch per solve, no device -> host traffic
// inside.  The graphs bake in w0 = 0.
static int run_solve_loop(Handle *h, const SolveOptions &o, int w0, int n, cudaStream_t st, bool init = true,
                          const uint8_t *named = nullptr) {
    StepCfg c;
    c.mu = -1.0; c.loop = 1; c.alias_bias = o.alias_bias; c.compute_scale = 0; c.w0 = w0; c.stream = st;
    const bool graphable = w0 == 0 && n * 2 < h->sm_count;
    const BatchShape b = batch_shape(h, w0, n, graphable, nullptr, named);
    const int bodies = o.max_iter + 2;               // spare bodies absorb retries of a failed linear solve (mu *= 10)
    if (init) {
        init_ctrl_kernel<<<n, 32, 0, st>>>(h->ctrl.d, 1e-8, o.radius0, o.max_iter, o.max_time, w0);
        ++h->launches;
        LAUNCH_CK(h, "init_ctrl_kernel");
    }
    if (!graphable) {
        for (int it = 0; it < bodies; ++it) TRY(iteration_body(h, n, c, b, it == 0));
        return 0;
    }
    const Handle::GraphKey key(1, n, o.max_iter, (o.alias_bias ? 1 : 0) | (b.inertial ? 2 : 0) | (b.planes ? 4 : 0) | (h->hs_double ? 8 : 0) | (b.N << 4) | (b.N_inertial << 9));
    auto it = h->graphs.find(key);
    if (it == h->graphs.end()) {
        if (h->graphs.size() >= 16) drop_graphs(h);
        const int64_t l0 = h->launches;
        cudaGraph_t g = nullptr;
        cudaGraphExec_t ge = nullptr;
        TRY(aux_stream(h));
        c.fork_aux = 1;                // a second branch of the graph (captured through h->stream_aux)
        CK(h, cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
        h->capturing = true;
        int rc = 0;
        for (int i = 0; i < bodies && rc == 0; ++i) rc = iteration_body(h, n, c, b, i == 0);
        h->capturing = false;
        const cudaError_t e = cudaStreamEndCapture(st, &g);
        if (rc != 0) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) return fail(h, PVIO_B200_ECUDA, "cudaStreamEndCapture", e);
        CK(h, cudaGraphInstantiate(&ge, g, 0));
        cudaGraphDestroy(g);
        const int nl = (int)(h->launches - l0);
        h->launches = l0;
        it = h->graphs.emplace(key, std::make_pair(ge, nl)).first;
    }
    CK(h, cudaGraphLaunch(it->second.first, st));
    h->launches += it->second.second;
    return 0;
}

static int run_postpass(Handle *h, int n, bool want_flags, double *err_acc, const int32_t *slots = nullptr) {
    postpass_kernel<<<dim3(n * 2 < h->sm_count ? 8 : 1, n), 256, 0, h->stream>>>(
        h->hdr.d, h->cst.d, h->obs.d, h->lms.d, h->rho.d, h->frames.d, want_flags ? h->valid.d : nullptr,
        want_flags ? h->quality.d : nullptr, err_acc, h->Ncap, h->Mcap, h->Kcap, 0, slots);
    ++h->launches;
    CK(h, cudaGetLastError());
    return 0;
}

int run_postpass_slots(Handle *h, int n, const int32_t *slots) { return run_postpass(h, n, true, nullptr, slots); }

int run_named_solve(Handle *h, const pvio_b200_options *opt, int n, const uint8_t *named, const uint8_t *named_h) {
    const SolveOptions o = solve_options(opt);
    init_ctrl_kernel<<<n, 32, 0, h->stream>>>(h->ctrl.d, 1e-8, o.radius0, o.max_iter, o.max_time, 0, named);
    ++h->launches;
    LAUNCH_CK(h, "init_ctrl_kernel");
    return run_solve_loop(h, o, 0, n, h->stream, false, named_h);
}

int launch_layout_tail(Handle *h, const int32_t *slots, int n, bool prior) {
    if (prior) {
        prior_lambda_kernel<<<dim3(n, n < 64 ? 32 : 1), 256, 0, h->stream>>>(h->hdr.d, h->prior_S.d, h->prior_L.d, h->Ncap, 0, slots);
        ++h->launches;
    }
    FobsArgs fa = launch_args<FobsArgs>(h);
    fa.slots = slots;
    fobs_build_kernel<<<n, 256, 0, h->stream>>>(fa);
    ++h->launches;
    CK(h, cudaGetLastError());
    return 0;
}

// per-landmark values of the packed window in slot i -> the caller's landmark order
template <typename T>
static void unpermute(const Handle *h, int i, T *dst, const T *src) {
    const std::vector<int32_t> &perm = h->slots[i].perm;
    const int M = h->hdr.h[i].M;
    if (perm.empty()) memcpy(dst, src, sizeof(T) * M);
    else for (int lp = 0; lp < M; ++lp) dst[perm[lp]] = src[lp];
}

// pinned staging -> caller arrays (landmark order un-permuted), windows [w0, w0 + n)
static int scatter_dx(Handle *h, int w0, int n, double *dx, int64_t dx_stride, double *costs) {
    for (int i = w0; i < w0 + n; ++i) {
        if (dx) {
            const int N = h->hdr.h[i].N;
            double *o = dx + (size_t)i * dx_stride;
            memcpy(o, h->dx_pose.slot(i), sizeof(double) * N * 15);
            unpermute(h, i, o + N * 15, h->dx_lm.slot(i));
        }
        if (costs) { costs[2 * i] = h->ctrl.h[i].cost; costs[2 * i + 1] = h->ctrl.h[i].cand_cost; }
        if (h->ctrl.h[i].solve_failed) return fail(h, PVIO_B200_ENUMERIC, "reduced system not positive definite");
    }
    return 0;
}

// device array src -> pinned array dst (same slot stride) of window slots [w0, w0 + n) on stream st (async)
template <typename T>
static int d2h(Handle *h, DevBuf<T> &dst, const DevBuf<T> &src, int w0, int n, cudaStream_t st) {
    CK(h, cudaMemcpyAsync(dst.slot(w0), src.dslot(w0), sizeof(T) * src.per * n, cudaMemcpyDeviceToHost, st));
    return 0;
}

// device -> host of the steps + summaries of windows [w0, w0 + n) on stream st (async)
static int download_dx_async(Handle *h, int w0, int n, cudaStream_t st) {
    TRY(d2h(h, h->dx_pose, h->dx_pose, w0, n, st));
    TRY(d2h(h, h->dx_lm, h->dx_lm, w0, n, st));
    return d2h(h, h->ctrl, h->ctrl, w0, n, st);
}

static int download_dx(Handle *h, int n, double *dx, int64_t dx_stride, double *costs) {
    if (n < 1 || n > h->W) return fail(h, PVIO_B200_EINVAL, "bad window count");
    TRY(download_dx_async(h, 0, n, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    return scatter_dx(h, 0, n, dx, dx_stride, costs);
}

// device -> host of the solved state + summaries of windows [w0, w0 + n) on stream st (async)
static int download_state_async(Handle *h, int w0, int n, cudaStream_t st) {
    TRY(d2h(h, h->frames_out, h->frames, w0, n, st));
    TRY(d2h(h, h->rho_out, h->rho, w0, n, st));
    return d2h(h, h->ctrl, h->ctrl, w0, n, st);
}

void fill_summary(const WinCtrl &c, pvio_b200_summary *sm) {
    memset(sm, 0, sizeof(*sm));
    sm->iterations = c.iteration; sm->accepted_steps = c.accepted; sm->termination = c.termination; sm->usable = c.usable;
    sm->initial_cost = c.initial_cost; sm->final_cost = c.cost; sm->final_radius = c.radius; sm->final_mu = c.mu;
}

static void scatter_state(Handle *h, int i, double *frames, double *inv_depth) {
    if (frames) memcpy(frames, h->frames_out.slot(i), sizeof(double) * h->hdr.h[i].N * kFrameStride);
    if (inv_depth) unpermute(h, i, inv_depth, h->rho_out.slot(i));
}

// pinned landing area -> caller arrays of windows [w0, w0 + n): states (landmark order un-permuted) and summaries
static void scatter_states(Handle *h, int w0, int n, double *frames, int64_t frames_stride, double *inv_depth,
                           int64_t inv_depth_stride, pvio_b200_summary *summaries) {
    for (int i = w0; i < w0 + n; ++i) {
        scatter_state(h, i, frames ? frames + (size_t)i * frames_stride : nullptr, inv_depth ? inv_depth + (size_t)i * inv_depth_stride : nullptr);
        if (summaries) fill_summary(h->ctrl.h[i], &summaries[i]);
    }
}

// sub-batch schedule of the pipelined host paths: small batches first and last (the first upload and the last
// kernels + download are the only parts of the pipeline that nothing overlaps), kPipeChunk-window batches in between
static constexpr int kPipeStreams = 6;     // sub-batches in flight on the SMs at once (each alone is latency-bound: one wave)
static constexpr int kPipeChunk = 512;
static std::vector<int> sub_batches(int n) {
    std::vector<int> sizes;
    if (n < 1024) { sizes.push_back(n); return sizes; }
    int mid = n - 2 * (128 + 256);
    sizes.push_back(128); sizes.push_back(256);
    while (mid > 0) { const int m = std::min(kPipeChunk, mid); sizes.push_back(m); mid -= m; }
    sizes.push_back(256); sizes.push_back(128);
    return sizes;
}

static int ensure_pipeline_streams(Handle *h, int nsub) {
    if (!h->stream_up) {
        CK(h, cudaStreamCreateWithFlags(&h->stream_up, cudaStreamNonBlocking));
        CK(h, cudaStreamCreateWithFlags(&h->stream_down, cudaStreamNonBlocking));
    }
    while ((int)h->ev_up.size() < nsub) {
        cudaEvent_t a, b, c_;
        CK(h, cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
        CK(h, cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
        CK(h, cudaEventCreateWithFlags(&c_, cudaEventDisableTiming));
        h->ev_up.push_back(a); h->ev_done.push_back(b); h->ev_down.push_back(c_);
    }
    if (h->stream_c.empty()) {
        h->stream_c.resize(kPipeStreams);
        for (auto &st : h->stream_c) CK(h, cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
        CK(h, cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    }
    return 0;
}

// The entry points that take packed windows (what: the one called) refuse a range [0, n) that holds a resident window.
static int check_packed(Handle *h, int n, const char *what) {
    for (int i = 0; i < std::min(n, h->W); ++i)
        if (h->slots[i].resident)
            return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": the range holds a resident window (pvio_b200_batch_window_*)").c_str());
    return 0;
}

// Upload, work and download of windows [0, n) with HOST buffers.  Below 1024 windows: one upload, the work and one
// download on the handle's stream.  Large batches are cut into sub-batches and pipelined: sub-batch i is uploaded on
// the copy stream, worked on compute stream i % kPipeStreams (a sub-batch is at most one wave of CTAs, so alone it runs
// at the latency of its kernel chain; several in flight fill the SMs) and downloaded on the second copy stream, so the
// host -> device copy of sub-batch i+1 overlaps the kernels of sub-batch i and the device -> host copy of sub-batch i-1
// (PCIe is full duplex) and the call costs max(copy, compute) instead of their sum; the windows of different sub-batches
// share nothing on the device.  Each sub-batch is scattered as soon as it has landed, while the GPU works on the later ones.
//   work(w0, m, st)     enqueues the kernels of windows [w0, w0 + m) on st (nullptr: the handle's stream)
//   download(w0, m, st) enqueues their device -> host copies into the pinned staging on st
//   scatter(w0, m)      hands the landed results to the caller
template <typename Work, typename Download, typename Scatter>
static int run_host_pipeline(Handle *h, int n, const char *what, Work work, Download download, Scatter scatter) {
    if (n < 1 || n > h->W) return fail(h, PVIO_B200_EINVAL, "bad window count");
    TRY(check_packed(h, n, what));
    const std::vector<int> sizes = sub_batches(n);
    const int nsub = (int)sizes.size();
    if (nsub == 1) {
        TRY(upload(h, n));
        TRY(work(0, n, nullptr));
        TRY(download(0, n, h->stream));
        CK(h, cudaStreamSynchronize(h->stream));
        return scatter(0, n);
    }
    std::vector<int> starts(nsub, 0);
    for (int i = 1; i < nsub; ++i) starts[i] = starts[i - 1] + sizes[i - 1];
    TRY(ensure_pipeline_streams(h, nsub));
    CK(h, cudaEventRecord(h->ev_fork, h->stream));
    CK(h, cudaStreamWaitEvent(h->stream_up, h->ev_fork, 0));
    for (auto &sc : h->stream_c) CK(h, cudaStreamWaitEvent(sc, h->ev_fork, 0));
    for (int i = 0; i < nsub; ++i) {
        const int w0 = starts[i], m = sizes[i];
        cudaStream_t sc = h->stream_c[i % kPipeStreams];
        TRY(upload_range(h, w0, m, h->stream_up));
        CK(h, cudaEventRecord(h->ev_up[i], h->stream_up));
        CK(h, cudaStreamWaitEvent(sc, h->ev_up[i], 0));
        TRY(work(w0, m, sc));
        CK(h, cudaEventRecord(h->ev_done[i], sc));
        CK(h, cudaStreamWaitEvent(h->stream_down, h->ev_done[i], 0));
        CK(h, cudaStreamWaitEvent(h->stream, h->ev_done[i], 0));      // later calls on the handle's stream see the result
        TRY(download(w0, m, h->stream_down));
        CK(h, cudaEventRecord(h->ev_down[i], h->stream_down));
    }
    h->n_uploaded = n;
    for (int i = 0; i < nsub; ++i) {
        CK(h, cudaEventSynchronize(h->ev_down[i]));
        TRY(scatter(starts[i], sizes[i]));
    }
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // namespace pvio

using namespace pvio;

// ======================================================================== C ABI
extern "C" {

const char *pvio_b200_version(void) { return "pvio_b200 0.2 (sm_90a)"; }

int pvio_b200_create(int device, int max_windows, int max_frames, int max_landmarks, int max_obs,
                     pvio_b200_handle *out) {
    if (!out) return PVIO_B200_EINVAL;
    *out = nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0 || device >= ndev || device < 0) return PVIO_B200_ENODEV;
    if (max_windows < 1 || max_frames < 1 || max_frames > kMaxFrames || max_landmarks < 1 || max_landmarks > 65534 || max_obs < 1)
        return PVIO_B200_EINVAL;
    Handle *h = new Handle();
    h->device = device; h->W = max_windows; h->Ncap = max_frames;
    h->Mcap = (max_landmarks + 3) & ~3;                      // the Schur kernel's bulk copies move 16-byte granules (4 masks)
    h->Kcap = max_obs;
    if (cudaSetDevice(device) != cudaSuccess) { delete h; return PVIO_B200_ENODEV; }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    h->sm_count = prop.multiProcessorCount;
    *out = reinterpret_cast<pvio_b200_handle>(h);
    CK(h, cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
    CK(h, cudaEventCreate(&h->ev0)); CK(h, cudaEventCreate(&h->ev1));
    const size_t W = h->W, N = h->Ncap, M = h->Mcap, K = h->Kcap, npc = N * (N + 1) / 2;
    const size_t X = N * kFrameStride;                        // doubles per window of the frame states
    TRY(alloc(h, h->hdr, W, kBoth, 1)); TRY(alloc(h, h->cst, W, kBoth, 1));
    TRY(alloc(h, h->obs, W * K, kBoth, K)); TRY(alloc(h, h->lms, W * M, kBoth, M));
    // flm is padded: the update sweep copies five 16-byte granules from the one holding a row's first index (row_prefetch)
    TRY(alloc(h, h->fz, W * K, kDevice)); TRY(alloc(h, h->flm, W * K + kFlmPad, kDevice));
    TRY(alloc(h, h->seg, W * kSegTab, kDevice));
    TRY(alloc(h, h->rho, W * M, kBoth, M)); TRY(alloc(h, h->frames, W * X, kBoth, X));
    TRY(alloc(h, h->ctrl, W, kBoth, 1));
    TRY(alloc(h, h->rho_cand, W * M, kDevice)); TRY(alloc(h, h->frames_cand, W * X, kDevice));
    // the linearisation lives in two buffer sets (LinBufs, ba_types.h): everything below up to the reduced system is doubled
    TRY(alloc(h, h->lm_scale, W * M, kDevice)); TRY(alloc(h, h->lm_aux, 2 * W * M, kDevice));
    TRY(alloc(h, h->hs, 2 * W * N * M * 6 * sizeof(float), kDevice)); TRY(alloc(h, h->jr, 2 * W * N * M * 2 * sizeof(float), kDevice));
    TRY(alloc(h, h->lm_w, 2 * W * M * 2 * sizeof(float), kDevice)); TRY(alloc(h, h->lm_msk, 2 * W * M, kDevice));
    TRY(alloc(h, h->frames_out, W * X, kPinned, X)); TRY(alloc(h, h->rho_out, W * M, kPinned, M));
    TRY(alloc(h, h->dx_lm, W * M, kBoth, M)); TRY(alloc(h, h->lm_v, W * M, kDevice)); TRY(alloc(h, h->dx_pose, W * N * 15, kBoth, N * 15));
    TRY(alloc(h, h->pose_scale, W * N * 15, kDevice)); TRY(alloc(h, h->v_pose, W * N * 15, kDevice));
    TRY(alloc(h, h->valid, W * M, kBoth, M)); TRY(alloc(h, h->quality, W * M, kBoth, M));
    // the reduced-system outputs of the linearise kernel (Hred, Hdd, gdir, gred, cost_vis: refresh_arrays) live in ONE
    // allocation so that the multi-CTA-per-window mode (atomic accumulation) needs a single memset per launch
    // set 1 of each array lies sys_set elements behind set 0, an even count: the Schur kernel pulls a window's Hred and
    // gred of either set by bulk copies, which need 16-byte aligned addresses (W cost_vis entries make the sum odd for odd W)
    h->sys_set = (W * (npc * 36 + N * 36 + N * 6 + N * 6 + 1) + 1) & ~(size_t)1;
    TRY(alloc(h, h->Hred, 2 * h->sys_set, kDevice));
    TRY(alloc(h, h->acc, W * kAcc, kBoth)); TRY(alloc(h, h->aux_cost, W, kDevice));
    TRY(alloc(h, h->Hfull, (15 * N) * (15 * N), kBoth)); TRY(alloc(h, h->gfull, 15 * N, kBoth));
    refresh_arrays(h);
    h->slots.resize(W);
    {   // opt in to large dynamic shared memory ONCE per kernel with the device limit: the attribute is process-wide, so a
        // per-handle value would be overwritten by the next handle with other capacities
        const int lim = (int)prop.sharedMemPerBlockOptin - 2048;
        h->smem_lim = lim;
        CK(h, cudaFuncSetAttribute(lin_obs_kernel<true, float, kLinWarps, kLinBlocks>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(lin_obs_kernel<true, float, kLinWarps, kLinPartMinBlocks, kLinPartRows>,
                                   cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(lin_obs_kernel<true, double, kLinWarps, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(lin_obs_kernel<false, double, kLinWarps, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(schur_kernel<float, kSchurThreads, kSchurBlocks>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(schur_kernel<double, kSchurThreads, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<float, kUpdWarps, kUpdBlocks, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<float, kUpdWarps, kUpdBlocks, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<float, 8, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<double, kUpdWarps, 4, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<float, kUpdWarps, kUpdBlocks, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<double, kUpdWarps, 4, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<double, 8, 2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(update_obs_kernel<double, kUpdWarps, 4, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, lim));
        CK(h, cudaFuncSetAttribute(solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
        CK(h, cudaFuncSetAttribute(solve_kernel_visual, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024));
        CK(h, cudaFuncSetAttribute(cov_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
        TRY(selftest_chol_opt_in(h));
        TRY(marg_opt_in(h));
    }
    init_ctrl_kernel<<<(int)W, 32, 0, h->stream>>>(h->ctrl.d, 1e-8, 1e4, 10, 0.0, 0);
    ++h->launches;
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

void pvio_b200_destroy(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return;
    cudaSetDevice(h->device);
    cudaStreamSynchronize(h->stream);
    drop_graphs(h);
    for (auto &e : h->kev) cudaEventDestroy(e);
    cudaEventDestroy(h->ev0); cudaEventDestroy(h->ev1);
    for (auto &e : h->ev_up) cudaEventDestroy(e);
    for (auto &e : h->ev_done) cudaEventDestroy(e);
    for (auto &e : h->ev_down) cudaEventDestroy(e);
    if (h->stream_up) cudaStreamDestroy(h->stream_up);
    if (h->stream_down) cudaStreamDestroy(h->stream_down);
    for (auto &st : h->stream_c) cudaStreamDestroy(st);
    if (h->ev_fork) cudaEventDestroy(h->ev_fork);
    if (h->stream_aux) { cudaStreamDestroy(h->stream_aux); cudaEventDestroy(h->ev_aux_fork); cudaEventDestroy(h->ev_aux_join); }
    if (h->stream_mark) { cudaStreamDestroy(h->stream_mark); for (auto &e : h->ev_stage) cudaEventDestroy(e); }
    cudaStreamDestroy(h->stream);
    delete h;                        // frees every buffer (DevBuf)
}

const char *pvio_b200_last_error(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    return h ? h->err.c_str() : "null handle";
}

int64_t pvio_b200_kernel_launches(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    return h ? h->launches : 0;
}

int pvio_b200_sync(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

int pvio_b200_timer_start(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    CK(h, cudaEventRecord(h->ev0, h->stream));
    return 0;
}

int pvio_b200_timer_stop(pvio_b200_handle hh, float *ms) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !ms) return PVIO_B200_EINVAL;
    CK(h, cudaEventRecord(h->ev1, h->stream));
    CK(h, cudaEventSynchronize(h->ev1));
    CK(h, cudaEventElapsedTime(ms, h->ev0, h->ev1));
    return 0;
}

// Device time of the linearise + Schur stage from the CUDA events recorded around its launches:
// which = 0 the most recent stage; 1 the MEAN stage over the launches since the last reset (at most the latest 256);
// 2 / 3 the mean of the linearise / the Schur kernel alone; -1 resets the accumulation.  A split step (run_gn_step_split)
// records the same three events for the whole batch.
int pvio_b200_last_kernel_ms(pvio_b200_handle hh, int which, float *ms) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (which < 0) { h->kev_count = 0; if (ms) *ms = 0.f; return 0; }
    if (!ms) return PVIO_B200_EINVAL;
    if (h->kev_count == 0) { *ms = 0.f; return 0; }     // graph-replayed launches are not individually timed
    CK(h, cudaStreamSynchronize(h->stream));
    const int n = which == 0 ? 1 : std::min(h->kev_count, 256);
    double tot = 0.0;
    for (int i = 0; i < n; ++i) {
        const int slot = ((h->kev_count - 1 - i) % 256) * 3;
        float t = 0.f;
        const int e0 = which == 3 ? 1 : 0, e1 = which == 2 ? 1 : 2;
        CK(h, cudaEventElapsedTime(&t, h->kev[slot + e0], h->kev[slot + e1]));
        tot += t;
    }
    *ms = (float)(tot / n);
    return 0;
}

int pvio_b200_batch_set_window(pvio_b200_handle hh, int slot, const pvio_b200_window *w, const pvio_b200_state *s) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !s) return PVIO_B200_EINVAL;
    return pack_window(h, slot, w, s);
}

int pvio_b200_batch_replicate(pvio_b200_handle hh, int n) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 1 || n > h->W) return fail(h, PVIO_B200_EINVAL, "bad window count");
    TRY(check_packed(h, n, "batch_replicate"));
    if (h->slots[0].prior_resident && h->hdr.h[0].n_prior > 0)
        return fail(h, PVIO_B200_EINVAL, "batch_replicate: slot 0's prior is device-resident, its staging does not hold it");
    for (int i = 1; i < n; ++i) {
        h->slots[i].prior_resident = 0;          // the slot takes slot 0's host prior from the staging
        h->slots[i].perm = h->slots[0].perm;
        for_each_staged(h, [&](auto &b, bool) { copy_slot(b, i, b, 0); return 0; });
    }
    return 0;
}

int pvio_b200_batch_upload(pvio_b200_handle hh, int n) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_packed(h, n, "batch_upload"));
    return upload(h, n);
}

int pvio_b200_batch_gn_step(pvio_b200_handle hh, int n, double mu, int apply) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 1 || n > h->n_uploaded) return fail(h, PVIO_B200_EINVAL, "windows not uploaded");
    TRY(check_packed(h, n, "batch_gn_step"));
    StepCfg c;
    c.mu = mu; c.apply = apply; c.compute_scale = 1;
    const BatchShape b = batch_shape(h, 0, n, false);
    const int parts = gn_step_parts(h, n);
    return parts > 1 ? run_gn_step_split(h, n, c, b, parts) : run_gn_step(h, n, c, b);
}

// Not in the public header: the sub-batch count of batch_gn_step forced (parts > 0, at most 4, fewer when the batch is
// too small to keep the launch shapes) or chosen from the batch (0).  For the bit-identity tests and the tuning tools.
int pvio_b200_internal_set_step_split(pvio_b200_handle hh, int parts) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || parts < 0 || parts > kStepPartsMax) return PVIO_B200_EINVAL;
    h->step_parts = parts;
    return 0;
}

int pvio_b200_batch_download(pvio_b200_handle hh, int n, double *dx, int64_t dx_stride, double *costs) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_packed(h, n, "batch_download"));
    return download_dx(h, n, dx, dx_stride, costs);
}

// End-to-end step with HOST buffers: upload, one plain Gauss-Newton step, download (run_host_pipeline).
int pvio_b200_batch_gn_step_host(pvio_b200_handle hh, int n, double mu, double *dx, int64_t dx_stride, double *costs) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return run_host_pipeline(h, n, "batch_gn_step_host",
        [&](int w0, int m, cudaStream_t st) {
            StepCfg c;
            c.mu = mu; c.apply = 0; c.compute_scale = 1; c.w0 = w0; c.stream = st;
            return run_gn_step(h, m, c, batch_shape(h, w0, m, false));
        },
        [&](int w0, int m, cudaStream_t st) { return download_dx_async(h, w0, m, st); },
        [&](int w0, int m) { return scatter_dx(h, w0, m, dx, dx_stride, costs); });
}

// Full trust-region solve (device-side loop, per-window termination) of the first n uploaded windows; the states on
// the device are overwritten with the solutions.
int pvio_b200_batch_solve(pvio_b200_handle hh, int n, const pvio_b200_options *opt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 1 || n > h->n_uploaded) return fail(h, PVIO_B200_EINVAL, "windows not uploaded");
    TRY(check_packed(h, n, "batch_solve"));
    return run_solve_loop(h, solve_options(opt), 0, n, h->stream);
}

int pvio_b200_batch_download_state(pvio_b200_handle hh, int n, double *frames, int64_t frames_stride, double *inv_depth,
                                   int64_t inv_depth_stride, pvio_b200_summary *summaries) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n < 1 || n > h->W) return fail(h, PVIO_B200_EINVAL, "bad window count");
    TRY(check_packed(h, n, "batch_download_state"));
    TRY(download_state_async(h, 0, n, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    scatter_states(h, 0, n, frames, frames_stride, inv_depth, inv_depth_stride, summaries);
    return 0;
}

// upload + solve + download with HOST buffers, pipelined over sub-batches like pvio_b200_batch_gn_step_host: one
// host -> device copy buys up to max_iterations Gauss-Newton iterations per window.
int pvio_b200_batch_solve_host(pvio_b200_handle hh, int n, const pvio_b200_options *opt, double *frames, int64_t frames_stride,
                               double *inv_depth, int64_t inv_depth_stride, pvio_b200_summary *summaries) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const SolveOptions o = solve_options(opt);
    return run_host_pipeline(h, n, "batch_solve_host",
        [&](int w0, int m, cudaStream_t st) { return run_solve_loop(h, o, w0, m, st ? st : h->stream); },
        [&](int w0, int m, cudaStream_t st) { return download_state_async(h, w0, m, st); },
        [&](int w0, int m) {
            scatter_states(h, w0, m, frames, frames_stride, inv_depth, inv_depth_stride, summaries);
            return 0;
        });
}

int pvio_b200_ba_gn_step(pvio_b200_handle hh, const pvio_b200_window *w, const pvio_b200_state *s, double mu,
                         double *dx, double *cost, double *new_cost, double *Hred, double *gred) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !s) return PVIO_B200_EINVAL;
    TRY(pack_window(h, 0, w, s));
    TRY(upload(h, 1));
    StepCfg c;
    c.mu = mu; c.apply = 0; c.compute_scale = 1; c.dump = (Hred || gred) ? 1 : 0;
    if (c.dump) {
        CK(h, cudaMemsetAsync(h->Hfull.d, 0, sizeof(double) * h->Hfull.n, h->stream));
        CK(h, cudaMemsetAsync(h->gfull.d, 0, sizeof(double) * h->gfull.n, h->stream));
    }
    TRY(run_gn_step(h, 1, c, batch_shape(h, 0, 1, false)));
    double costs[2];
    const int N = w->n_frames, M = w->n_landmarks;
    TRY(download_dx(h, 1, dx, (int64_t)N * 15 + M, costs));
    if (cost) *cost = costs[0];
    if (new_cost) *new_cost = costs[1];
    if (c.dump) {
        const size_t Df = 15 * (size_t)h->Ncap, Dn = 15 * (size_t)N;
        CK(h, cudaMemcpyAsync(h->Hfull.h, h->Hfull.d, sizeof(double) * Df * Df, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaMemcpyAsync(h->gfull.h, h->gfull.d, sizeof(double) * Df, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaStreamSynchronize(h->stream));
        if (Hred) for (size_t i = 0; i < Dn; ++i) memcpy(Hred + i * Dn, h->Hfull.h + i * Df, sizeof(double) * Dn);
        if (gred) memcpy(gred, h->gfull.h, sizeof(double) * Dn);
    }
    return 0;
}

// BundleAdjustorSolver::solve (bundle_adjustor.cpp:63-299) behind the shim's gather: pack, one host -> device copy,
// the device-side trust-region loop (ONE graph launch, ba_tr.cuh), the landmark post-pass, one device -> host copy.
int pvio_b200_ba_solve(pvio_b200_handle hh, const pvio_b200_window *w, pvio_b200_state *s,
                       const pvio_b200_options *opt, pvio_b200_summary *summary, uint8_t *valid, double *quality) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !s) return PVIO_B200_EINVAL;
    TRY(pack_window(h, 0, w, s));
    TRY(upload(h, 1));
    CK(h, cudaEventRecord(h->ev0, h->stream));
    TRY(run_solve_loop(h, solve_options(opt), 0, 1, h->stream));
    CK(h, cudaEventRecord(h->ev1, h->stream));
    const int M = w->n_landmarks;
    const bool post = (!opt || opt->run_postpass) && (valid || quality);
    if (post) {
        TRY(run_postpass(h, 1, true, nullptr));
        CK(h, cudaMemcpyAsync(h->valid.h, h->valid.d, (size_t)std::max(M, 1), cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaMemcpyAsync(h->quality.h, h->quality.d, sizeof(double) * std::max(M, 1), cudaMemcpyDeviceToHost, h->stream));
    }
    TRY(download_state_async(h, 0, 1, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    scatter_state(h, 0, s->frames, s->inv_depth);
    if (post && valid) unpermute(h, 0, valid, h->valid.h);
    if (post && quality) unpermute(h, 0, quality, h->quality.h);
    if (summary) {
        fill_summary(h->ctrl.h[0], summary);
        float ms = 0.f;
        cudaEventElapsedTime(&ms, h->ev0, h->ev1);
        summary->solve_seconds = ms * 1e-3;
    }
    return 0;
}

int pvio_b200_reprojection_error(pvio_b200_handle hh, const pvio_b200_window *w, const pvio_b200_state *s, double *error) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !s || !error) return PVIO_B200_EINVAL;
    TRY(pack_window(h, 0, w, s));
    TRY(upload(h, 1));
    CK(h, cudaMemsetAsync(h->acc.d, 0, sizeof(double) * 8, h->stream));
    TRY(run_postpass(h, 1, false, h->acc.d));
    CK(h, cudaMemcpyAsync(h->acc.h, h->acc.d, sizeof(double) * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    *error = h->acc.h[0] / std::max(h->acc.h[1], 1.0);
    return 0;
}

int pvio_b200_ba_marginalize(pvio_b200_handle hh, const pvio_b200_window *w, const pvio_b200_state *s, int index,
                             double *S_out, double *e_out, double *H_out, double *b_out) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !s) return PVIO_B200_EINVAL;
    return marginalize_impl(h, w, s, index, S_out, e_out, H_out, b_out);
}

int pvio_b200_batch_marginalize(pvio_b200_handle hh, int n, double *S_out, int64_t S_stride, double *e_out, int64_t e_stride) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    TRY(check_packed(h, n, "batch_marginalize"));
    return batch_marginalize_impl(h, n, S_out, S_stride, e_out, e_stride);
}

int pvio_b200_pnp_solve(pvio_b200_handle hh, const pvio_b200_pnp_problem *problem, double *frame,
                        const pvio_b200_options *opt, pvio_b200_summary *summary) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !problem || !frame) return PVIO_B200_EINVAL;
    return pnp_solve_impl(h, problem, frame, opt, summary);
}

int pvio_b200_batch_pnp_solve(pvio_b200_handle hh, int n, const pvio_b200_pnp_problem *problems, double *frames,
                              int64_t frames_stride, const pvio_b200_options *opt, pvio_b200_summary *summaries) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_pnp_solve_impl(h, n, problems, frames, frames_stride, opt, summaries);
}

int pvio_b200_klt_track(pvio_b200_handle hh, const uint8_t *prev, const uint8_t *next, int width, int height, int stride,
                        const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                        int max_level, int max_iter, double eps) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !prev || !next || !prev_pts || !next_pts || !status) return PVIO_B200_EINVAL;
    return klt_track_impl(h, prev, next, width, height, stride, prev_pts, next_pts, status, err, n_points, max_level,
                          max_iter, eps);
}

int pvio_b200_klt_track_raw(pvio_b200_handle hh, const uint8_t *prev, const uint8_t *next, int width, int height, int stride,
                            const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                            int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                            uint8_t *prev_eq, uint8_t *next_eq) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !prev || !next || !prev_pts || !next_pts || !status) return PVIO_B200_EINVAL;
    if (!(clahe_clip > 0.0)) return fail(h, PVIO_B200_EINVAL, "klt_track_raw: clahe_clip must be positive");
    return klt_track_impl(h, prev, next, width, height, stride, prev_pts, next_pts, status, err, n_points, max_level,
                          max_iter, eps, clahe_clip, tiles_x, tiles_y, prev_eq, next_eq);
}

int pvio_b200_klt_track_cached(pvio_b200_handle hh, uint64_t prev_id, const uint8_t *prev, uint64_t next_id, const uint8_t *next,
                               int width, int height, int stride, const float *prev_pts, float *next_pts, uint8_t *status, float *err,
                               int n_points, int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                               int border) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !prev_pts || !next_pts || !status) return PVIO_B200_EINVAL;
    if (clahe_clip < 0.0) return fail(h, PVIO_B200_EINVAL, "klt_track_cached: clahe_clip must be >= 0 (0: frames are already equalised)");
    return klt_track_impl(h, prev, next, width, height, stride, prev_pts, next_pts, status, err, n_points, max_level,
                          max_iter, eps, clahe_clip, tiles_x, tiles_y, nullptr, nullptr, prev_id, next_id, border);
}

int pvio_b200_find_fundamental_mask(pvio_b200_handle hh, int n, const float *p, const float *q, double threshold, double confidence,
                                    int max_iters, const int32_t *schedule, int n_schedule, uint8_t *mask, double *F, int32_t *info) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || n < 0 || (n > 0 && (!p || !q || !mask))) return PVIO_B200_EINVAL;
    return fm_ransac_impl(h, n, p, q, threshold, confidence, max_iters, schedule, n_schedule, mask, F, info);
}

int pvio_b200_fm_sample_schedule(int n, const float *p, const float *q, int iters, int32_t *schedule) {
    if (n < 8 || !p || !q || iters < 1 || !schedule) return PVIO_B200_EINVAL;
    return fm_cv_schedule(n, p, q, iters, schedule);
}

int pvio_b200_track_keypoints(pvio_b200_handle hh, uint64_t prev_id, const uint8_t *prev, uint64_t next_id, const uint8_t *next,
                              int width, int height, int stride, const float *prev_pts, float *next_pts, uint8_t *status,
                              int n_points, int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                              int border, double ransac_threshold, double ransac_confidence) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !prev_pts || !next_pts || !status) return PVIO_B200_EINVAL;
    if (clahe_clip < 0.0) return fail(h, PVIO_B200_EINVAL, "track_keypoints: clahe_clip must be >= 0 (0: frames are already equalised)");
    if (n_points <= 0) return 0;
    TRY(klt_track_impl(h, prev, next, width, height, stride, prev_pts, next_pts, status, nullptr, n_points, max_level,
                       max_iter, eps, clahe_clip, tiles_x, tiles_y, nullptr, nullptr, prev_id, next_id, border));
    // opencv_image.cpp:112-129: the survivors, in order, through findFundamentalMat(FM_RANSAC, 1.0, 0.99) when there are >= 8
    std::vector<int> l;
    std::vector<float> p, q;
    l.reserve(n_points); p.reserve(2 * n_points); q.reserve(2 * n_points);
    for (int i = 0; i < n_points; ++i)
        if (status[i]) {
            l.push_back(i);
            p.push_back(prev_pts[2 * i]); p.push_back(prev_pts[2 * i + 1]);
            q.push_back(next_pts[2 * i]); q.push_back(next_pts[2 * i + 1]);
        }
    if (l.size() >= 8) {
        std::vector<uint8_t> mask(l.size());
        TRY(fm_ransac_impl(h, (int)l.size(), p.data(), q.data(), ransac_threshold, ransac_confidence, 1000, nullptr, 0, mask.data(),
                           nullptr, nullptr));
        for (size_t i = 0; i < l.size(); ++i)
            if (!mask[i]) status[l[i]] = 0;
    }
    return 0;
}

int pvio_b200_batch_track_keypoints(pvio_b200_handle hh, int n, const pvio_b200_klt_pair *pairs, int max_level, int max_iter,
                                    double eps, double clahe_clip, int tiles_x, int tiles_y, int border,
                                    double ransac_threshold, double ransac_confidence) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_track_impl(h, n, pairs, max_level, max_iter, eps, clahe_clip, tiles_x, tiles_y, border, ransac_threshold,
                            ransac_confidence);
}

int pvio_b200_batch_feature_track(pvio_b200_handle hh, int n, const pvio_b200_feature_frame *frames, int max_level, int max_iter,
                                  double eps, double clahe_clip, int tiles_x, int tiles_y, int border,
                                  double ransac_threshold, double ransac_confidence, double keypoint_distance) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    const KltBatchOptions o{max_level, max_iter, eps, clahe_clip, tiles_x, tiles_y, border, ransac_threshold, ransac_confidence};
    return batch_feature_track_impl(h, n, frames, o, keypoint_distance);
}

int pvio_b200_batch_detect_keypoints(pvio_b200_handle hh, int n, const pvio_b200_detect_request *requests, double clahe_clip,
                                     int tiles_x, int tiles_y) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_detect_impl(h, n, requests, clahe_clip, tiles_x, tiles_y);
}

int pvio_b200_clahe(pvio_b200_handle hh, const uint8_t *src, int width, int height, int stride, double clip_limit,
                    int tiles_x, int tiles_y, uint8_t *dst) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !src || !dst) return PVIO_B200_EINVAL;
    return clahe_impl(h, src, width, height, stride, clip_limit, tiles_x, tiles_y, dst);
}

int pvio_b200_selftest_lie(pvio_b200_handle hh, int n, const double *w, double *out) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !w || !out || n < 1) return PVIO_B200_EINVAL;
    return selftest_lie_impl(h, n, w, out);
}

int pvio_b200_selftest_eig(pvio_b200_handle hh, int n, const int32_t *dk, const double *A, const double *b, double *S_out,
                           double *e_out) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !dk || !A || !b || !S_out || !e_out) return PVIO_B200_EINVAL;
    return selftest_eig_impl(h, n, dk, A, b, S_out, e_out);
}

int pvio_b200_selftest_chol(pvio_b200_handle hh, int n, int mode, const int32_t *D, const double *A, const double *b,
                            double *x_out, int32_t *ok_out) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !D || !A || !b || !x_out || !ok_out) return PVIO_B200_EINVAL;
    return selftest_chol_impl(h, n, mode, D, A, b, x_out, ok_out);
}

#ifdef PVIO_SOLVE_STAMPS
int pvio_b200_debug_solve_stamps(long long *out) {      // tuning builds only (tools/solve_stamps.py); not declared in include/pvio_b200.h
    return cudaMemcpyFromSymbol(out, pvio::g_solve_stamps, sizeof(long long) * 16) == cudaSuccess ? 0 : PVIO_B200_ECUDA;
}
#endif

}  // extern "C"
