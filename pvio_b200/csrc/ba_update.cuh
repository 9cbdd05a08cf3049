// Back-substitution of the inverse depths, Plus() update and candidate-cost sweep.
//
// After the reduced system has been solved for the pose step, this kernel does what ceres
// does after the Schur solve of an iteration (bundle_adjustor.cpp:249, inside ceres::Solve):
//   d rho_l = -(g_l + h_l . dxi) / (H_ll + reg)                 back-substitution
//   candidate = Plus(x, dx)         (quaternion_parameterization.h:28-31, plain + elsewhere)
//   candidate cost = sum rho(|r|^2)/2 over the reprojection blocks   (step acceptance)
// and accumulates the scalars the trust-region logic needs.  sqrt(w_l) h_l comes from the linearise kernel
// (LinArgs::hs_out: one record of 6 N floats per landmark slot, written there by bulk copies).  Recomputing it from the observation table costs one full linearisation per observation and was
// most of this kernel's instructions; the kernels are issue-bound and HBM is far from its bandwidth, so
// 2 x 108 KB of extra traffic per window are the cheaper side of the trade.
#pragma once
#include "ba_linearize.cuh"
#include "ba_tr.cuh"

namespace pvio {

struct UpdArgs : BatchArrays {
    double mu_override;
    int w0;
    // step = step_b * dx_gn - step_a * v, v = S^2 g / clamp(S^2 diag H) the scaled steepest-descent direction:
    // (0, 1) Gauss-Newton, (0, beta) truncated GN, (a, b) dogleg interpolation, (a, 0) Cauchy leg
    double step_a, step_b;
    int loop;                 // 1: hs / lm_aux of the window's current buffer set (WinCtrl::buf); jv_vision_kernel: only
                              // windows whose GN step left the trust region (WinCtrl::need_jv)
};

template <typename real>
__host__ __device__ inline size_t upd_smem_layout(int N, int Mp, int warps, size_t *o_dxi, size_t *o_x, size_t *o_seg, size_t *o_red, size_t *o_ring) {
    size_t off = sizeof(FrameSm) * (size_t)N;                      // candidate camera poses
    *o_dxi = off; off += sizeof(double) * 6 * (size_t)N;           // xi = T delta per frame
    *o_x = off; off += sizeof(double) * 3 * (size_t)Mp;            // candidate world points (SoA)
    *o_red = off; off += sizeof(double) * 8;
    *o_seg = off; off += sizeof(int32_t) * kSegTab;
    off = (off + 15) & ~(size_t)15;
    *o_ring = off; off += sizeof(RowSlot) * kRing * (size_t)warps;
    return off;
}
template <typename real>
__host__ __device__ inline size_t upd_smem_bytes(int N, int Mp, int warps) {
    size_t a, b, c, d, e;
    return upd_smem_layout<real>(N, Mp, warps, &a, &b, &c, &d, &e);
}

// Residual-only evaluation of one block (candidate cost): fp64 numerators, the rest in `real`.  Returns t = 1 + s / b of
// the Cauchy loss; the caller accumulates b/2 log t (LogAcc).
template <typename real>
__device__ __forceinline__ real residual_cost_blk(const double (&Rwc)[9], const double (&c)[3], double x0, double x1, double x2,
                                                  float zx, float zy, const real (&W)[4], bool diag_w, real inv_cauchy_b) {
    const double d0 = x0 - c[0], d1 = x1 - c[1], d2 = x2 - c[2];
    const double y0 = Rwc[0] * d0 + Rwc[3] * d1 + Rwc[6] * d2;
    const double y1 = Rwc[1] * d0 + Rwc[4] * d1 + Rwc[7] * d2;
    const double y2 = Rwc[2] * d0 + Rwc[5] * d1 + Rwc[8] * d2;
    const double nx = y0 - (double)zx * y2, ny = y1 - (double)zy * y2;
    const real iz = rcp_r((real)y2);
    const real u0 = (real)nx * iz, u1 = (real)ny * iz;
    real r0 = W[0] * u0, r1 = W[3] * u1;
    if (!diag_w) { r0 += W[1] * u1; r1 += W[2] * u0; }
    const real s = r0 * r0 + r1 * r1;
    return (real)1 + s * inv_cauchy_b;
}

// Back-substitution (thread per landmark, coalesced reads of the frame-major h records), Plus, and the
// candidate cost over the frame-major table (thread per residual block, target pose in registers).
//   kMode 0  everything in one launch with the step (step_a, step_b) given by the caller: the plain Gauss-Newton
//            iteration of pvio_b200_ba_gn_step / batch_gn_step.  gridDim.x CTAs may share a window (landmark l
//            belongs to CTA (l / 32) mod gridDim.x, the rows are cut as in lin_obs_kernel).
//   kMode 1  back-substitution only (gridDim.x = 1): GN step of the inverse depths and its scalars, then the
//            trust-region test of the step (tr_after_backsub): first half of an iteration of the device-side loop.
//   kMode 2  candidate only: Plus(x, step_b dx_gn - step_a v) with the step chosen by tr_after_jv (its cost comes from
//            the speculative linearise sweep that follows, ba_tr.cuh).
template <typename real, int kWarps, int kMinBlocks, int kMode>
__global__ void __launch_bounds__(kWarps * 32, kMinBlocks)
update_obs_kernel(UpdArgs a) {
    constexpr int kThreads = kWarps * 32;
    const int w = blockIdx.y + a.w0;
    WinCtrl &ctrl = a.ctrl[w];
    if (kMode == 1 && ctrl.done) return;
    if (kMode == 2 && (ctrl.done || ctrl.skip)) return;
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int N = H.N, M = H.M, Mp = (M + 31) & ~31;
    const int tid = threadIdx.x, lane = tid & 31, wv = tid >> 5;
    const int nsp = N * (N - 1) / 2;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    size_t o_dxi, o_x, o_seg, o_red, o_ring;
    upd_smem_layout<real>(N, Mp, kWarps, &o_dxi, &o_x, &o_seg, &o_red, &o_ring);
    FrameSm *Fc = reinterpret_cast<FrameSm *>(smem_raw);                // [N] candidate camera poses
    double *dxi = reinterpret_cast<double *>(smem_raw + o_dxi);         // [N][6]
    double *xs = reinterpret_cast<double *>(smem_raw + o_x);            // [3][Mp]
    double *red = reinterpret_cast<double *>(smem_raw + o_red);         // [8]
    int32_t *sg = reinterpret_cast<int32_t *>(smem_raw + o_seg);

    const double step_a = kMode == 2 ? ctrl.step_a : a.step_a;
    const double step_b = kMode == 2 ? ctrl.step_b : a.step_b;
    // the candidate poses (warp 0) and the frame steps xi (warp 1) are independent: in separate warps, neither adds to
    // the other's registers
    static_assert(kThreads >= 32 + kMaxFrames, "update_obs_kernel: warp 1 computes the frame steps");
    if (kMode != 1 && tid < N) {
        const double *fs = a.frames + ((size_t)w * a.Ncap + tid) * kFrameStride;
        const double *d = a.dx_pose + ((size_t)w * a.Ncap + tid) * 15;
        const double *vp = a.v_pose + ((size_t)w * a.Ncap + tid) * 15;
        // only the candidate pose stays in registers; the rest of the candidate state goes straight to frames_cand
        auto step = [&](int i) { return step_b * d[i] - (step_a != 0.0 ? step_a * vp[i] : 0.0); };
        double fc[7];
        {
            const double dr[3] = {step(0), step(1), step(2)};
            quat_plus(fs, dr, fc);
        }
#pragma unroll
        for (int i = 4; i < 7; ++i) fc[i] = fs[i] + step(i - 1);
        if (blockIdx.x == 0) {
            double *o = a.frames_cand + ((size_t)w * a.Ncap + tid) * kFrameStride;
            double amb = 0.0;
#pragma unroll
            for (int i = 0; i < kFrameStride; ++i) {
                const double v = i < 7 ? fc[i] : fs[i] + step(i - 1);
                o[i] = v;
                const bool pose = i < 7;
                const bool live = pose ? !((H.fixed_mask >> tid) & 1) : (H.use_inertial != 0);
                if (live) amb += (v - fs[i]) * (v - fs[i]);
            }
            atomicAdd(&a.acc[(size_t)w * kAcc + 6], amb);
        }
        make_frame(fc, wc, Fc[tid]);
    }
    if (kMode != 2 && tid >= 32 && tid < 32 + N) {
        const int f = tid - 32;
        const double *fs = a.frames + ((size_t)w * a.Ncap + f) * kFrameStride;
        const double *d = a.dx_pose + ((size_t)w * a.Ncap + f) * 15;
        double R[9], om[3];
        quat_to_mat(fs, R);
        mat3_vec(R, d, om);
        const double p0 = fs[4] - wc.origin[0], p1 = fs[5] - wc.origin[1], p2 = fs[6] - wc.origin[2];
        dxi[f * 6 + 0] = om[0]; dxi[f * 6 + 1] = om[1]; dxi[f * 6 + 2] = om[2];
        dxi[f * 6 + 3] = -(p1 * om[2] - p2 * om[1]) - d[3];
        dxi[f * 6 + 4] = -(p2 * om[0] - p0 * om[2]) - d[4];
        dxi[f * 6 + 5] = -(p0 * om[1] - p1 * om[0]) - d[5];
    }
    if (tid < 8) red[tid] = 0.0;
    if (kMode == 0) for (int i = tid; i < kSegTab; i += kThreads) sg[i] = a.seg[(size_t)w * kSegTab + i];
    __syncthreads();

    const size_t bsel = a.loop ? (size_t)ctrl.buf : 0;
    const LmAux *aux = a.lm_aux + bsel * a.bufs.lm_aux;
    const real *hs = reinterpret_cast<const real *>(reinterpret_cast<const char *>(a.hs) + bsel * a.bufs.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    const unsigned fixed = (unsigned)H.fixed_mask & ((1u << N) - 1u);

    // ---- phase 1a: h_l . dxi = sum_t h_lt . (dxi_t - dxi_a) of the thread's landmarks, in frame order, parked in xs[l]
    // (the slot the landmark's candidate world point takes in phase 1b; the same thread reads it back).  Nothing but
    // the records in flight is live here.
    if (kMode != 2) {
        constexpr int kGroup = 6;       // records in flight: the <= 9 target frames of a 10-frame window in two groups
        for (int l = tid; l < M; l += kThreads) {
            const int meta = a.lms[(size_t)w * a.Mcap + l].meta;
            if (lm_nobs(meta) == 0) continue;
            const int anchor = lm_anchor(meta);
            double hdx = 0.0;
            typedef typename Vec2<real>::type real2;
            unsigned fm = lm_mask(meta);
            if ((fixed >> anchor) & 1u) fm &= ~fixed;                  // record not written; both steps are zero
            const double *da = dxi + anchor * 6;
            // the loads of a group are independent of each other; the anchor block of a residual is minus its target block
            while (fm) {
                int fr[kGroup];
                real2 h[kGroup][3];
#pragma unroll
                for (int q = 0; q < kGroup; ++q) {
                    fr[q] = fm ? __ffs(fm) - 1 : -1;
                    fm &= fm - 1;
                    if (fr[q] >= 0) {
                        const real2 *hp = reinterpret_cast<const real2 *>(hs + ((size_t)fr[q] * a.Mcap + l) * 6);
                        h[q][0] = hp[0]; h[q][1] = hp[1]; h[q][2] = hp[2];
                    }
                }
#pragma unroll
                for (int q = 0; q < kGroup; ++q) {
                    if (fr[q] < 0) continue;
                    const double *df = dxi + fr[q] * 6;
                    hdx += (double)h[q][0].x * (df[0] - da[0]) + (double)h[q][0].y * (df[1] - da[1]) + (double)h[q][1].x * (df[2] - da[2]) +
                           (double)h[q][1].y * (df[3] - da[3]) + (double)h[q][2].x * (df[4] - da[4]) + (double)h[q][2].y * (df[5] - da[5]);
                }
            }
            xs[l] = hdx;
        }
    }

    // ---- phase 1b: back-substitution, candidate inverse depth and world point
    double s_gdx = 0.0, s_reg = 0.0, s_gn = 0.0, s_dx2 = 0.0, s_x2 = 0.0, s_g2 = 0.0, s_vrd = 0.0;
    for (int l = tid; l < Mp; l += kThreads) {
        double x0 = 0.0, x1 = 0.0, x2 = 1.0;
        if (l < M) {
            const size_t gi = (size_t)w * a.Mcap + l;
            const int meta = a.lms[gi].meta;
            const int n_obs = lm_nobs(meta), anchor = lm_anchor(meta);
            const double rl = a.rho[gi];
            const bool mine = ((l >> 5) % (int)gridDim.x) == (int)blockIdx.x;
            double drho = 0.0, vl = 0.0;
            if (n_obs > 0 && kMode != 2) {
                const double hdx = xs[l];
                const LmAux ax = aux[gi];
                const double wl = 1.0 / ax.hll_reg;
                const double hll = ax.hll;
                drho = isfinite(wl) ? -(ax.gl + hdx) * wl : 0.0;
                const double sc = a.lm_scale[gi];
                const double mu = a.mu_override >= 0.0 ? a.mu_override : ctrl.mu;
                const double reg = mu > 0.0 ? lm_reg(hll, sc, mu) : 0.0;
                double d2 = sc * sc * hll;
                d2 = fmin(fmax(d2, 1.0e-6), 1.0e32);
                vl = sc * sc * ax.gl / d2;                       // scaled steepest-descent direction
                if (mine) {
                    s_gdx += hdx * ax.gl * wl + ax.gl * drho;
                    s_reg += reg * drho * drho;
                    s_gn += d2 * (drho / sc) * (drho / sc);
                    s_g2 += vl * ax.gl;
                    s_vrd += vl * reg * drho;
                    s_x2 += rl * rl;
                }
            }
            if (kMode == 1) { a.dx_lm[gi] = drho; a.lm_v[gi] = vl; continue; }
            if (kMode == 2 && n_obs > 0) { drho = a.dx_lm[gi]; vl = a.lm_v[gi]; }
            drho = step_b * drho - step_a * vl;
            if (mine) { s_dx2 += drho * drho; a.rho_cand[gi] = rl + drho; a.dx_lm[gi] = drho; }
            if (kMode != 2 && n_obs > 0) {
                const double *R = Fc[anchor].Rwc, *ca = Fc[anchor].c;
                const double ir = 1.0 / (rl + drho);
                const LmRec &lr = a.lms[gi];
                const double zx = (double)lr.zrx, zy = (double)lr.zry;
                x0 = (R[0] * zx + R[1] * zy + R[2]) * ir + ca[0];
                x1 = (R[3] * zx + R[4] * zy + R[5]) * ir + ca[1];
                x2 = (R[6] * zx + R[7] * zy + R[8]) * ir + ca[2];
            }
        }
        if (kMode == 0) { xs[l] = x0; xs[Mp + l] = x1; xs[2 * Mp + l] = x2; }
    }
    {   // the back-substitution scalars are complete: reduced here, so that the row walk carries s_cost alone
        double v[7] = {s_gdx, s_reg, s_gn, s_dx2, s_x2, s_g2, s_vrd};
#pragma unroll
        for (int k = 0; k < 7; ++k) {
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], off);
            if (lane == 0 && v[k] != 0.0) atomicAdd(&red[k + 1], v[k]);
        }
    }
    __syncthreads();

    // ---- phase 2: candidate cost over the rows of the frame-major table
    if (kMode == 0) {
        double s_cost = 0.0;
        const real W[4] = {(real)wc.sic[0], (real)wc.sic[1], (real)wc.sic[2], (real)wc.sic[3]};
        const real cb = (real)(wc.cauchy_a * wc.cauchy_a), inv_cb = (real)(1.0 / (wc.cauchy_a * wc.cauchy_a));
        const bool diag_w = wc.sic[1] == 0.0 && wc.sic[2] == 0.0;
        const float2 *fz = a.fz + (size_t)w * a.Kcap;
        const FLm *flm = a.flm + (size_t)w * a.Kcap;
        const int32_t *sbeg = sg, *srow = sg + kMaxSeg + 1;
        const int rows = srow[nsp];
        const int nwt = gridDim.x * kWarps, wid = blockIdx.x * kWarps + wv;
        const int r_begin = (int)((long long)rows * wid / nwt), r_end = (int)((long long)rows * (wid + 1) / nwt);
        // rows through a per-warp cp.async ring of kRing rows
        RowSlot *ring = reinterpret_cast<RowSlot *>(smem_raw + o_ring) + (size_t)wv * kRing;
        RowCursor pf(sbeg, srow, r_begin, rows), cs(sbeg, srow, r_begin, rows);
#pragma unroll
        for (int d = 0; d < kRing; ++d) row_prefetch(pf, r_end, fz, flm, ring + d, lane);
        int slot = 0;
        while (cs.r < r_end) {
            const int sp = cs.sp, t = cs.t;
            const int seg_end = sbeg[sp + 1];
            const int r_stop = min(r_end, srow[sp + 1]);
            double Rwc[9], c[3];
#pragma unroll
            for (int i = 0; i < 9; ++i) Rwc[i] = Fc[t].Rwc[i];
#pragma unroll
            for (int i = 0; i < 3; ++i) c[i] = Fc[t].c[i];
            LogAcc<real> la;
            int nfold = 0;
            for (; cs.r < r_stop; cs.advance()) {
                const int k = cs.k0() + lane;
                asm volatile("cp.async.wait_group %0;" :: "n"(kRing - 1) : "memory");
                __syncwarp();                     // the index granules of the row were copied by lanes 0-4
                const float2 z = ring[slot].z[lane];
                const int l = row_lm(ring[slot], lane);     // stale past the segment's end, and unused there
                __syncwarp();                     // every lane has read the slot before it is refilled
                row_prefetch(pf, r_end, fz, flm, ring + slot, lane);
                slot = slot + 1 == kRing ? 0 : slot + 1;
                if (k < seg_end)
                    la.add(residual_cost_blk<real>(Rwc, c, xs[l], xs[Mp + l], xs[2 * Mp + l], z.x, z.y, W, diag_w, inv_cb));
                if ((++nfold & 3) == 0) la.fold();
            }
            s_cost += (double)((real)0.5 * cb * la.total());
        }
        asm volatile("cp.async.wait_all;" ::: "memory");
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) s_cost += __shfl_xor_sync(0xffffffffu, s_cost, off);
        if (lane == 0 && s_cost != 0.0) atomicAdd(&red[0], s_cost);
    }
    __syncthreads();
    double *acc = a.acc + (size_t)w * kAcc;
    if (kMode == 1) {
        // one CTA owns the window: plain stores; also clears the slots the later sweeps of this iteration add to
        if (tid < kAcc) {
            double o = 0.0;
            if (tid >= 1 && tid <= 3) o = red[tid];
            else if (tid == 5) o = red[5];
            else if (tid == 7) o = red[6];
            else if (tid == 8) o = red[7];
            acc[tid] = o;
        }
        __syncthreads();
        if (tid == 0) { WinCtrl c = ctrl; tr_after_backsub(c, acc); ctrl = c; }
    } else if (tid < 8) {
        const int slot = tid < 6 ? tid : tid + 1;            // slot 6 is the frames' ambient step norm
        if (kMode == 2 && tid != 4) return;                  // the GN scalars were written by the back-substitution
        if (red[tid] != 0.0) atomicAdd(acc + slot, red[tid]);
    }
}

// |J v|^2 over the reprojection blocks (loss-corrected Jacobians), for the Cauchy point of the dogleg
// step: alpha = |grad|^2 / |J S D^-1 grad|^2 (ceres dogleg_strategy.cc ComputeCauchyPoint).
__global__ void __launch_bounds__(kLinThreads, 2)
jv_vision_kernel(UpdArgs a) {
    const int w = blockIdx.y + a.w0;
    if (a.loop && (a.ctrl[w].done || a.ctrl[w].skip || !a.ctrl[w].need_jv)) return;
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int N = H.N;
    const int tid = threadIdx.x, lane = tid & 31, wv = tid >> 5;
    __shared__ FrameSm F[kMaxFrames];
    __shared__ double vxi[kMaxFrames][6];
    __shared__ double red;
    if (tid < N) {
        const double *fs = a.frames + ((size_t)w * a.Ncap + tid) * kFrameStride;
        const double *d = a.v_pose + ((size_t)w * a.Ncap + tid) * 15;
        make_frame(fs, wc, F[tid]);
        double R[9], om[3];
        quat_to_mat(fs, R);
        mat3_vec(R, d, om);
        const double p0 = fs[4] - wc.origin[0], p1 = fs[5] - wc.origin[1], p2 = fs[6] - wc.origin[2];
        vxi[tid][0] = om[0]; vxi[tid][1] = om[1]; vxi[tid][2] = om[2];
        vxi[tid][3] = -(p1 * om[2] - p2 * om[1]) - d[3];
        vxi[tid][4] = -(p2 * om[0] - p0 * om[2]) - d[4];
        vxi[tid][5] = -(p0 * om[1] - p1 * om[0]) - d[5];
    }
    if (tid == 0) red = 0.0;
    __syncthreads();
    const float W[4] = {(float)wc.sic[0], (float)wc.sic[1], (float)wc.sic[2], (float)wc.sic[3]};
    const float cb = (float)(wc.cauchy_a * wc.cauchy_a);
    const ObsRec *obs = a.obs + (size_t)w * a.Kcap;
    const LmRec *lms = a.lms + (size_t)w * a.Mcap;
    const double *rho = a.rho + (size_t)w * a.Mcap;
    const double *lm_scale = a.lm_scale + (size_t)w * a.Mcap;
    const LmAux *aux = a.lm_aux + (a.loop ? (size_t)a.ctrl[w].buf * a.bufs.lm_aux : 0) + (size_t)w * a.Mcap;
    double acc = 0.0;
    for (int ci = wv;; ci += 8) {
        const int ch = ci * gridDim.x + blockIdx.x;
        if (ch >= H.n_chunks) break;
        const int lm0 = H.chunk_begin[ch], cnt = H.chunk_meta[ch] & 0xff, anchor = H.chunk_meta[ch] >> 8;
        if (lane >= cnt) continue;
        const int l = lm0 + lane;
        const LmRec lr = lms[l];
        const int n_obs = lm_nobs(lr.meta);
        if (n_obs == 0) continue;
        double x[3];
        float xf[3], cl[3];
        world_point(F[anchor], lr.zrx, lr.zry, rho[l], x, xf, cl);
        const float ir = (float)(1.0 / rho[l]);
        // first pass: H_ll for the landmark's scaled direction, second pass: the products
        double hll = 0.0;
        for (unsigned j = 0, fm = lm_mask(lr.meta); j < (unsigned)n_obs; ++j, fm &= fm - 1) {
            const ObsRec o = obs[lr.obs_begin + j];
            const int of = __ffs(fm) - 1;
            float bt[3];
            baseline_in(F[of], F[anchor], bt);
            ObsLin ol;
            linearize_obs<true>(F[of], x, xf, ir, bt, o.zx, o.zy, W, cb, ol);
            hll += (double)(ol.j0 * ol.j0 + ol.j1 * ol.j1);
        }
        const double sc = lm_scale[l];
        double d2 = sc * sc * hll;
        d2 = fmin(fmax(d2, 1.0e-6), 1.0e32);
        const double vl = sc * sc * aux[l].gl / d2;
        for (unsigned j = 0, fm = lm_mask(lr.meta); j < (unsigned)n_obs; ++j, fm &= fm - 1) {
            const ObsRec o = obs[lr.obs_begin + j];
            const int of = __ffs(fm) - 1;
            float bt[3];
            baseline_in(F[of], F[anchor], bt);
            ObsLin ol;
            linearize_obs<true>(F[of], x, xf, ir, bt, o.zx, o.zy, W, cb, ol);
            double r0 = (double)ol.j0 * vl, r1 = (double)ol.j1 * vl;
#pragma unroll
            for (int i = 0; i < 6; ++i) {
                const double dv = vxi[of][i] - vxi[anchor][i];
                r0 += (double)ol.Y0[i] * dv; r1 += (double)ol.Y1[i] * dv;
            }
            acc += r0 * r0 + r1 * r1;
        }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
    if (lane == 0 && acc != 0.0) atomicAdd(&red, acc);
    __syncthreads();
    if (tid == 0 && red != 0.0) atomicAdd(a.acc + (size_t)w * kAcc + 9, red);
}

}  // namespace pvio
