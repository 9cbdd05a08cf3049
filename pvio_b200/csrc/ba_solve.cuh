// Reduced-system kernel: assembles the dense pose/velocity/bias system of one window and
// solves it.  One CTA per window.
//
//   * vision part: block-lower-triangular Schur-reduced system from schur_kernel (ba_schur.cuh) in xi
//     coordinates, mapped to the reference's local coordinates delta = [dtheta dp] with
//     H_delta[f,g] = T_f^T H_xi[f,g] T_g  (T_f = [[R_f,0],[-[p_f]x R_f,-I]])
//   * the IMU, prior and plane factors of ba_factors.cuh
//   * constant blocks (FF_FIX_POSE, bundle_adjustor.cpp:79-82), Jacobi scaling and the
//     mu*diag regulariser of ceres' dogleg Gauss-Newton solve, dense Cholesky, and the
//     scalars of the trust-region step.
// Everything here is fp64: it is O(D^3/6) flops on a D <= 210 system, off the HBM-bound path.
#pragma once
#include <type_traits>
#include "ba_factors.cuh"
#include "ba_lin.cuh"
#include "ba_tr.cuh"
#include "ba_chol.cuh"

namespace pvio {

struct SolveArgs : BatchArrays {
    int alias_bias;            // 1: dbg = dba = 0 at the linearisation point (quirk Q1)
    double *Hfull;             // optional [W][(15 Ncap)^2] dump of the reduced system (delta coords, before regularisation)
    double *gfull;             // optional [W][15 Ncap]
    int compute_scale;         // ignored when loop != 0 (then: WinCtrl::have_scale == 0)
    int w0;
    double mu_override;
    int loop;                  // 1: iteration of the device-side trust-region loop (ba_tr.cuh): obey the window's flags
};

constexpr int kSolveImuSlab = 15 * 30 + 16;     // raw J + r per factor
constexpr int kImuRound = 8;                    // IMU factors linearised concurrently by solve_kernel
constexpr int kImuJx = 15 * 32;                 // whitened Jacobian + residual column of one factor, row pitch 32

// Cov = NoCov: the reduced-system solve of solve_kernel / solve_kernel_visual.  Otherwise the body of the covariance
// kernel (ba_cov.cuh): window Cov::window(a), and once the system is assembled -- without regulariser, scaling or constant
// blocks -- Cov::finish takes over.
struct NoCov {};
template <bool kFull, class Cov = NoCov>
static __device__ __forceinline__ void solve_body(const SolveArgs &a) {
    constexpr bool kCov = !std::is_same<Cov, NoCov>::value;
    int w;
    if constexpr (kCov) w = Cov::window(a);
    else w = blockIdx.x + a.w0;
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int N = H.N;
    const int inertial = H.use_inertial;
    const int stride = inertial ? 15 : 6;
    // Visual-only windows: FF_FIX_POSE frames are constant parameter blocks (bundle_adjustor.cpp:82-87), so the
    // lean kernel leaves them out of the system altogether (cfg2: 48 instead of 60 unknowns, half the
    // factorisation); the full kernel keeps every frame (velocity / bias blocks stay free) and pins the pose rows.
    const unsigned allm = (1u << N) - 1u;
    const bool compact = !kFull && ((~(unsigned)H.fixed_mask) & allm) != 0u;
    const unsigned freem = compact ? (allm & ~(unsigned)H.fixed_mask) : allm;
    const int nfr = __popc(freem);
    const int D = stride * nfr;
    const int mask_c = compact ? 0 : H.fixed_mask;           // pose rows to pin, in the system's own frame numbering
    const int tid = threadIdx.x, nt = blockDim.x;
    const double *frames = a.frames + (size_t)w * a.Ncap * kFrameStride;
    WinCtrl &ctrl = a.ctrl[w];
    if (a.loop && (ctrl.done || ctrl.reuse)) return;         // finished, or the rejected step's linearisation is still valid
    const size_t bsel = a.loop ? (size_t)ctrl.buf : 0;       // buffer set holding the linearisation of the state (LinBufs)
    const int compute_scale = a.loop ? (ctrl.have_scale == 0) : a.compute_scale;
    const double mu = a.mu_override >= 0.0 ? a.mu_override : ctrl.mu;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int nb = (D + 3) >> 2, Dp = nb * 4;               // block rows of 4; rows >= D are identity padding
    const int nA = (nb + 1) * (nb + 2) / 2 * kTP;           // + the rhs block row
    double *A = reinterpret_cast<double *>(smem_raw);       // packed lower 4x4 tiles
    double *g = A + nA;                                     // [Dp] reduced gradient
    double *gu = g + Dp;                                    // [Dp] unreduced gradient (for |g|_inf)
    double *hcorr = gu + Dp;                                // [Dp] direct - reduced diagonal
    double *xs = hcorr + Dp;                                // [Dp] solution
    double *T = xs + Dp;                                    // [N][36] change of variables
    double *scr = T + N * 36;                               // scratch: staging / IMU slabs / prior vectors / reg copy
    __shared__ double cost_sm[4];
    __shared__ int flag_sm;

    SOLVE_STAMP(0);
    for (int i = tid; i < nA; i += nt) A[i] = 0.0;
    for (int i = tid; i < 4 * Dp; i += nt) g[i] = 0.0;      // g, gu, hcorr, xs contiguous
    if (tid < 4) cost_sm[tid] = 0.0;
    __shared__ double x2_sm[kMaxFrames];                    // |x|^2 of each frame's ambient parameter blocks
    if (tid < N) {
        const double *fs = frames + tid * kFrameStride;
        {   // ceres takes norms of the 4-vector quaternion; constant pose blocks are not parameters
            double x2 = 0.0;
            if (!((H.fixed_mask >> tid) & 1)) for (int k = 0; k < 7; ++k) x2 += fs[k] * fs[k];
            if (inertial) for (int k = 7; k < 16; ++k) x2 += fs[k] * fs[k];
            x2_sm[tid] = x2;
        }
        frame_T(fs, wc, T + tid * 36);
    }
    __syncthreads();
    const int npairs = N * (N + 1) / 2;
    const int npairs_cap = a.Ncap * (a.Ncap + 1) / 2;
    if (!kFull) {
        // Lean path (batched visual-only windows): no full staging of the xi blocks -- groups of 6 threads
        // pull one 6x6 block at a time through a small shared buffer, so that ~9 windows fit per SM.
        const double *Hred = a.Hred + bsel * a.bufs.Hred + (size_t)w * npairs_cap * 36;
        const double *Hdd = a.Hdd + bsel * a.bufs.Hdd + (size_t)w * a.Ncap * 36;
        const double *gdir = a.gdir + bsel * a.bufs.g + (size_t)w * a.Ncap * 6;
        const double *gred = a.gred + bsel * a.bufs.g + (size_t)w * a.Ncap * 6;
        double *Ms = scr + Dp;                       // [G][36]
        for (int e = tid; e < nfr * 6; e += nt) {    // direct diagonal diag(T_f^T Xd T_f)
            const int cf = e / 6, i = e - cf * 6;
            const int f = __fns(freem, 0, cf + 1);
            const double *Tf = T + f * 36, *X = Hdd + f * 36;
            double sd = 0.0;
            for (int aa = 0; aa < 6; ++aa) {
                double t = 0.0;
                for (int bb = 0; bb < 6; ++bb) t += X[aa * 6 + bb] * Tf[bb * 6 + i];
                sd += Tf[aa * 6 + i] * t;
            }
            hcorr[cf * stride + i] = sd;
        }
        const int G = nt / 6;
        const int q = tid / 6, i6 = tid - q * 6;
        const int npf = nfr * (nfr + 1) / 2;         // block pairs of the free frames
        for (int p0 = 0; p0 < npf; p0 += G) {
            const int p = p0 + q;
            const bool act = q < G && p < npf;
            int f = 0, gf = 0, cf = 0, cg = 0;
            if (act) {
                while ((cf + 1) * (cf + 2) / 2 <= p) ++cf;
                cg = p - cf * (cf + 1) / 2;
                f = __fns(freem, 0, cf + 1); gf = __fns(freem, 0, cg + 1);
                const double *X = Hred + (f * (f + 1) / 2 + gf) * 36 + i6 * 6, *Tg = T + gf * 36;
                double x[6];
#pragma unroll
                for (int bb = 0; bb < 6; ++bb) x[bb] = X[bb];
#pragma unroll
                for (int j = 0; j < 6; ++j) {
                    double v = 0.0;
#pragma unroll
                    for (int bb = 0; bb < 6; ++bb) v += x[bb] * Tg[bb * 6 + j];
                    Ms[q * 36 + i6 * 6 + j] = v;       // M = X T_g, row i6
                }
            }
            __syncthreads();
            if (act) {
                const double *Tf = T + f * 36;
                const int j = i6;                        // this thread produces column j of T_f^T M
#pragma unroll
                for (int i = 0; i < 6; ++i) {
                    if (cf == cg && j > i) continue;
                    double sv = 0.0;
#pragma unroll
                    for (int aa = 0; aa < 6; ++aa) sv += Tf[aa * 6 + i] * Ms[q * 36 + aa * 6 + j];
                    const int gi = cf * stride + i, gj = cg * stride + j;
                    A[tri(gi, gj)] = sv;
                    if (cf == cg && i == j) hcorr[gi] -= sv;
                }
            }
            __syncthreads();
        }
        for (int e = tid; e < nfr * 6; e += nt) {
            const int cf = e / 6, i = e - cf * 6;
            const int f = __fns(freem, 0, cf + 1);
            const double *Tf = T + f * 36;
            double sr = 0.0, sd = 0.0;
            for (int aa = 0; aa < 6; ++aa) { sr += Tf[aa * 6 + i] * gred[f * 6 + aa]; sd += Tf[aa * 6 + i] * gdir[f * 6 + aa]; }
            g[cf * stride + i] = sr;
            gu[cf * stride + i] = sd;
        }
    } else
    // ---- vision blocks: H_delta[f,gf] = T_f^T X T_g.  Stage the xi-coordinate blocks in shared
    // memory (coalesced), X <- X T_g in place, then T_f^T (X T_g) into the packed system.
    {
        const double *Hred = a.Hred + bsel * a.bufs.Hred + (size_t)w * npairs_cap * 36;
        const double *Hdd = a.Hdd + bsel * a.bufs.Hdd + (size_t)w * a.Ncap * 36;
        const double *gdir = a.gdir + bsel * a.bufs.g + (size_t)w * a.Ncap * 6;
        const double *gred = a.gred + bsel * a.bufs.g + (size_t)w * a.Ncap * 6;
        double *Xs = scr;                        // [npairs][36]
        double *Xd = Xs + npairs * 36;           // [N][36]
        double *gx = Xd + N * 36;                // [2][N][6]
        for (int i = tid; i < npairs * 36; i += nt) Xs[i] = Hred[i];
        for (int i = tid; i < N * 36; i += nt) Xd[i] = Hdd[i];
        for (int i = tid; i < N * 6; i += nt) { gx[i] = gred[i]; gx[N * 6 + i] = gdir[i]; }
        __syncthreads();
        // direct (pre-Schur) diagonal, for the Jacobi scaling / LM diagonal: diag(T_f^T Xd T_f)
        for (int e = tid; e < N * 6; e += nt) {
            const int f = e / 6, i = e - f * 6;
            const double *Tf = T + f * 36, *X = Xd + f * 36;
            double sd = 0.0;
            for (int aa = 0; aa < 6; ++aa) {
                double t = 0.0;
                for (int bb = 0; bb < 6; ++bb) t += X[aa * 6 + bb] * Tf[bb * 6 + i];
                sd += Tf[aa * 6 + i] * t;
            }
            hcorr[f * stride + i] = sd;
        }
        // M = X T_g into a second buffer (one barrier; the in-place form needed two per pass of 252 entries), then
        // T_f^T M into the packed system
        double *Ms = gx + 2 * N * 6;             // [npairs][36]
        for (int e = tid; e < npairs * 36; e += nt) {
            const int p = e / 36, ij = e - p * 36, i = ij / 6, j = ij - i * 6;
            int f = 0;
            while ((f + 1) * (f + 2) / 2 <= p) ++f;
            const int gf = p - f * (f + 1) / 2;
            const double *X = Xs + p * 36 + i * 6, *Tg = T + gf * 36 + j;
            double v = 0.0;
#pragma unroll
            for (int bb = 0; bb < 6; ++bb) v += X[bb] * Tg[bb * 6];
            Ms[e] = v;
        }
        __syncthreads();
        for (int e = tid; e < npairs * 36; e += nt) {
            const int p = e / 36, ij = e - p * 36, i = ij / 6, j = ij - i * 6;
            int f = 0;
            while ((f + 1) * (f + 2) / 2 <= p) ++f;
            const int gf = p - f * (f + 1) / 2;
            if (f == gf && j > i) continue;
            const double *Tf = T + f * 36 + i, *Mx = Ms + p * 36 + j;
            double sv = 0.0;
#pragma unroll
            for (int aa = 0; aa < 6; ++aa) sv += Tf[aa * 6] * Mx[aa * 6];
            const int gi = f * stride + i, gj = gf * stride + j;
            A[tri(gi, gj)] = sv;
            if (f == gf && i == j) hcorr[gi] -= sv;     // direct - reduced diagonal
        }
        for (int e = tid; e < N * 6; e += nt) {
            const int f = e / 6, i = e - f * 6;
            const double *Tf = T + f * 36;
            double sr = 0.0, sd = 0.0;
            for (int aa = 0; aa < 6; ++aa) { sr += Tf[aa * 6 + i] * gx[f * 6 + aa]; sd += Tf[aa * 6 + i] * gx[N * 6 + f * 6 + aa]; }
            g[f * stride + i] = sr;
            gu[f * stride + i] = sd;
        }
    }
    __syncthreads();
    SOLVE_STAMP(1);
    const WinFactors F(a, w);
    // ---- IMU factors (bundle_adjustor.cpp:220-242): no loss
    if (kFull && inertial && F.n_imu() > 0) {
        for (int n0 = 0; n0 < F.n_imu(); n0 += kImuRound) {  // up to kImuRound factors per round (scratch: raw + whitened J of each)
            const int nb = min(kImuRound, F.n_imu() - n0);
            double *Jraw = scr;                              // [R][450], r at [R*450 + n*16]
            double *rraw = scr + kImuRound * 450;
            double *Jx = rraw + kImuRound * 16;              // [R][15][32] whitened [J | r | 0]
            double *Wsm = Jx + kImuRound * kImuJx;           // [R][225] sqrt information matrices of the round
            __shared__ int imu_fr[2 * kImuRound];            // frame pair of each factor of the round (read in every inner loop)
            __shared__ int imu_chain;
            __shared__ double imu_cost[kImuRound];           // r^T r of each factor of the round
            if (tid >= 32 && tid < 32 + 2 * nb) imu_fr[tid - 32] = F.imu_idx()[2 * n0 + tid - 32];
            if (tid < nb) {
                const int n = n0 + tid;
                imu_factor_raw(frames + F.imu_idx()[2 * n] * kFrameStride, frames + F.imu_idx()[2 * n + 1] * kFrameStride,
                               F.imu_rec() + (size_t)n * kImuStride, wc, a.alias_bias, rraw + tid * 16, Jraw + tid * 450);
            } else if (tid >= 32) {
                // the other warps meanwhile stage W (one coalesced pass instead of 15 L2 loads per whitened entry)
                for (int e = tid - 32; e < nb * 225; e += nt - 32) {      // (lanes nb..31 of warp 0 idle with the factor threads)
                    const int n = e / 225;
                    Wsm[e] = __ldg(F.imu_rec() + (size_t)(n0 + n) * kImuStride + 11 + (e - n * 225));
                }
            }
            __syncthreads();
            SOLVE_STAMP(2);
            // whiten: Jx = [W J | W r | 0] (15 x 32 per factor)      :157 and the "sqrt_inv_cov *" lines
            // One thread per COLUMN of a factor: the raw column sits in registers, the rows of W are broadcast loads --
            // one shared-memory load per multiply-add instead of two (the entry-per-thread form was shared-memory bound).
            for (int e = tid; e < nb * 32; e += nt) {
                const int n = e >> 5, col = e & 31;
                double *out = Jx + n * kImuJx + col;
                if (col == 31) { for (int row = 0; row < 15; ++row) out[row * 32] = 0.0; continue; }
                double cv[15];
#pragma unroll
                for (int k = 0; k < 15; ++k) cv[k] = col < 30 ? Jraw[n * 450 + k * 30 + col] : rraw[n * 16 + k];
                const double *Wm = Wsm + n * 225;
                for (int row = 0; row < 15; ++row) {
                    double s = 0.0;
#pragma unroll
                    for (int k = 0; k < 15; ++k) s += Wm[row * 15 + k] * cv[k];
                    out[row * 32] = s;
                }
            }
            if (tid == 0) {
                bool ch = true;                              // no two factors of equal parity share a frame
                for (int n = 0; n < nb && ch; ++n)
                    for (int m = n + 2; m < nb; m += 2) {
                        const int a0 = imu_fr[2 * n], a1 = imu_fr[2 * n + 1], b0 = imu_fr[2 * m], b1 = imu_fr[2 * m + 1];
                        ch &= (a0 != b0 && a0 != b1 && a1 != b0 && a1 != b1);
                    }
                imu_chain = ch ? 1 : 0;
            }
            __syncthreads();
            // accumulate Jx^T Jx: rows / columns 0..29 are the 30 x 30 block of the system, row 30 the gradient, entry
            // (30, 30) twice the cost.  One thread per 4 x 4 tile of the lower triangle (36 tiles per factor), 15 steps of
            // 2 x 4 loaded values for 16 multiply-adds.  Two factors touch the same entries of the system only if they
            // share a frame; the reference's factors form a chain (frame n, n + 1), so the factors at even positions of
            // the round go first, all at once, then the odd ones.  Any other round: one factor at a time.
            const bool chain = imu_chain != 0;
            const int phases = chain ? 2 : nb;
            for (int ph = 0; ph < phases; ++ph) {
                const int first = ph, step = chain ? 2 : nb, cnt = chain ? (nb - ph + 1) / 2 : 1;
                for (int e = tid; e < cnt * 36; e += nt) {
                    const int q = e / 36, t = e - q * 36;
                    const int n = first + q * step;
                    int tr = 0;
                    while ((tr + 1) * (tr + 2) / 2 <= t) ++tr;
                    const int tc = t - tr * (tr + 1) / 2;    // tile (tr, tc), tc <= tr < 8
                    const double *Jn = Jx + n * kImuJx;
                    double acc[4][4];
#pragma unroll
                    for (int i = 0; i < 4; ++i)
#pragma unroll
                        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;
#pragma unroll 5
                    for (int k = 0; k < 15; ++k) {
                        const double2 a0 = *reinterpret_cast<const double2 *>(Jn + k * 32 + 4 * tr);
                        const double2 a1 = *reinterpret_cast<const double2 *>(Jn + k * 32 + 4 * tr + 2);
                        const double2 b0 = *reinterpret_cast<const double2 *>(Jn + k * 32 + 4 * tc);
                        const double2 b1 = *reinterpret_cast<const double2 *>(Jn + k * 32 + 4 * tc + 2);
                        const double av[4] = {a0.x, a0.y, a1.x, a1.y}, bv[4] = {b0.x, b0.y, b1.x, b1.y};
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int j = 0; j < 4; ++j) acc[i][j] += av[i] * bv[j];
                    }
                    const int fi = imu_fr[2 * n], fj = imu_fr[2 * n + 1];
#pragma unroll
                    for (int i = 0; i < 4; ++i) {
                        const int ra = 4 * tr + i;
                        if (ra > 30) continue;
#pragma unroll
                        for (int j = 0; j < 4; ++j) {
                            const int cb_ = 4 * tc + j;
                            if (cb_ > ra || cb_ > 30) continue;          // the lower triangle of the 31 x 31 product, once
                            const double v = acc[i][j];
                            if (ra == 30) {
                                if (cb_ == 30) imu_cost[n] = v;
                                else { const int gb = (cb_ < 15 ? fi * 15 + cb_ : fj * 15 + cb_ - 15); g[gb] += v; gu[gb] += v; }
                            } else {
                                const int ga = (ra < 15 ? fi * 15 + ra : fj * 15 + ra - 15);
                                const int gb = (cb_ < 15 ? fi * 15 + cb_ : fj * 15 + cb_ - 15);
                                A[ga >= gb ? tri(ga, gb) : tri(gb, ga)] += v;
                            }
                        }
                    }
                }
                __syncthreads();
            }
            if (tid == 0) {                                  // in factor order: the cost does not depend on the schedule
                double c = 0.0;
                for (int n = 0; n < nb; ++n) c += imu_cost[n];
                cost_sm[1] += 0.5 * c;
            }
        }
    }

    SOLVE_STAMP(3);
    // ---- marginalisation prior (bundle_adjustor.cpp:126-139): no loss
    if (kFull && inertial && F.n_prior() > 0) {
        const int n = F.n_prior(), d = F.d();
        const double *S = F.prior_S();
        double *r0 = scr;                 // [d] raw residual
        double *rr = r0 + d;              // [d] r = S r0 + e
        double *vv = rr + d;              // [d] S^T r
        double *Ji = vv + d;              // [n][9] Jr^-1
        double *Bs = Ji + 9 * n;          // [warps][225] block staging of the Hessian pass
        __shared__ int pf_s[kMaxFrames];
        if (tid >= 32 && tid < 32 + n) pf_s[tid - 32] = F.prior_frames()[tid - 32];
        if (tid < n)
            prior_frame_raw(frames + F.prior_frames()[tid] * kFrameStride, F.prior_x0() + tid * kFrameStride, r0 + 15 * tid, Ji + 9 * tid);
        __syncthreads();
        prior_residual(S, F.prior_e(), r0, d, [=](int i, double r) { rr[i] = r; });
        __syncthreads();
        for (int i = tid; i < d; i += nt) {                    // S^T r: column i, the loads of 8 rows ahead of the sum
            double s = 0.0;
            int k = 0;
            for (; k + 8 <= d; k += 8) {
                double sv[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) sv[u] = __ldg(S + (size_t)(k + u) * d + i);
#pragma unroll
                for (int u = 0; u < 8; ++u) s += sv[u] * rr[k + u];
            }
            for (; k < d; ++k) s += __ldg(S + (size_t)k * d + i) * rr[k];
            vv[i] = s;
        }
        if (tid == 0) { double c = 0.0; for (int k = 0; k < d; ++k) c += rr[k] * rr[k]; cost_sm[2] = 0.5 * c; }
        __syncthreads();
        SOLVE_STAMP(4);
        // g += E^T vv ; H += E^T Lambda E  with E = blockdiag(Jr^-1, I, I, I, I) per frame  (:72-88)
        prior_grad(Ji, vv, d, pf_s, [=](int gi, double s) { g[gi] += s; gu[gi] += s; });
        // H += E^T Lambda E by 15 x 15 frame blocks, one warp per block (fi, fj) of the lower triangle: the block of
        // Lambda comes in with 8 loads per lane in flight at once (the per-entry loop it replaces was a chain of exposed
        // L2 round trips), the Jr^-1 factors are applied to its first three columns, then rows, in shared memory
        {
            const int lane = tid & 31, wp = tid >> 5, nw = nt >> 5;
            double *B = Bs + wp * 225;
            for (int blk = wp; blk < n * n; blk += nw) {
                const int fi = blk / n, fj = blk - fi * n;
                const int gfi = pf_s[fi], gfj = pf_s[fj];
                if (gfj > gfi) continue;                              // (warp-uniform) the transposed block covers it
                double lv[8];
#pragma unroll
                for (int u = 0; u < 8; ++u) {
                    const int e = lane + 32 * u;
                    const int r = e / 15, c = e - r * 15;
                    lv[u] = e < 225 ? __ldg(F.prior_L() + (size_t)(15 * fi + r) * d + 15 * fj + c) : 0.0;
                }
#pragma unroll
                for (int u = 0; u < 8; ++u) if (lane + 32 * u < 225) B[lane + 32 * u] = lv[u];
                __syncwarp();
                double t0 = 0.0, t1 = 0.0;                            // columns 0..2 <- B[:, 0..2] Jr_j^-1
                {
                    const double *Jj = Ji + 9 * fj;
                    const int e0 = lane, e1 = lane + 32;              // 45 outputs (r, cj)
                    if (e0 < 45) { const int r = e0 / 3, cj = e0 - r * 3; for (int m = 0; m < 3; ++m) t0 += B[r * 15 + m] * Jj[3 * m + cj]; }
                    if (e1 < 45) { const int r = e1 / 3, cj = e1 - r * 3; for (int m = 0; m < 3; ++m) t1 += B[r * 15 + m] * Jj[3 * m + cj]; }
                    __syncwarp();
                    if (e0 < 45) B[(e0 / 3) * 15 + e0 % 3] = t0;
                    if (e1 < 45) B[(e1 / 3) * 15 + e1 % 3] = t1;
                    __syncwarp();
                }
                {
                    const double *Jf = Ji + 9 * fi;                   // rows 0..2 <- Jr_i^-T B[0..2, :]
                    const int e0 = lane, e1 = lane + 32;              // 45 outputs (ci, c)
                    t0 = 0.0; t1 = 0.0;
                    if (e0 < 45) { const int ci = e0 / 15, c = e0 - ci * 15; for (int k = 0; k < 3; ++k) t0 += Jf[3 * k + ci] * B[k * 15 + c]; }
                    if (e1 < 45) { const int ci = e1 / 15, c = e1 - ci * 15; for (int k = 0; k < 3; ++k) t1 += Jf[3 * k + ci] * B[k * 15 + c]; }
                    __syncwarp();
                    if (e0 < 45) B[e0] = t0;
                    if (e1 < 45) B[e1] = t1;
                    __syncwarp();
                }
                for (int e = lane; e < 225; e += 32) {                // each (gi, gj) has a unique owner: prior frames are distinct
                    const int r = e / 15, c = e - r * 15;
                    if (fi == fj && c > r) continue;
                    A[tri(gfi * 15 + r, gfj * 15 + c)] += B[e];
                }
                __syncwarp();
            }
        }
        __syncthreads();
    }

    SOLVE_STAMP(5);
    // ---- plane factors (bundle_adjustor.cpp:162-196): CauchyLoss
    if (kFull && F.n_ptracks() > 0) {
        const double cb = F.cb();
        // thread per track: the corrected 1 x 6K Jacobian row, spread over the window's frames (zeros where the track has
        // no observation), and the corrected residual go to a scratch row; then thread per ENTRY of the pose block of the
        // system sums over the tracks -- no atomics (fp64 atomicAdd on shared memory is a compare-and-swap loop, and all
        // tracks of a plane hit the same frames: the atomic version took 600 us of the kernel's 820 on cfg4)
        const int PW = 6 * N + 2;                                   // row: [6 N] Jacobian, residual
        // the rows live in the kernel's shared scratch when they fit (inertial windows: the IMU slabs are free again),
        // otherwise in the per-window global scratch
        unsigned dyn_bytes;
        asm("mov.u32 %0, %%dynamic_smem_size;" : "=r"(dyn_bytes));
        const size_t scr_words = dyn_bytes / sizeof(double) - (size_t)(scr - reinterpret_cast<double *>(smem_raw));
        double *PJ = (size_t)F.n_ptracks() * PW <= scr_words ? scr : a.pt_J + (size_t)w * a.Tcap * (6 * a.Ncap + 2);
        for (int t = tid; t < F.n_ptracks(); t += nt) {
            const int b0 = F.pt_begin()[t], K = F.pt_begin()[t + 1] - b0;
            double r, J[6 * kMaxFrames];
            plane_factor(K, F.pt_frame() + b0, F.pt_z() + 2 * b0, frames, wc, F.plane() + 4 * F.pt_plane()[t], wc.plane_sic, &r, J);
            const double s = r * r, tt = 1.0 + s / cb;
            const double sc = sqrt(1.0 / tt);
            atomicAdd(&cost_sm[3], 0.5 * cb * log(tt));
            double *row = PJ + (size_t)t * PW;
            for (int i = 0; i < 6 * N; ++i) row[i] = 0.0;
            for (int i = 0; i < 6 * K; ++i) row[F.pt_frame()[b0 + i / 6] * 6 + (i % 6)] = J[i] * sc;
            row[6 * N] = r * sc;
        }
        __syncthreads();
        const int P6 = 6 * N, T = F.n_ptracks();
        for (int e = tid; e < P6 * (P6 + 1) / 2 + P6; e += nt) {
            if (e >= P6 * (P6 + 1) / 2) {                            // gradient entries
                const int i = e - P6 * (P6 + 1) / 2;
                double sg = 0.0;
                for (int t = 0; t < T; ++t) sg += PJ[(size_t)t * PW + i] * PJ[(size_t)t * PW + P6];
                const int gi = (i / 6) * stride + (i % 6);
                g[gi] += sg; gu[gi] += sg;
                continue;
            }
            int i = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
            while ((i + 1) * (i + 2) / 2 <= e) ++i;
            while (i * (i + 1) / 2 > e) --i;
            const int j = e - i * (i + 1) / 2;                       // j <= i
            double sh = 0.0;
            for (int t = 0; t < T; ++t) sh += PJ[(size_t)t * PW + i] * PJ[(size_t)t * PW + j];
            const int gi = (i / 6) * stride + (i % 6), gj = (j / 6) * stride + (j % 6);
            A[tri(gi, gj)] += sh;                                    // gi >= gj since i >= j
        }
        __syncthreads();
    }

    // ---- optional dump of the assembled reduced system (delta coordinates, no regulariser)
    if (a.Hfull) {
        const int Df = 15 * a.Ncap;
        double *Ho = a.Hfull + (size_t)w * Df * Df, *go = a.gfull + (size_t)w * Df;
        for (int e = tid; e < D * D; e += nt) {
            const int i = e / D, j = e - i * D;
            int fi = i / stride, fj = j / stride;
            const int ci = i - fi * stride, cj = j - fj * stride;
            if (compact) { fi = __fns(freem, 0, fi + 1); fj = __fns(freem, 0, fj + 1); }     // back to the window's frame ids
            Ho[(size_t)(fi * 15 + ci) * Df + fj * 15 + cj] = (i >= j) ? A[tri(i, j)] : A[tri(j, i)];
        }
        for (int i = tid; i < D; i += nt) {
            const int fi = i / stride;
            go[(compact ? __fns(freem, 0, fi + 1) : fi) * 15 + (i % stride)] = g[i];
        }
    }
    if constexpr (kCov) {
        __syncthreads();
        Cov::finish(a, w, N, stride, D, nb, A, hcorr, gu, xs, T, scr, &flag_sm);
        return;
    }
    SOLVE_STAMP(6);
    // ---- Jacobi scale, LM diagonal, constant blocks
    double *scale = a.pose_scale + (size_t)w * 15 * a.Ncap;
    double my_gdx = 0.0;
    for (int i = tid; i < D; i += nt) {
        const int f = i / stride, c = i - f * stride;
        const double hii = A[tri(i, i)] + hcorr[i];          // diagonal of the UNREDUCED J^T J
        double sc;
        if (compute_scale) { sc = 1.0 / (1.0 + sqrt(fmax(hii, 0.0))); scale[i] = sc; }
        else sc = scale[i];
        const double reg = mu > 0.0 ? lm_reg(hii, sc, mu) : 0.0;
        xs[i] = reg;                                          // keep reg for the scalars below
        A[tri(i, i)] += reg;
        hcorr[i] = hii;                                       // now holds the unreduced diagonal
    }
    __syncthreads();
    const int fixed_mask = mask_c;
    {
        // identity rows / columns for the pinned unknowns: the pose rows of constant frames and the padding rows >= D.
        // Work item (q, j): the q-th pinned index m against column j; a pair of pinned indices is written by the larger one.
        const unsigned fm = (unsigned)fixed_mask & ((1u << nfr) - 1u);
        const int nfix6 = 6 * __popc(fm), npin = nfix6 + (Dp - D);
        for (int e = tid; e < npin * Dp; e += nt) {
            const int q = e / Dp, j = e - q * Dp;
            int m;
            if (q < nfix6) { const int fq = q / 6; m = __fns(fm, 0, fq + 1) * stride + (q - fq * 6); }
            else m = D + (q - nfix6);
            const int fj = j / stride;
            const bool pj = j >= D || (((fm >> fj) & 1u) && (j - fj * stride) < 6);
            if (pj && j > m) continue;
            A[j > m ? tri(j, m) : tri(m, j)] = (j == m) ? 1.0 : 0.0;
        }
    }
    double *reg_keep = scr;       // [D]
    for (int i = tid; i < D; i += nt) {
        const int f = i / stride, c = i - f * stride;
        const bool m = ((fixed_mask >> f) & 1) && c < 6;
        reg_keep[i] = xs[i];
        if (m) { g[i] = 0.0; gu[i] = 0.0; }
        xs[i] = -g[i];
    }
    __syncthreads();
    SOLVE_STAMP(7);
    const bool ok = chol_solve<kFull>(A, xs, nb, &flag_sm);
    SOLVE_STAMP(8);

    // ---- outputs
    double *dxo = a.dx_pose + (size_t)w * a.Ncap * 15;
    for (int i = tid; i < N * 15; i += nt) {
        const int f = i / 15, c = i - f * 15;
        const bool in_sys = (freem >> f) & 1u;               // dropped (constant) frames do not move
        dxo[i] = (ok && c < stride && in_sys) ? xs[__popc(freem & ((1u << f) - 1u)) * stride + c] : 0.0;
    }
    {
        double gdx = 0.0, rdx = 0.0, gn2 = 0.0, dx2 = 0.0, gmax = 0.0, g2 = 0.0, vrd = 0.0;
        double *vpo = a.v_pose + (size_t)w * a.Ncap * 15;
        for (int i = tid; i < N * 15; i += nt) vpo[i] = 0.0;
        for (int i = tid; i < D; i += nt) {
            const int f = i / stride, c = i - f * stride;
            const bool m = ((fixed_mask >> f) & 1) && c < 6;
            if (m) continue;
            const double dx = ok ? xs[i] : 0.0;
            const double sc = scale[i];
            double d2 = sc * sc * hcorr[i];
            d2 = fmin(fmax(d2, 1.0e-6), 1.0e32);
            // NOTE: the reduced gradient g and the unreduced gu differ only through the Schur term;
            // g . dx over the full system is completed by the landmark sweep (acc[1])
            const double v = sc * sc * gu[i] / d2;
            vpo[(compact ? __fns(freem, 0, f + 1) : f) * 15 + c] = v;
            gdx += g[i] * dx;
            rdx += reg_keep[i] * dx * dx;
            gn2 += d2 * (dx / sc) * (dx / sc);
            dx2 += dx * dx;
            g2 += v * gu[i];
            vrd += v * reg_keep[i] * dx;
            gmax = fmax(gmax, fabs(gu[i]));
        }
        __syncthreads();
        double *red = A;                 // the factor is no longer needed
        if (tid < D) { red[tid * 7 + 0] = gdx; red[tid * 7 + 1] = rdx; red[tid * 7 + 2] = gn2; red[tid * 7 + 3] = dx2; red[tid * 7 + 4] = gmax;
                       red[tid * 7 + 5] = g2; red[tid * 7 + 6] = vrd; }
        __syncthreads();
        if (tid < 32) {                  // warp 0: strided partial sums, then a shuffle tree (fixed order: reproducible)
            gdx = rdx = gn2 = dx2 = gmax = g2 = vrd = 0.0;
            const int nred = min(nt, D);
            for (int t = tid; t < nred; t += 32) {
                gdx += red[t * 7]; rdx += red[t * 7 + 1]; gn2 += red[t * 7 + 2]; dx2 += red[t * 7 + 3];
                gmax = fmax(gmax, red[t * 7 + 4]); g2 += red[t * 7 + 5]; vrd += red[t * 7 + 6];
            }
#pragma unroll
            for (int off = 16; off > 0; off >>= 1) {
                gdx += __shfl_xor_sync(0xffffffffu, gdx, off); rdx += __shfl_xor_sync(0xffffffffu, rdx, off);
                gn2 += __shfl_xor_sync(0xffffffffu, gn2, off); dx2 += __shfl_xor_sync(0xffffffffu, dx2, off);
                gmax = fmax(gmax, __shfl_xor_sync(0xffffffffu, gmax, off));
                g2 += __shfl_xor_sync(0xffffffffu, g2, off); vrd += __shfl_xor_sync(0xffffffffu, vrd, off);
            }
        }
        if (tid == 0) {
            ctrl.grad2 = g2;
            ctrl.v_reg_dx = vrd;
            double x2 = 0.0;
            for (int f = 0; f < N; ++f) x2 += x2_sm[f];
            ctrl.g_dot_dx = gdx;
            ctrl.dx_reg_dx = rdx;
            ctrl.gn_norm2 = gn2;
            ctrl.dxnorm2 = dx2;
            ctrl.xnorm2 = x2;
            ctrl.gmax = gmax;
            const double cv = a.cost_vis[bsel * a.bufs.cost + w];
            ctrl.cost_vis = cv;
            ctrl.cost = cv + cost_sm[1] + cost_sm[2] + cost_sm[3];
            ctrl.have_lin = 1;
            ctrl.solve_failed = ok ? 0 : 1;
            if (compute_scale) ctrl.have_scale = 1;
            ctrl.fresh = 1;
        }
    }
    // plain step: clear the scalars the back-substitution sweep adds to (in the loop it stores them, ba_update.cuh)
    if (!a.loop && tid < kAcc) a.acc[(size_t)w * kAcc + tid] = 0.0;
    SOLVE_STAMP(9);
}

static __global__ void __launch_bounds__(256) solve_kernel(SolveArgs a) { solve_body<true>(a); }
// visual-only windows (no IMU / prior / plane factors): small register footprint, many CTAs per SM
static __global__ void __launch_bounds__(64, 10) solve_kernel_visual(SolveArgs a) { solve_body<false>(a); }

// Non-vision part of the cost at the candidate state (IMU + prior + plane), one CTA per window.
struct CostArgs : BatchArrays {
    int alias_bias;                // 1: candidate dbg = cand.bg - current.bg
    int w0;
    int loop;                      // 1: tr_decide (device-side trust-region loop); 0: plain Gauss-Newton step, `apply` decides
    int apply;
    double beta;                   // loop == 0: the step was beta * dx_gn (model change of the truncated step)
};

// kPart 0: cost of the IMU / prior / plane blocks at the candidate + the step decision (one launch, batches);
// 1: the cost only (-> a.aux_cost[w]); 2: the decision only, cost read from a.aux_cost[w].  The latency path launches part 1
// on a parallel branch of the solve graph, beside the candidate's linearisation sweep: both only need the candidate.  In the
// loop the candidate's reprojection cost is in the window's OTHER buffer set of cost_vis.
template <int kPart>
static __global__ void aux_cost_kernel(CostArgs a) {
    const int w = blockIdx.x + a.w0;
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int tid = threadIdx.x, nt = blockDim.x;
    const double *fc = a.frames_cand + (size_t)w * a.Ncap * kFrameStride;
    const double *fcur = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinFactors F(a, w);
    __shared__ double acc;
    __shared__ int accept_sm;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *r0 = reinterpret_cast<double *>(smem_raw);
    WinCtrl &ctrl = a.ctrl[w];
    if (a.loop && (ctrl.done || ctrl.skip)) { if (tid == 0 && kPart != 1) ctrl.fresh = 0; return; }
    if (tid == 0) acc = kPart == 2 ? a.aux_cost[w] : 0.0;
    __syncthreads();
    if (kPart != 2 && H.use_inertial) {
        __shared__ double imu_c[kMaxFrames];
        const int n_pr = F.n_prior(), d = 15 * n_pr;
        double *rc = r0 + 15 * kMaxFrames;                    // [d] squared whitened prior residuals
        for (int n = tid; n < F.n_imu(); n += nt) {
            // residual only: the raw evaluator without Jacobian.  Q1 (alias_bias): the bias linearisation point is the
            // CURRENT (accepted) bias of frame i while the state is the candidate
            double r[15];
            const double *rec = F.imu_rec() + (size_t)n * kImuStride;
            imu_factor_raw(fc + F.imu_idx()[2 * n] * kFrameStride, fc + F.imu_idx()[2 * n + 1] * kFrameStride, rec, wc, 0, r, nullptr,
                           a.alias_bias ? fcur + F.imu_idx()[2 * n] * kFrameStride + 10 : nullptr);
            imu_c[n] = imu_whitened_norm2(rec, r);
        }
        {   // the prior's raw residuals meanwhile on the second warp (a CTA of one warp: after the IMU factors)
            const int pt = nt > 32 ? tid - 32 : tid;
            double Ji[9];
            if (pt >= 0 && pt < n_pr)
                prior_frame_raw(fc + F.prior_frames()[pt] * kFrameStride, F.prior_x0() + pt * kFrameStride, r0 + 15 * pt, Ji);
        }
        __syncthreads();
        if (n_pr > 0) {
            prior_residual(F.prior_S(), F.prior_e(), r0, d, [=](int i, double r) { rc[i] = r * r; });
            __syncthreads();
        }
        if (tid == 0) {                                        // fixed summation order: the cost is reproducible
            double c = 0.0;
            for (int n = 0; n < F.n_imu(); ++n) c += imu_c[n];
            double cp = 0.0;
            for (int i = 0; i < d; ++i) cp += rc[i];
            acc += 0.5 * c + 0.5 * cp;
        }
        __syncthreads();
    }
    if (kPart != 2 && F.n_ptracks() > 0) {
        const double cb = F.cb();
        for (int t = tid; t < F.n_ptracks(); t += nt) {
            const int b0 = F.pt_begin()[t], K = F.pt_begin()[t + 1] - b0;
            double r, J[6 * kMaxFrames];
            plane_factor(K, F.pt_frame() + b0, F.pt_z() + 2 * b0, fc, wc, F.plane() + 4 * F.pt_plane()[t], wc.plane_sic, &r, J);
            atomicAdd(&acc, 0.5 * cb * log(1.0 + r * r / cb));
        }
    }
    __syncthreads();
    if (kPart == 1) { if (tid == 0) a.aux_cost[w] = acc; return; }
    // ---- step acceptance: what ceres does after evaluating the candidate (trust_region_minimizer.cc)
    if (tid == 0) {
        a.aux_cost[w] = acc;
        const double *av = a.acc + (size_t)w * kAcc;
        bool accept;
        if (a.loop) {
            WinCtrl c = ctrl;                   // one round trip of the record instead of a dependent chain of global accesses
            accept = tr_decide(c, av, a.cost_vis[(size_t)(1 - c.buf) * a.bufs.cost + w], acc);
            if (accept) c.buf ^= 1;             // the candidate's linearisation becomes the state's
            ctrl = c;
        }
        else {
            ctrl.cand_cost_vis = av[0];
            ctrl.cand_cost = av[0] + acc;
            const double gdx = ctrl.g_dot_dx + av[1];           // g . dx over poses + landmarks (full GN step)
            const double rdx = ctrl.dx_reg_dx + av[2];          // dx^T (mu D) dx
            // model cost change of the step beta * dx_gn:  -(beta g.dx + beta^2/2 dx^T H dx),
            // with dx^T H dx = -g.dx - dx^T (mu D) dx for the regularised Gauss-Newton step
            ctrl.model_change = -a.beta * gdx + 0.5 * a.beta * a.beta * (gdx + rdx);
            accept = a.apply != 0;
        }
        accept_sm = accept ? 1 : 0;
    }
    __syncthreads();
    if (accept_sm) {             // the candidate becomes the state
        const int N = H.N, M = H.M;
        for (int i = tid; i < N * kFrameStride; i += nt) a.frames[(size_t)w * a.Ncap * kFrameStride + i] = fc[i];
        for (int i = tid; i < M; i += nt) a.rho[(size_t)w * a.Mcap + i] = a.rho_cand[(size_t)w * a.Mcap + i];
    }
}

// |J v|^2 over the IMU / prior / plane blocks (loss-corrected) at the current state, one CTA per window, into acc slot 10:
// the non-vision part of the Cauchy-point denominator of the dogleg step.  a.loop != 0: runs only for windows whose GN
// step left the trust region, then picks the dogleg step (tr_after_jv).
static __global__ void jv_aux_kernel(CostArgs a) {
    const int w = blockIdx.x + a.w0;
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int tid = threadIdx.x, nt = blockDim.x;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const double *v = a.v_pose + (size_t)w * a.Ncap * 15;
    const WinFactors F(a, w);
    __shared__ double acc;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    double *ev = reinterpret_cast<double *>(smem_raw);      // [15 n_prior] E v
    WinCtrl &ctrl = a.ctrl[w];
    if (a.loop && (ctrl.done || ctrl.skip)) return;
    if (a.loop && !ctrl.need_jv) { if (tid == 0) { WinCtrl c = ctrl; tr_after_jv(c, a.acc + (size_t)w * kAcc); ctrl = c; } return; }
    if (tid == 0) acc = 0.0;
    __syncthreads();
    if (H.use_inertial) {
        for (int n = tid; n < F.n_imu(); n += nt) {
            double r[15], J[450], u[15];
            const double *rec = F.imu_rec() + (size_t)n * kImuStride;
            const int fi = F.imu_idx()[2 * n], fj = F.imu_idx()[2 * n + 1];
            imu_factor_raw(fr + fi * kFrameStride, fr + fj * kFrameStride, rec, wc, a.alias_bias, r, J);
            for (int k = 0; k < 15; ++k) {
                double s = 0.0;
                for (int c = 0; c < 15; ++c) s += J[k * 30 + c] * v[fi * 15 + c] + J[k * 30 + 15 + c] * v[fj * 15 + c];
                u[k] = s;
            }
            atomicAdd(&acc, imu_whitened_norm2(rec, u));
        }
        if (F.n_prior() > 0) {
            const int n = F.n_prior(), d = 15 * n;
            if (tid < n) {
                double r15[15], Ji[9];
                prior_frame_raw(fr + F.prior_frames()[tid] * kFrameStride, F.prior_x0() + tid * kFrameStride, r15, Ji);
                const double *vf = v + F.prior_frames()[tid] * 15;
                for (int k = 0; k < 3; ++k) ev[15 * tid + k] = Ji[3 * k] * vf[0] + Ji[3 * k + 1] * vf[1] + Ji[3 * k + 2] * vf[2];
                for (int k = 3; k < 15; ++k) ev[15 * tid + k] = vf[k];
            }
            __syncthreads();
            double c2 = 0.0;
            for (int i = tid; i < d; i += nt) {
                double s = 0.0;
                for (int k = 0; k < d; ++k) s += F.prior_S()[(size_t)i * d + k] * ev[k];
                c2 += s * s;
            }
            atomicAdd(&acc, c2);
        }
    }
    if (F.n_ptracks() > 0) {
        const double cb = F.cb();
        for (int t = tid; t < F.n_ptracks(); t += nt) {
            const int b0 = F.pt_begin()[t], K = F.pt_begin()[t + 1] - b0;
            double r, J[6 * kMaxFrames];
            plane_factor(K, F.pt_frame() + b0, F.pt_z() + 2 * b0, fr, wc, F.plane() + 4 * F.pt_plane()[t], wc.plane_sic, &r, J);
            const double sc2 = 1.0 / (1.0 + r * r / cb);             // rho'
            double s = 0.0;
            for (int i = 0; i < 6 * K; ++i) s += J[i] * v[F.pt_frame()[b0 + i / 6] * 15 + (i % 6)];
            atomicAdd(&acc, sc2 * s * s);
        }
    }
    __syncthreads();
    if (tid == 0) {
        double *av = a.acc + (size_t)w * kAcc;
        if (acc != 0.0) av[10] += acc;           // one CTA per window owns slot 10
        if (a.loop) { WinCtrl c = ctrl; tr_after_jv(c, av); ctrl = c; }
    }
}

}  // namespace pvio
