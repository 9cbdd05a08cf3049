// Covariance of resident windows (pvio_b200_batch_window_covariance): the inverse of J^T J of every residual block the
// solve adds, at the window's state, in the solve's local coordinates and without the trust-region regulariser -- what
// ceres::Covariance returns for the problem bundle_adjustor.cpp:63-249 builds (GetCovarianceBlockInTangentSpace).
//
//   cov_kernel     one CTA per record: the reduced system as solve_kernel assembles it (assemble_system, ba_solve.cuh)
//                  from the mu = 0 sweeps, Jacobi scaling, constant rows pinned to the identity, Cholesky (ba_chol.cuh),
//                  then L^-1 in place of the factor and Sigma = S L^-T L^-1 S.  The landmarks are eliminated exactly, so
//                  Sigma is the true marginal of the frame coordinates.  Out: the named frames' joint block, and every
//                  frame pair's pose block in xi coordinates, Sigma_xi = T_f Sigma_delta T_g^T, for the landmark kernel.
//   cov_lm_kernel  one warp per named track: Var(rho_l) = 1 / H_ll + h_l^T Sigma_xi h_l / H_ll^2 from the landmark's
//                  pivot and its Schur records h_l (the same elimination the update sweep back-substitutes).
#pragma once
#include <math_constants.h>
#include "ba_solve.cuh"

namespace pvio {

struct CovArgs : SolveArgs {
    const CovRec *recs;      // [n]
    const int32_t *frames;   // the named frames of every record (CovRec::frames_off)
    const CovLm *lms;        // [n_lm] the named tracks of every record, in record order
    int n_lm;
    double *cov;             // out: the records' frame blocks (CovRec::cov_off)
    double *var;             // out: [n_lm]
    int32_t *status;         // out: [n]
    double *sig;             // scratch: Sigma_delta of each record, [D][D] at CovRec::sig_off (D = stride * N)
    double *sig_xi;          // scratch: [n][Ncap][Ncap][36] Sigma_xi of every frame pair
};

// cov_kernel: solve_kernel's assembly (solve_body), then this
struct CovBody {
    static __device__ __forceinline__ int window(const SolveArgs &a) { return static_cast<const CovArgs &>(a).recs[blockIdx.x].slot; }
    static __device__ __forceinline__ void finish(const SolveArgs &sa, int w, int N, int stride, int D, int nb, double *A,
                                                  const double *hcorr, double *sc, double *xs, const double *Tm, double *scr, int *flag_sm);
};

static __global__ void __launch_bounds__(256) cov_kernel(CovArgs a) { solve_body<true, CovBody>(a); }

__device__ __forceinline__ void CovBody::finish(const SolveArgs &sa, int w, int N, int stride, int D, int nb, double *A,
                                                const double *hcorr, double *sc, double *xs, const double *Tm, double *scr, int *flag_sm) {
    const CovArgs &a = static_cast<const CovArgs &>(sa);
    const CovRec R = a.recs[blockIdx.x];
    const WinHdr &H = a.hdr[w];
    const int tid = threadIdx.x, nt = blockDim.x, Dp = nb * 4;
    // Jacobi scaling by the unreduced diagonal, as the solve takes it; the pose rows of constant frames and the padding
    // rows are pinned to the identity (scale 0: their rows and columns of Sigma are 0)
    const unsigned fixed = (unsigned)H.fixed_mask & ((1u << N) - 1u);
    auto pinned = [&](int i) { const int f = i / stride; return i >= D || (((fixed >> f) & 1u) && i - f * stride < 6); };
    for (int i = tid; i < Dp; i += nt) {
        sc[i] = pinned(i) ? 0.0 : 1.0 / (1.0 + sqrt(fmax(A[tri(i, i)] + hcorr[i], 0.0)));
        xs[i] = 0.0;
    }
    __syncthreads();
    for (int e = tid; e < Dp * (Dp + 1) / 2; e += nt) {
        int i, j;
        tri_unrank(e, i, j);
        double *p = A + tri(i, j);
        *p = (pinned(i) || pinned(j)) ? (i == j ? 1.0 : 0.0) : *p * sc[i] * sc[j];
    }
    __syncthreads();
    const bool ok = chol_solve_tiled<true>(A, xs, nb, flag_sm);   // (the register-resident form spills here)

    const int K15 = 15 * R.n_frames;
    const int32_t *fr = a.frames + R.frames_off;
    double *co = a.cov + R.cov_off;
    double *X = a.sig_xi + (size_t)blockIdx.x * a.Ncap * a.Ncap * 36;
    if (!ok) {
        for (int e = tid; e < K15 * K15; e += nt) co[e] = CUDART_NAN;
        for (int e = tid; e < N * N * 36; e += nt) X[e] = CUDART_NAN;
        if (tid == 0) a.status[blockIdx.x] = PVIO_B200_ENUMERIC;
        return;
    }
    // L^-1 in place, block column by block column from the last: X_IJ = -(sum_{J<K<=I} X_IK L_KJ) L_JJ^-1.  The diagonal
    // tiles already hold L_JJ^-1; column J is built in scratch and stored once no thread reads its L_KJ any more.
    double *colJ = scr;                                   // [nb - 1][16]
    for (int J = nb - 2; J >= 0; --J) {
        const int rows = (nb - 1 - J) * 4;
        for (int e = tid; e < rows; e += nt) {
            const int I = J + 1 + (e >> 2), r = e & 3;
            double t[4] = {0.0, 0.0, 0.0, 0.0};
            for (int K = J + 1; K <= I; ++K) {
                const double *Xr = A + tile_off(I, K) + r * 4, *L = A + tile_off(K, J);
#pragma unroll
                for (int m = 0; m < 4; ++m)
#pragma unroll
                    for (int c = 0; c < 4; ++c) t[c] += Xr[m] * L[m * 4 + c];
            }
            const double *Li = A + tile_off(J, J);
            double *o = colJ + (I - J - 1) * 16 + r * 4;
#pragma unroll
            for (int c = 0; c < 4; ++c) o[c] = -(t[0] * Li[c] + t[1] * Li[4 + c] + t[2] * Li[8 + c] + t[3] * Li[12 + c]);
        }
        __syncthreads();
        for (int e = tid; e < rows * 4; e += nt) A[tile_off(J + 1 + (e >> 4), J) + (e & 15)] = colJ[e];
        __syncthreads();
    }
    // Sigma_delta = S X^T X S over the system's D coordinates (rows of X at and past the padding are 0 below the diagonal)
    double *S = a.sig + R.sig_off;
    for (int e = tid; e < D * (D + 1) / 2; e += nt) {
        int i, j;
        tri_unrank(e, i, j);
        double s = 0.0;
        for (int k = i; k < D; ++k) s += A[tri(k, i)] * A[tri(k, j)];
        s *= sc[i] * sc[j];
        S[(size_t)i * D + j] = s;
        S[(size_t)j * D + i] = s;
    }
    __syncthreads();
    // the named frames' joint block, 15 coordinates per frame (0 where the window has no such coordinate)
    for (int e = tid; e < K15 * K15; e += nt) {
        const int r = e / K15, c = e - r * K15;
        const int p = r / 15, q = c / 15, cr = r - 15 * p, cq = c - 15 * q;
        co[e] = (cr < stride && cq < stride) ? S[(size_t)(fr[p] * stride + cr) * D + fr[q] * stride + cq] : 0.0;
    }
    // Sigma_xi[f, g] = T_f Sigma_delta[f, g] T_g^T over the pose coordinates
    for (int e = tid; e < N * N * 36; e += nt) {
        const int fg = e / 36, ij = e - fg * 36, f = fg / N, g = fg - f * N, i = ij / 6, j = ij - i * 6;
        const double *Tf = Tm + f * 36 + i * 6, *Tg = Tm + g * 36 + j * 6;
        const double *Sfg = S + (size_t)f * stride * D + g * stride;
        double s = 0.0;
        for (int aa = 0; aa < 6; ++aa) {
            double t = 0.0;
#pragma unroll
            for (int bb = 0; bb < 6; ++bb) t += Sfg[(size_t)aa * D + bb] * Tg[bb];
            s += Tf[aa] * t;
        }
        X[e] = s;
    }
    if (tid == 0) a.status[blockIdx.x] = PVIO_B200_OK;
}

constexpr int kCovLmWarps = 4;

// One warp per named track.  bw_landmark_cov_kernel (bw_query.cu) forms the same Var(rho) through ba_cov_lm.cuh,
// which restates this body operation for operation so that both calls give the same bits: a change to the arithmetic
// here must be made there too (tests/test_gpu_batch_window_landmarks.py checks the two for bit equality).
// h_l over the free frames: the landmark's Schur records (the anchor's materialised when the anchor is free, zero
// blocks for the free frames that do not see it); constant frames take no part (Sigma_xi is 0 there).
template <typename real>
static __global__ void __launch_bounds__(32 * kCovLmWarps) cov_lm_kernel(CovArgs a) {
    __shared__ double u_sm[kCovLmWarps][6 * kMaxFrames];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int t = blockIdx.x * kCovLmWarps + wv;
    if (t >= a.n_lm) return;
    const CovLm L = a.lms[t];
    if (L.lm < 0) {                                         // a plane track or a track with one observation
        if (lane == 0) a.var[t] = CUDART_NAN;
        return;
    }
    const int w = L.slot, N = a.hdr[w].N;
    const unsigned fixed = (unsigned)a.hdr[w].fixed_mask & ((1u << N) - 1u);
    const real *hs = reinterpret_cast<const real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    double *u = u_sm[wv];
    for (int i = lane; i < 6 * N; i += 32) {
        const int f = i / 6;
        u[i] = ((fixed >> f) & 1u) ? 0.0 : (double)hs[((size_t)f * a.Mcap + L.lm) * 6 + (i - 6 * f)];
    }
    __syncwarp();
    const double *X = a.sig_xi + (size_t)L.rec * a.Ncap * a.Ncap * 36;
    double q = 0.0;
    for (int i = lane; i < 6 * N; i += 32) {
        const int f = i / 6, ii = i - 6 * f;
        const double *Xf = X + (size_t)f * N * 36 + ii * 6;
        double s = 0.0;
        for (int g = 0; g < N; ++g)
#pragma unroll
            for (int jj = 0; jj < 6; ++jj) s += Xf[g * 36 + jj] * u[6 * g + jj];
        q += u[i] * s;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
    if (lane == 0) {
        const double hll = a.lm_aux[(size_t)w * a.Mcap + L.lm].hll;
        a.var[t] = 1.0 / hll + q / (hll * hll);
    }
}

}  // namespace pvio
