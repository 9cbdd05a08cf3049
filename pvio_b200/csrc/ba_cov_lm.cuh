// The per-landmark arithmetic of cov_lm_kernel (ba_cov.cuh), one warp per landmark: h_l in xi coordinates from the
// Schur records, and h_l^T Sigma_xi h_l.  bw_landmark_cov_kernel (bw_query.cu: the world points' covariance of
// pvio_b200_batch_window_landmarks) forms Var(rho) with it, so that both calls give the same bits: the floating-point
// operations here are cov_lm_kernel's, in the same order.  cov_lm_kernel keeps its own copy of them: through these
// helpers nvcc lays out its address arithmetic differently, and its SASS is held to what it was.
#pragma once
#include <cuda_runtime.h>
#include "ba_types.h"

namespace pvio {

// u[6 N] (the warp's shared row) = h_l over the window's frames: landmark lm's Schur records hs (the anchor's
// materialised when the anchor is free, zero blocks for the free frames that do not see it), 0 on the constant frames
template <typename real>
__device__ __forceinline__ void cov_lm_h(const real *hs, int Mcap, int lm, int N, unsigned fixed, int lane, double *u) {
    for (int i = lane; i < 6 * N; i += 32) {
        const int f = i / 6;
        u[i] = ((fixed >> f) & 1u) ? 0.0 : (double)hs[((size_t)f * Mcap + lm) * 6 + (i - 6 * f)];
    }
}

// q = u^T Sigma_xi u on every lane of the warp, X the record's Sigma_xi [N][N][36].  kRow: also (Sigma_xi u) over the
// six rows of frame an, which the lanes (6 an + i) & 31 (i < 6) hold in `row` -- products the sum is made of anyway.
template <bool kRow>
__device__ __forceinline__ double cov_lm_quad(const double *u, const double *X, int N, int lane, int an, double &row) {
    double q = 0.0;
    for (int i = lane; i < 6 * N; i += 32) {
        const int f = i / 6, ii = i - 6 * f;
        const double *Xf = X + (size_t)f * N * 36 + ii * 6;
        double s = 0.0;
        for (int g = 0; g < N; ++g)
#pragma unroll
            for (int jj = 0; jj < 6; ++jj) s += Xf[g * 36 + jj] * u[6 * g + jj];
        if constexpr (kRow) {
            if (f == an) row = s;
        }
        q += u[i] * s;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
    return q;
}

// Var(rho) from the pivot and the quadratic form (1 / H_ll + h^T Sigma_xi h / H_ll^2)
__device__ __forceinline__ double cov_lm_var(double hll, double q) { return 1.0 / hll + q / (hll * hll); }

}  // namespace pvio
