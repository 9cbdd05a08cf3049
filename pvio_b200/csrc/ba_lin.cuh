// Reprojection factor in xi coordinates: shared definitions of the linearise / Schur / update sweeps
// (ba_linearize.cuh, ba_schur.cuh, ba_update.cuh), which together replace, per Gauss-Newton iteration, what
// ceres::Solve (bundle_adjustor.cpp:249) does with ReprojectionErrorCost::Evaluate
// (estimation/ceres/reprojection_error_cost.h:40-120) over every residual block, the CauchyLoss(1.0) corrector
// (bundle_adjustor.cpp:58) and the SPARSE_SCHUR elimination of the inverse-depth blocks (solver_options.h:27).
//
// Formulation (DESIGN.md "xi coordinates").  For target frame t, anchor a, landmark l:
//     x_l  = R_wc(a) [z_ref;1]/rho + c_a                 world point (fp64)
//     y    = R_wc(t)^T (x_l - c_t)                        point in the target camera (fp64)
//     r    = W (y.xy/y.z - z_tgt)                         residual; numerator in fp64
//     G    = W dpi(y) R_wc(t)^T                           d r / d x_world  (2x3, fp32)
//     dr   = G X_l (xi_t - xi_a) + G c_l d rho,   X_l = [[x_l]x, I],  c_l = -(x_l - c_a)/rho
// where xi_f = T_f [dtheta_f; dp_f],  T_f = [[R_f, 0], [-[p_f]x R_f, -I]] is a per-frame
// change of variables applied once per iteration in the solve kernel.  This reproduces the
// reference Jacobians :94-113 exactly (J_delta = J_xi T) while making the target and
// anchor blocks of a residual +-the same 2x6 matrix Y = G X_l, so that every direct
// J^T J contribution is one symmetric 6x6 product per observation.
//
#pragma once
#include "ba_math.cuh"
#include "ba_types.h"

namespace pvio {

constexpr int kGroup = 16;                  // lanes per landmark group of the post-pass (>= frames)
constexpr int kLinThreads = 256;
constexpr int kChunk = 32;                  // landmarks per chunk (<= 32 consecutive landmarks with a common anchor)

struct FrameSm {
    double Rwc[9];       // body->world times cam->body: camera-to-world rotation
    double c[3];         // camera centre, window-origin relative
    float R32[9];
    float pad[3];
};

// Build the per-frame camera pose from the fp64 frame state.
__device__ __forceinline__ void make_frame(const double *fs, const WinConst &wc, FrameSm &o) {
    double R[9], Rcs[9];
    quat_to_mat(fs, R);
    quat_to_mat(wc.cam_q, Rcs);
    mat3_mul(R, Rcs, o.Rwc);
    double t[3];
    mat3_vec(R, wc.cam_p, t);
#pragma unroll
    for (int i = 0; i < 3; ++i) o.c[i] = fs[4 + i] - wc.origin[i] + t[i];
#pragma unroll
    for (int i = 0; i < 9; ++i) o.R32[i] = (float)o.Rwc[i];
}

// symmetric 6x6 index (i<=j) -> 0..20
__host__ __device__ constexpr int sym6(int i, int j) { return i * 6 - i * (i - 1) / 2 + (j - i); }

// pair index of block (f, g) with g <= f in the block-lower-triangular storage
__host__ __device__ __forceinline__ int pair_idx(int f, int g) { return f * (f + 1) / 2 + g; }

struct ObsLin {            // linearisation of one observation in xi coordinates (loss-corrected)
    float Y0[6], Y1[6];    // rows of Y = sqrt(rho') G X_l
    float r0, r1;          // sqrt(rho') r
    float j0, j1;          // sqrt(rho') G c_l   (d r / d rho)
    float cost;            // rho(s) / 2
};

// bt = Rwc_t^T (c_a - c_t): the anchor camera's centre in the target camera's axes (fp64, rounded once)
__device__ __forceinline__ void baseline_in(const FrameSm &Ft, const FrameSm &Fa, float bt[3]) {
    const double d0 = Fa.c[0] - Ft.c[0], d1 = Fa.c[1] - Ft.c[1], d2 = Fa.c[2] - Ft.c[2];
#pragma unroll
    for (int j = 0; j < 3; ++j) bt[j] = (float)(Ft.Rwc[j] * d0 + Ft.Rwc[3 + j] * d1 + Ft.Rwc[6 + j] * d2);
}

// Evaluate one observation.  x: world point (fp64), xf: (float)x, ir = 1 / rho, bt = Rwc^T (c_anchor - c_target)
// (the baseline in the target camera): d r / d rho = ir W dpi bt (see linearize_blk in ba_linearize.cuh).
template <bool kLoss>
__device__ __forceinline__ void linearize_obs(const FrameSm &F, const double x[3], const float xf[3],
                                              float ir, const float bt[3], float zx, float zy,
                                              const float W[4], float cauchy_b, ObsLin &o) {
    const double d0 = x[0] - F.c[0], d1 = x[1] - F.c[1], d2 = x[2] - F.c[2];
    const double y0 = F.Rwc[0] * d0 + F.Rwc[3] * d1 + F.Rwc[6] * d2;
    const double y1 = F.Rwc[1] * d0 + F.Rwc[4] * d1 + F.Rwc[7] * d2;
    const double y2 = F.Rwc[2] * d0 + F.Rwc[5] * d1 + F.Rwc[8] * d2;
    const double nx = y0 - (double)zx * y2;          // fp64: the cancellation happens here
    const double ny = y1 - (double)zy * y2;
    const float iz = 1.0f / (float)y2;
    const float u0 = (float)nx * iz, u1 = (float)ny * iz;
    float r0 = W[0] * u0 + W[1] * u1;
    float r1 = W[2] * u0 + W[3] * u1;
    const float yx = (float)y0 * iz, yy = (float)y1 * iz;
    // A = W * dpi, dpi = [[iz, 0, -yx iz], [0, iz, -yy iz]]
    const float A00 = W[0] * iz, A01 = W[1] * iz, A02 = -(W[0] * yx + W[1] * yy) * iz;
    const float A10 = W[2] * iz, A11 = W[3] * iz, A12 = -(W[2] * yx + W[3] * yy) * iz;
    // G = A * Rwc^T  ->  G[i][k] = sum_m A[i][m] Rwc[k][m]
    float G0[3], G1[3];
    const float m0 = iz * ir * (bt[0] - yx * bt[2]), m1 = iz * ir * (bt[1] - yy * bt[2]);     // ir dpi bt
    float j0 = W[0] * m0 + W[1] * m1, j1 = W[2] * m0 + W[3] * m1;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        G0[k] = A00 * F.R32[3 * k] + A01 * F.R32[3 * k + 1] + A02 * F.R32[3 * k + 2];
        G1[k] = A10 * F.R32[3 * k] + A11 * F.R32[3 * k + 1] + A12 * F.R32[3 * k + 2];
    }
    float cost;
    if (kLoss) {
        // ceres::CauchyLoss(a), b = a^2: rho = b log(1 + s/b), rho' = 1/(1 + s/b); rho'' < 0 so the
        // Corrector scales r and J by sqrt(rho') (corrector.cc)
        const float s = r0 * r0 + r1 * r1;
        const float t = 1.0f + s / cauchy_b;
        const float sc = rsqrtf(t);
        cost = 0.5f * cauchy_b * logf(t);
        r0 *= sc; r1 *= sc; j0 *= sc; j1 *= sc;
#pragma unroll
        for (int k = 0; k < 3; ++k) { G0[k] *= sc; G1[k] *= sc; }
    } else {
        cost = 0.5f * (r0 * r0 + r1 * r1);
    }
    // Y rows: [g x x_l, g]
    o.Y0[0] = G0[1] * xf[2] - G0[2] * xf[1];
    o.Y0[1] = G0[2] * xf[0] - G0[0] * xf[2];
    o.Y0[2] = G0[0] * xf[1] - G0[1] * xf[0];
    o.Y1[0] = G1[1] * xf[2] - G1[2] * xf[1];
    o.Y1[1] = G1[2] * xf[0] - G1[0] * xf[2];
    o.Y1[2] = G1[0] * xf[1] - G1[1] * xf[0];
#pragma unroll
    for (int k = 0; k < 3; ++k) { o.Y0[3 + k] = G0[k]; o.Y1[3 + k] = G1[k]; }
    o.j0 = j0; o.j1 = j1;
    o.r0 = r0; o.r1 = r1; o.cost = cost;
}

__device__ __forceinline__ void world_point(const FrameSm &Fa, float zrx, float zry, double rho,
                                            double x[3], float xf[3], float cl[3]) {
    const double ir = 1.0 / rho;
    const double zx = (double)zrx, zy = (double)zry;
    const double v0 = (Fa.Rwc[0] * zx + Fa.Rwc[1] * zy + Fa.Rwc[2]) * ir;
    const double v1 = (Fa.Rwc[3] * zx + Fa.Rwc[4] * zy + Fa.Rwc[5]) * ir;
    const double v2 = (Fa.Rwc[6] * zx + Fa.Rwc[7] * zy + Fa.Rwc[8]) * ir;
    x[0] = v0 + Fa.c[0]; x[1] = v1 + Fa.c[1]; x[2] = v2 + Fa.c[2];
    xf[0] = (float)x[0]; xf[1] = (float)x[1]; xf[2] = (float)x[2];
    cl[0] = (float)(-v0 * ir); cl[1] = (float)(-v1 * ir); cl[2] = (float)(-v2 * ir);
}

// Jacobi scaling / LM regularisation of a diagonal entry, as ceres' dogleg strategy applies
// it (dogleg_strategy.cc): reg = mu * clamp(scale^2 H_ii, 1e-6, 1e32) / scale^2.
__device__ __forceinline__ double lm_reg(double hii, double scale, double mu) {
    const double s2 = scale * scale;
    double d2 = s2 * hii;
    d2 = fmin(fmax(d2, 1.0e-6), 1.0e32);
    return mu * d2 / s2;
}

}  // namespace pvio
