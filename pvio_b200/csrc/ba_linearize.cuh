// Linearise sweep of the reprojection blocks: residuals, Jacobians, Cauchy weights, the DIRECT part of the
// reduced pose system and the per-landmark records the Schur kernel (ba_schur.cuh) and the update sweep
// (ba_update.cuh) consume.
//
// Replaces, per Gauss-Newton iteration, what ceres::Solve (bundle_adjustor.cpp:249) does with
// ReprojectionErrorCost::Evaluate (estimation/ceres/reprojection_error_cost.h:40-120) over every residual block
// and the CauchyLoss(1.0) corrector (bundle_adjustor.cpp:58); with kLoss = false / victim_only = 1 it is the
// reprojection part of BundleAdjustor::marginalize_frame (bundle_adjustor.cpp:453-533).
// Formulation: the xi coordinates of ba_lin.cuh (target and anchor blocks of a residual are +-Y).
//
// Work decomposition (third generation; the first two walked the table by landmark and paid a 31-shuffle
// transpose-reduction per observation step):
//   phase 0   thread per landmark: world point x_l (fp64) and 1 / rho into shared memory.
//   phase 1   the frame-major table (ba_fobs.cuh) is cut into rows of 32 entries of ONE (target, anchor)
//             segment; a warp owns a contiguous range of rows.  Thread = residual block.  The target pose sits
//             in registers for the whole segment; Y^T Y, Y^T r of the segment are REGISTER sums (float2
//             pairs of fma.rn.f32), reduced across the warp once per segment; h_t = Y^T j leaves as one coalesced
//             24-byte store per lane into the frame-major record array hs[t][l][6].  (j.j, j.r): when one CTA
//             owns the window (and the shared layout fits, PipeArgs::lm_part), added into the warp's own
//             per-landmark partial in shared memory; otherwise one 8-byte store into jr[t][l][2].  lm_finish
//             sums either per landmark, in frame order.
//   epilogue  direct blocks -> Hred / gred (the Schur kernel subtracts its sum).
// real = float: fp32 Jacobians, fp64 residual numerators (the visual-only throughput path);
// real = double: everything fp64 (inertial windows, whose reduced system is too ill-conditioned for fp32
// Jacobians at the 1e-5 tolerance, and the marginaliser).
#pragma once
#include <cuda_runtime.h>
#include "ba_fobs.cuh"
#include "ba_lin.cuh"

namespace pvio {

constexpr int kDta = 28;                        // doubles per (target, anchor) block: 21 sym + 6 grad + 1 pad

struct PipeArgs : BatchArrays {
    int compute_scale;           // 1: iteration 0, (re)compute lm_scale
    int victim_only;             // marginaliser: only landmarks flagged in_victim
    double mu_override;          // >= 0: use this mu instead of ctrl->mu
    int w0;                      // first window of this launch
    int loop;                    // 1: iteration of the device-side trust-region loop (ba_tr.cuh): obey the window's flags
    int spec;                    // loop only. 1: linearise the CANDIDATE (frames_cand, rho_cand) into the window's other buffer set
    int lm_part;                 // 1 (one CTA per window only): the (j.j, j.r) sums stay in shared memory, jr is not touched
    const int32_t *slots;        // may be NULL: CTA row b works on window slots[b] instead of w0 + b (a named-slot list)
};

__device__ __forceinline__ void pipe_select(PipeArgs &a, int b) {
    if (!b) return;
    a.hs = reinterpret_cast<char *>(a.hs) + a.bufs.hs; a.jr = reinterpret_cast<char *>(a.jr) + a.bufs.jr;
    a.lm_w = reinterpret_cast<char *>(a.lm_w) + a.bufs.lm_w; a.lm_msk += a.bufs.lm_msk; a.lm_aux += a.bufs.lm_aux;
    a.Hred += a.bufs.Hred; a.Hdd += a.bufs.Hdd; a.gdir += a.bufs.g; a.gred += a.bufs.g; a.cost_vis += a.bufs.cost;
}
// which buffer set a sweep of window w works on, or -1: nothing to do for this window
__device__ __forceinline__ int pipe_buffer(const PipeArgs &a, int w) {
    if (!a.loop) return 0;
    const WinCtrl &c = a.ctrl[w];
    if (a.spec) {
        if (c.done) return -1;
        // a skipped iteration whose linearisation was invalidated (failed linear solve, mu * 10: ba_tr.cuh): this sweep
        // linearises the STATE again, with the new mu, into the state's own buffer set -- the next body starts from it
        if (c.skip) return c.have_lin ? -1 : c.buf;
        return 1 - c.buf;
    }
    return (c.done || c.have_lin) ? -1 : c.buf;
}
// the speculative sweep of a body looks at the CANDIDATE; its retry form (above) at the state
__device__ __forceinline__ bool pipe_at_candidate(const PipeArgs &a, int w) { return a.spec && !(a.loop && a.ctrl[w].skip); }
// the pivots of a speculative sweep use the mu the next iteration will have IF its step is accepted (tr_decide)
__device__ __forceinline__ double pipe_mu(const PipeArgs &a, int w) {
    if (a.mu_override >= 0.0) return a.mu_override;
    const double mu = a.ctrl[w].mu;
    return pipe_at_candidate(a, w) ? fmax(1e-8, 2.0 * mu / 10.0) : mu;
}

// ---- pairs with a scalar-broadcast operand: two FFMA (Hopper has no packed fp32 FMA) for float, two DFMA for double.
// The _rn intrinsics keep the rounding of every product and sum fixed (no contraction of bmul into a later add).
template <typename real> struct Vec2;
template <> struct Vec2<float> { typedef float2 type; };
template <> struct Vec2<double> { typedef double2 type; };
__device__ __forceinline__ float2 mk2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ double2 mk2(double a, double b) { return make_double2(a, b); }
__device__ __forceinline__ float2 bfma(float a, float2 b, float2 c) { return make_float2(__fmaf_rn(a, b.x, c.x), __fmaf_rn(a, b.y, c.y)); }
__device__ __forceinline__ double2 bfma(double a, double2 b, double2 c) { return make_double2(fma(a, b.x, c.x), fma(a, b.y, c.y)); }
__device__ __forceinline__ float2 bmul(float a, float2 b) { return make_float2(__fmul_rn(a, b.x), __fmul_rn(a, b.y)); }
__device__ __forceinline__ double2 bmul(double a, double2 b) { return make_double2(a * b.x, a * b.y); }
__device__ __forceinline__ float rsqrt_r(float x) {        // rsqrt.approx: 1 ulp; the argument is 1 + s/b >= 1 (no denormal path)
    float y;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ double rsqrt_r(double x) { return 1.0 / sqrt(x); }
__device__ __forceinline__ float log_r(float x) { return logf(x); }
__device__ __forceinline__ double log_r(double x) { return log(x); }
__device__ __forceinline__ float rcp_r(float x) {          // rcp.approx: 1 ulp, no slow path (depths are far from the fp32 range limits)
    float y;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
    return y;
}
__device__ __forceinline__ double rcp_r(double x) { return 1.0 / x; }

template <typename real>
struct FrameR {              // target pose of a segment, register resident
    double Rwc[9], c[3];
    real R[9];
};

template <typename real>
struct ObsL {                // linearisation of one residual block in xi coordinates (loss-corrected)
    typename Vec2<real>::type Y0[3], Y1[3];   // rows of Y = sqrt(rho') G X_l as pairs (0,1) (2,3) (4,5)
    real r0, r1;             // sqrt(rho') r
    real j0, j1;             // sqrt(rho') d r / d rho
    real cost;               // with the loss: t = 1 + s / b (the caller accumulates b/2 log t); without: s / 2
};

// reprojection_error_cost.h:58-117 in xi coordinates (see ba_lin.cuh).  x: world point (fp64), xf = (real)x,
// ir = 1 / rho, bt = Rwc^T (c_anchor - c_target) (the baseline in the target camera, fp64 rounded once).
// d r / d rho = G d x / d rho = -ir W dpi Rwc^T (x - c_anchor) = ir W dpi bt, because dpi y = 0: the form
// G . (d x / d rho) cancels to |bt| / depth of its terms and loses eps * depth / baseline in `real` (1e-4 of the
// inverse-depth Jacobian at a 1/1000 baseline in fp32); dpi bt has no such cancellation.
template <bool kLoss, typename real>
__device__ __forceinline__ void linearize_blk(const FrameR<real> &F, double x0, double x1, double x2, real xf0, real xf1,
                                              real xf2, real ir, const real (&bt)[3], float zx, float zy, const real (&W)[4],
                                              bool diag_w, real inv_cauchy_b, ObsL<real> &o) {
    const double d0 = x0 - F.c[0], d1 = x1 - F.c[1], d2 = x2 - F.c[2];
    const double y0 = F.Rwc[0] * d0 + F.Rwc[3] * d1 + F.Rwc[6] * d2;
    const double y1 = F.Rwc[1] * d0 + F.Rwc[4] * d1 + F.Rwc[7] * d2;
    const double y2 = F.Rwc[2] * d0 + F.Rwc[5] * d1 + F.Rwc[8] * d2;
    const double nx = y0 - (double)zx * y2;          // fp64: the cancellation happens here
    const double ny = y1 - (double)zy * y2;
    const real iz = rcp_r((real)y2);
    const real u0 = (real)nx * iz, u1 = (real)ny * iz;
    const real yx = (real)y0 * iz, yy = (real)y1 * iz;
    // A = W dpi, dpi = [[iz, 0, -yx iz], [0, iz, -yy iz]];  G = A Rwc^T.  W = sqrt_inv_cov is diag(fx, fy) / sigma in the
    // reference (core/core.cpp:114-116): the diagonal case (uniform per window) skips the zero products
    real r0, r1, G0[3], G1[3], j0, j1;
    const real m0 = iz * ir * (bt[0] - yx * bt[2]), m1 = iz * ir * (bt[1] - yy * bt[2]);     // ir dpi bt
    if (diag_w) {
        r0 = W[0] * u0; r1 = W[3] * u1;
        j0 = W[0] * m0; j1 = W[3] * m1;
        const real A00 = W[0] * iz, A02 = -A00 * yx, A11 = W[3] * iz, A12 = -A11 * yy;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            G0[k] = A00 * F.R[3 * k] + A02 * F.R[3 * k + 2];
            G1[k] = A11 * F.R[3 * k + 1] + A12 * F.R[3 * k + 2];
        }
    } else {
        r0 = W[0] * u0 + W[1] * u1;
        r1 = W[2] * u0 + W[3] * u1;
        j0 = W[0] * m0 + W[1] * m1;
        j1 = W[2] * m0 + W[3] * m1;
        const real A00 = W[0] * iz, A01 = W[1] * iz, A02 = -(W[0] * yx + W[1] * yy) * iz;
        const real A10 = W[2] * iz, A11 = W[3] * iz, A12 = -(W[2] * yx + W[3] * yy) * iz;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            G0[k] = A00 * F.R[3 * k] + A01 * F.R[3 * k + 1] + A02 * F.R[3 * k + 2];
            G1[k] = A10 * F.R[3 * k] + A11 * F.R[3 * k + 1] + A12 * F.R[3 * k + 2];
        }
    }
    if (kLoss) {
        // ceres::CauchyLoss(a), b = a^2: rho = b log(1 + s/b), rho' = 1/(1 + s/b); rho'' < 0 so the Corrector
        // scales r and J by sqrt(rho') (corrector.cc).  The caller turns t into the cost (b/2 log t).
        const real s = r0 * r0 + r1 * r1;
        const real t = (real)1 + s * inv_cauchy_b;
        const real sc = rsqrt_r(t);
        o.cost = t;
        r0 *= sc; r1 *= sc; j0 *= sc; j1 *= sc;
#pragma unroll
        for (int k = 0; k < 3; ++k) { G0[k] *= sc; G1[k] *= sc; }
    } else {
        o.cost = (real)0.5 * (r0 * r0 + r1 * r1);
    }
    // Y rows: [g x x_l, g]
    o.Y0[0] = mk2(G0[1] * xf2 - G0[2] * xf1, G0[2] * xf0 - G0[0] * xf2);
    o.Y0[1] = mk2(G0[0] * xf1 - G0[1] * xf0, G0[0]);
    o.Y0[2] = mk2(G0[1], G0[2]);
    o.Y1[0] = mk2(G1[1] * xf2 - G1[2] * xf1, G1[2] * xf0 - G1[0] * xf2);
    o.Y1[1] = mk2(G1[0] * xf1 - G1[1] * xf0, G1[0]);
    o.Y1[2] = mk2(G1[1], G1[2]);
    o.j0 = j0; o.j1 = j1;
    o.r0 = r0; o.r1 = r1;
}

// sum of log(t_i), t_i >= 1.  fp32: the logarithm of a running product, folded at least every 4 terms (t itself carries
// a rounding error of 6e-8, so log(t_1 t_2 t_3 t_4) loses nothing against four logf calls and costs a quarter of them);
// a term that could overflow the product (t > 1e9: a residual of > 3e4 sigma) takes its own logarithm.
template <typename real> struct LogAcc;
template <> struct LogAcc<float> {
    float prod = 1.f, sum = 0.f;
    __device__ __forceinline__ void add(float t) { if (t > 1e9f) sum += logf(t); else prod *= t; }
    __device__ __forceinline__ void fold() { sum += logf(prod); prod = 1.f; }
    __device__ __forceinline__ float total() { return sum + logf(prod); }
};
template <> struct LogAcc<double> {
    double sum = 0.0;
    __device__ __forceinline__ void add(double t) { sum += log(t); }
    __device__ __forceinline__ void fold() {}
    __device__ __forceinline__ double total() { return sum; }
};

// Per-landmark record of the linearise sweep in shared memory, 48 bytes = three 16-byte loads by the lane that owns an
// observation of the landmark: world point x (fp64), (real) x, c = (1 / rho, 0, 0).
constexpr int kLmSm = 48;
__device__ __forceinline__ void lm_sm_store(unsigned char *rec, double x0, double x1, double x2, float c0, float c1, float c2) {
    reinterpret_cast<double2 *>(rec)[0] = make_double2(x0, x1);
    reinterpret_cast<double *>(rec)[2] = x2;
    reinterpret_cast<float2 *>(rec)[3] = make_float2((float)x0, (float)x1);
    reinterpret_cast<float4 *>(rec)[2] = make_float4((float)x2, c0, c1, c2);
}
__device__ __forceinline__ void lm_sm_store(unsigned char *rec, double x0, double x1, double x2, double c0, double c1, double c2) {
    reinterpret_cast<double2 *>(rec)[0] = make_double2(x0, x1);
    reinterpret_cast<double2 *>(rec)[1] = make_double2(x2, c0);
    reinterpret_cast<double2 *>(rec)[2] = make_double2(c1, c2);
}
// rec: shared-space address of the record (three ld.shared.v*: the address is one multiply-add from an opaque base)
__device__ __forceinline__ void lm_sm_load(unsigned rec, double (&x)[3], float (&xf)[3], float (&c)[3]) {
    double bx, by;
    float d0, d1, d2, d3;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x[0]), "=d"(x[1]) : "r"(rec));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2+16];" : "=d"(bx), "=d"(by) : "r"(rec));
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4+32];" : "=f"(d0), "=f"(d1), "=f"(d2), "=f"(d3) : "r"(rec));
    x[2] = bx;
    xf[0] = __int_as_float(__double2loint(by)); xf[1] = __int_as_float(__double2hiint(by)); xf[2] = d0;
    c[0] = d1; c[1] = d2; c[2] = d3;
}
__device__ __forceinline__ void lm_sm_load(unsigned rec, double (&x)[3], double (&xf)[3], double (&c)[3]) {
    double bx, by, dx, dy;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x[0]), "=d"(x[1]) : "r"(rec));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2+16];" : "=d"(bx), "=d"(by) : "r"(rec));
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2+32];" : "=d"(dx), "=d"(dy) : "r"(rec));
    x[2] = bx; xf[0] = x[0]; xf[1] = x[1]; xf[2] = bx;
    c[0] = by; c[1] = dx; c[2] = dy;
}
// *addr += v for a (j.j, j.r) partial at a shared-space address (phase 1 of lin_obs_kernel with lm_part)
__device__ __forceinline__ void part_add(unsigned addr, double2 v) {
    double x, y;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(x), "=d"(y) : "r"(addr) : "memory");
    x = __dadd_rn(x, v.x); y = __dadd_rn(y, v.y);
    asm volatile("st.shared.v2.f64 [%0], {%1, %2};" :: "r"(addr), "d"(x), "d"(y) : "memory");
}
// read-ahead of [p, p + bytes) into L2 by the whole CTA (the sweeps are latency-bound: 16 warps per SM)
__device__ __forceinline__ void l2_prefetch(const void *p, size_t bytes, int tid, int nthreads) {
    const char *c = reinterpret_cast<const char *>(p);
    for (size_t off = (size_t)tid * 128; off < bytes; off += (size_t)nthreads * 128)
        asm volatile("prefetch.global.L2 [%0];" :: "l"(c + off));
}

// Sum over the 32 lanes of q[i] for i = 0..31; lane i returns the total of entry i.  Transpose-reduction:
// 16 + 8 + 4 + 2 + 1 = 31 shuffles instead of 32 x 5.
template <typename T>
__device__ __forceinline__ T transpose_reduce(const T (&q)[32], int lane) {
    T v[16];
    {
        const bool up = lane & 16;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const T send = up ? q[k] : q[k + 16], keep = up ? q[k + 16] : q[k];
            v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
        }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const bool up = lane & 8;
        const T send = up ? v[k] : v[k + 8], keep = up ? v[k + 8] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const bool up = lane & 4;
        const T send = up ? v[k] : v[k + 4], keep = up ? v[k + 4] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
#pragma unroll
    for (int k = 0; k < 2; ++k) {
        const bool up = lane & 2;
        const T send = up ? v[k] : v[k + 2], keep = up ? v[k + 2] : v[k];
        v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
    }
    {
        const bool up = lane & 1;
        const T send = up ? v[0] : v[1], keep = up ? v[1] : v[0];
        v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 1);
    }
    return v[0];
}

// The 15 pair accumulators of a segment: rows i = 0..5 of the upper triangle of Y^T Y as column pairs
// (0: (0,01) (0,23) (0,45) | 1: (1,01) (1,23) (1,45) | 2: (2,23) (2,45) | 3: (3,23) (3,45) | 4: (4,45) | 5: (5,45))
// then Y^T r as (01) (23) (45).  Entry e of the flattened 30 floats -> slot of the (target, anchor) block
// (sym6 index, 21 + i for the gradient), -1 for the three below-diagonal halves and the two padding lanes.
__device__ __constant__ signed char kQSlot[32] = {0, 1, 2, 3, 4, 5, -1, 6, 7, 8, 9, 10, 11, 12, 13, 14,
                                                  -1, 15, 16, 17, 18, 19, -1, 20, 21, 22, 23, 24, 25, 26, -1, -1};

// strictly-lower pair index (t > a)
__device__ __forceinline__ int spair(int t, int a) { return t * (t - 1) / 2 + a; }

constexpr int kRing = 4;                        // rows of the frame-major table in flight per warp (cp.async ring)
constexpr int kLmBatch = 4;                     // landmarks per thread whose records lin_obs_kernel loads together

// Walks the rows of a warp: row r lies in segment sp = (t, an), its first table entry is k0()
struct RowCursor {
    const int32_t *sbeg, *srow;
    int r, sp, t, an, rows;
    __device__ __forceinline__ RowCursor(const int32_t *sb, const int32_t *sr, int r0, int n_rows)
        : sbeg(sb), srow(sr), r(r0), sp(0), t(1), an(0), rows(n_rows) { seek(); }
    __device__ __forceinline__ void seek() { if (r < rows) while (srow[sp + 1] <= r) { ++sp; if (++an == t) { ++t; an = 0; } } }
    __device__ __forceinline__ void advance() { ++r; seek(); }
    __device__ __forceinline__ int k0() const { return sbeg[sp] + (r - srow[sp]) * 32; }
};

// One row of the frame-major table in shared memory: the 32 keypoints (lane i copies and reads entry i), then the five
// 16-byte granules of flm from the one that holds the row's first index (a row starts anywhere in a granule), copied
// by lanes 0-4 and read by every lane, so the consumer needs __syncwarp around them.
constexpr int kFlmPad = 40;                     // entries of flm allocated beyond the last table entry
struct RowSlot {
    float2 z[32];
    uint4 lm[5];
    int off;                                    // halfword of the row's first index in lm[0]
};
__device__ __forceinline__ int row_lm(const RowSlot &s, int lane) {
    return reinterpret_cast<const FLm *>(s.lm)[s.off + lane];
}

// request row pf.r (if the warp owns it) into `dst` and move the prefetch cursor on; one commit group per call, empty
// or not, so that the consumer's wait_group count stays uniform
__device__ __forceinline__ void row_prefetch(RowCursor &pf, int r_end, const float2 *fz, const FLm *flm, RowSlot *dst, int lane) {
    if (pf.r < r_end) {
        const int k0 = pf.k0();
        if (k0 + lane < pf.sbeg[pf.sp + 1])
            asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" :: "r"((uint32_t)__cvta_generic_to_shared(dst->z + lane)), "l"(fz + k0 + lane) : "memory");
        // always all five granules (flm is allocated kFlmPad entries beyond the table for this)
        const uintptr_t p = reinterpret_cast<uintptr_t>(flm + k0), g0 = p & ~(uintptr_t)15;
        if (lane < 5)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" :: "r"((uint32_t)__cvta_generic_to_shared(dst->lm + lane)), "l"(g0 + 16 * (uintptr_t)lane) : "memory");
        if (lane == 0) dst->off = (int)(p & 15) >> 1;
        pf.advance();
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
}

// Per-landmark completion of the linearise sweep (thread per landmark; in the epilogue of lin_obs_kernel when one
// CTA owns the window, as lm_finish_kernel otherwise): H_ll = sum j.j and g_l = sum j.r over the landmark's
// residual blocks in frame order (deterministic), Jacobi scale, w_l = 1 / (H_ll + mu clamp(.)) -- the pivot the
// Schur complement divides by (bundle_adjustor.cpp:537-538: skipped when not finite) --, the anchor block
// h_la = -sum_t h_lt when the anchor frame is free, zero blocks for the free frames that do not see the landmark
// (the Schur tiles then need no per-block predicate).
// part: the per-warp partial sums [nwarps][Mp] of the CTA's shared memory (lin_obs_kernel with lm_part), each a sum
// in frame order; summed here in warp order, which is again frame order.  nullptr: the per-block pairs in jr.
// lr_pre: the landmark's record, already loaded by the caller (nullptr: loaded here).
// the whole 32-byte record in two 16-byte stores (three 8-byte ones would touch each of its sectors three times)
__device__ __forceinline__ void lm_aux_store(LmAux *p, double hll_reg, double gl, double hll) {
    double2 *q = reinterpret_cast<double2 *>(p);
    q[0] = make_double2(hll_reg, gl);
    q[1] = make_double2(hll, 0.0);
}

template <typename real>
__device__ __forceinline__ void lm_finish(const PipeArgs &a, int w, int l, int N, int M, unsigned fixed, double mu, int compute_scale,
                                          const double2 *part = nullptr, int nwarps = 0, int Mp = 0, const LmRec *lr_pre = nullptr) {
    typedef typename Vec2<real>::type real2;
    const LmRec *lms = a.lms + (size_t)w * a.Mcap;
    real2 *wv = reinterpret_cast<real2 *>(a.lm_w) + (size_t)w * a.Mcap;
    int32_t *msk = a.lm_msk + (size_t)w * a.Mcap;
    if (l >= M) { wv[l] = mk2((real)0, (real)0); msk[l] = 0; return; }      // padding up to the copy granule of the Schur kernel
    const LmRec lr = lr_pre ? *lr_pre : lms[l];
    const int n_obs = lm_nobs(lr.meta), anchor = lm_anchor(lr.meta);
    const unsigned targets = lm_mask(lr.meta);
    const bool live = n_obs > 0 && !(a.victim_only && !lm_victim(lr.meta));
    LmAux *aux = a.lm_aux + (size_t)w * a.Mcap;
    if (!live) {
        wv[l] = mk2((real)0, (real)0); msk[l] = 0;
        if (!a.victim_only) lm_aux_store(aux + l, 1.0, 0.0, 0.0);
        return;
    }
    real *hs = reinterpret_cast<real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    double hll = 0.0, gl = 0.0;
    if (part) {
        for (int q = 0; q < nwarps; ++q) { const double2 v = part[q * Mp + l]; hll += v.x; gl += v.y; }
    } else {   // all loads first (independent, predicated), then the sums in frame order
        const real2 *jr = reinterpret_cast<const real2 *>(a.jr) + (size_t)w * a.Ncap * a.Mcap;
        real2 v[kMaxFrames];
#pragma unroll
        for (int f = 0; f < kMaxFrames; ++f) {
            v[f] = mk2((real)0, (real)0);
            if ((targets >> f) & 1u) v[f] = jr[(size_t)f * a.Mcap + l];
        }
#pragma unroll
        for (int f = 0; f < kMaxFrames; ++f) { hll += (double)v[f].x; gl += (double)v[f].y; }
    }
    double *lm_scale = a.lm_scale + (size_t)w * a.Mcap;
    double sc;
    if (compute_scale) { sc = 1.0 / (1.0 + sqrt(hll)); lm_scale[l] = sc; }
    else sc = lm_scale[l];
    const double hreg = hll + (mu > 0.0 ? lm_reg(hll, sc, mu) : 0.0);
    const double wl = 1.0 / hreg;
    const bool finite = isfinite(wl);
    lm_aux_store(aux + l, hreg, gl, hll);
    const real wr = finite ? (real)wl : (real)0;
    wv[l] = mk2(wr, wr * (real)gl);
    msk[l] = finite ? (int)(targets | (1u << anchor)) : 0;
    const unsigned freem = ~fixed & ((1u << N) - 1u);
    if ((freem >> anchor) & 1u) {                    // free anchor: materialise its block
        real2 ha[3] = {mk2((real)0, (real)0), mk2((real)0, (real)0), mk2((real)0, (real)0)};
#pragma unroll 4
        for (int f = 0; f < kMaxFrames; ++f) {
            if (!((targets >> f) & 1u)) continue;
            const real2 *p = reinterpret_cast<const real2 *>(hs + ((size_t)f * a.Mcap + l) * 6);
#pragma unroll
            for (int e = 0; e < 3; ++e) { const real2 v = p[e]; ha[e].x -= v.x; ha[e].y -= v.y; }
        }
        real2 *p = reinterpret_cast<real2 *>(hs + ((size_t)anchor * a.Mcap + l) * 6);
        p[0] = ha[0]; p[1] = ha[1]; p[2] = ha[2];
    }
    for (unsigned fm = freem & ~(targets | (1u << anchor)); fm; fm &= fm - 1) {
        real2 *p = reinterpret_cast<real2 *>(hs + ((size_t)(__ffs(fm) - 1) * a.Mcap + l) * 6);
        p[0] = mk2((real)0, (real)0); p[1] = p[0]; p[2] = p[0];
    }
}

template <typename real>
__global__ void __launch_bounds__(128) lm_finish_kernel(PipeArgs a_in) {
    PipeArgs a = a_in;
    const int w = a.slots ? a.slots[blockIdx.y] : blockIdx.y + a.w0;
    const int bsel = pipe_buffer(a, w);
    if (bsel < 0) return;
    pipe_select(a, bsel);
    const WinHdr &H = a.hdr[w];
    const int l = blockIdx.x * blockDim.x + threadIdx.x;
    if (l >= ((H.M + 3) & ~3)) return;
    const double mu = pipe_mu(a, w);
    const int compute_scale = a.loop ? (a.ctrl[w].have_scale == 0) : a.compute_scale;
    lm_finish<real>(a, w, l, H.N, H.M, (unsigned)H.fixed_mask & ((1u << H.N) - 1u), mu, compute_scale);
}

template <typename real>
__host__ __device__ inline size_t lin_smem_layout(int N, int Mp, int warps, bool part, size_t *o_dta, size_t *o_seg, size_t *o_rec,
                                                  size_t *o_rs, size_t *o_skip, size_t *o_part) {
    const size_t nsp = (size_t)N * (N - 1) / 2;
    size_t off = sizeof(double) * 12 * (size_t)N;                              // frames: Rwc[9], c[3]
    *o_dta = off; off += sizeof(double) * ((nsp + 1 + (size_t)N) * kDta + 8);  // direct blocks (pairs, then per frame), cost
    *o_seg = off; off += sizeof(int32_t) * kSegTab;
    off = (off + 15) & ~(size_t)15;
    *o_rec = off; off += (size_t)kLmSm * Mp;                                   // landmark records (lm_sm_store)
    *o_part = off; if (part) off += sizeof(double2) * (size_t)warps * Mp;      // per-warp (j.j, j.r) sums (PipeArgs::lm_part)
    *o_rs = off; off += sizeof(real) * 12 * (size_t)N;                         // (real) Rwc of every frame
    *o_skip = off; off += (size_t)Mp;                                          // 1: landmark not linearised (victim-only sweeps)
    return (off + 15) & ~(size_t)15;
}

template <typename real>
__host__ __device__ inline size_t lin_smem_bytes(int N, int Mp, int warps, bool part) {
    size_t a, b, c, d, e, f;
    return lin_smem_layout<real>(N, Mp, warps, part, &a, &b, &c, &d, &e, &f);
}

// kRows: rows of a piece a lane linearises per iteration (1 or 2: two independent blocks in flight against the latency
// of the fp64 -> cvt -> MUFU chains, at the price of registers); the results do not depend on it
template <bool kLoss, typename real, int kWarps, int kMinBlocks, int kRows = 1>
__global__ void __launch_bounds__(kWarps * 32, kMinBlocks)
lin_obs_kernel(PipeArgs a_in) {
    static_assert(kRows == 1 || kRows == 2, "one or two rows per iteration");
    typedef typename Vec2<real>::type real2;
    constexpr int kThreads = kWarps * 32;
    PipeArgs a = a_in;
    const int w = a.slots ? a.slots[blockIdx.y] : blockIdx.y + a.w0;
    const int bsel = pipe_buffer(a, w);
    if (bsel < 0) return;
    pipe_select(a, bsel);
    if (pipe_at_candidate(a, w)) { a.frames = a.frames_cand; a.rho = a.rho_cand; }
    const WinHdr &H = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int N = H.N, M = H.M;
    const int Mp = (M + 31) & ~31;
    const int tid = threadIdx.x, lane = tid & 31, wv = tid >> 5;
    const int nsp = N * (N - 1) / 2;

    extern __shared__ __align__(16) unsigned char smem_raw[];
    const bool lpart = a.lm_part != 0;
    size_t o_dta, o_seg, o_rec, o_rs, o_skip, o_part;
    lin_smem_layout<real>(N, Mp, kWarps, lpart, &o_dta, &o_seg, &o_rec, &o_rs, &o_skip, &o_part);
    double *Fs = reinterpret_cast<double *>(smem_raw);                       // [N][12]
    double *Dta = reinterpret_cast<double *>(smem_raw + o_dta);              // [nsp + 1][kDta]
    double *Ddg = Dta + (nsp + 1) * kDta;                                    // [N][kDta] sum of the blocks touching frame f (signed gradient)
    double *cost_sm = Ddg + N * kDta;                                        // [8]
    int32_t *sg = reinterpret_cast<int32_t *>(smem_raw + o_seg);             // seg_begin | seg_row
    unsigned char *recs = smem_raw + o_rec;                                  // [Mp] landmark records
    real *Rs = reinterpret_cast<real *>(smem_raw + o_rs);                    // [N][12] (real) Rwc
    unsigned char *skip = smem_raw + o_skip;
    double2 *part = reinterpret_cast<double2 *>(smem_raw + o_part);         // [kWarps][Mp] when lpart

    // The CTA's set-up is a chain of dependent loads at the latency of a loaded memory system, with at most three CTAs per
    // SM to hide it; so the loads that depend only on w (segment table, frame states) are issued first, ahead of the L2
    // read-ahead, and the per-landmark loads of phase 0 and of the epilogue go out kLmBatch at a time.
    constexpr int kSegPer = (kSegTab + kThreads - 1) / kThreads;
    int32_t sgv[kSegPer];
#pragma unroll
    for (int j = 0; j < kSegPer; ++j) {
        const int i = tid + j * kThreads;
        sgv[j] = i < kSegTab ? a.seg[(size_t)w * kSegTab + i] : 0;
    }
    FrameSm f;
    if (tid < a.Ncap) make_frame(a.frames + ((size_t)w * a.Ncap + tid) * kFrameStride, wc, f);   // stored for tid < N
    if (gridDim.x == 1) {          // everything this CTA will read from HBM, requested before the first dependent load
        l2_prefetch(a.fz + (size_t)w * a.Kcap, sizeof(float2) * (size_t)H.K, tid, kThreads);
        l2_prefetch(a.flm + (size_t)w * a.Kcap, sizeof(FLm) * (size_t)H.K, tid, kThreads);
        l2_prefetch(a.lms + (size_t)w * a.Mcap, sizeof(LmRec) * (size_t)M, tid, kThreads);
        l2_prefetch(a.rho + (size_t)w * a.Mcap, sizeof(double) * (size_t)M, tid, kThreads);
    }
    if (tid < N) {
#pragma unroll
        for (int i = 0; i < 9; ++i) Fs[tid * 12 + i] = f.Rwc[i];
#pragma unroll
        for (int i = 0; i < 3; ++i) Fs[tid * 12 + 9 + i] = f.c[i];
#pragma unroll
        for (int i = 0; i < 9; ++i) Rs[tid * 12 + i] = (real)f.Rwc[i];
    }
    for (int i = tid; i < (nsp + 1 + N) * kDta + 8; i += kThreads) Dta[i] = 0.0;
#pragma unroll
    for (int j = 0; j < kSegPer; ++j) if (tid + j * kThreads < kSegTab) sg[tid + j * kThreads] = sgv[j];
    if (lpart) for (int i = tid; i < kWarps * Mp; i += kThreads) part[i] = make_double2(0.0, 0.0);
    __syncthreads();

    // ---- phase 0: world points (reprojection_error_cost.h:58-60)
    const LmRec *lms = a.lms + (size_t)w * a.Mcap;
    const double *rho = a.rho + (size_t)w * a.Mcap;
    for (int l0 = tid; l0 < Mp; l0 += kLmBatch * kThreads) {
        LmRec lr[kLmBatch] = {};
        double rh[kLmBatch] = {};
#pragma unroll
        for (int j = 0; j < kLmBatch; ++j) {
            const int l = l0 + j * kThreads;
            if (l < M) { lr[j] = lms[l]; rh[j] = rho[l]; }
        }
#pragma unroll
        for (int j = 0; j < kLmBatch; ++j) {
            const int l = l0 + j * kThreads;
            if (l >= Mp) break;
            unsigned char sk = 1;
            double x0 = 0.0, x1 = 0.0, x2 = 1.0;
            real c0 = 0, c1 = 0, c2 = 0;
            if (l < M && lm_nobs(lr[j].meta) > 0 && !(a.victim_only && !lm_victim(lr[j].meta))) {
                const double *Fa = Fs + lm_anchor(lr[j].meta) * 12;
                const double ir = 1.0 / rh[j];
                const double zx = (double)lr[j].zrx, zy = (double)lr[j].zry;
                const double v0 = (Fa[0] * zx + Fa[1] * zy + Fa[2]) * ir;
                const double v1 = (Fa[3] * zx + Fa[4] * zy + Fa[5]) * ir;
                const double v2 = (Fa[6] * zx + Fa[7] * zy + Fa[8]) * ir;
                x0 = v0 + Fa[9]; x1 = v1 + Fa[10]; x2 = v2 + Fa[11];
                c0 = (real)ir;          // linearize_blk forms d r / d rho from 1 / rho and the segment's baseline
                sk = 0;
            }
            lm_sm_store(recs + (size_t)l * kLmSm, x0, x1, x2, c0, c1, c2);
            skip[l] = sk;
        }
    }
    __syncthreads();

    // ---- phase 1: rows of the frame-major table
    const real W[4] = {(real)wc.sic[0], (real)wc.sic[1], (real)wc.sic[2], (real)wc.sic[3]};
    const real inv_cb = (real)(1.0 / (wc.cauchy_a * wc.cauchy_a));
    const bool diag_w = wc.sic[1] == 0.0 && wc.sic[2] == 0.0;
    const bool vo = a.victim_only != 0;      // only then can a landmark of the table be left out (skip[])
    const float2 *fz = a.fz + (size_t)w * a.Kcap;
    const FLm *flm = a.flm + (size_t)w * a.Kcap;
    real *hs = reinterpret_cast<real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    real2 *jr = reinterpret_cast<real2 *>(a.jr) + (size_t)w * a.Ncap * a.Mcap;
    const unsigned fixed = (unsigned)H.fixed_mask & ((1u << N) - 1u);
    const int32_t *sbeg = sg, *srow = sg + kMaxSeg + 1;
    const int rows = srow[nsp];
    const int nwt = gridDim.x * kWarps, wid = blockIdx.x * kWarps + wv;
    const int r_begin = (int)((long long)rows * wid / nwt), r_end = (int)((long long)rows * (wid + 1) / nwt);

    unsigned recs_a = (unsigned)__cvta_generic_to_shared(recs);
    asm volatile("" : "+r"(recs_a));           // opaque: ptxas would otherwise re-derive the base from (N, Mp) in every row
    unsigned part_w = (unsigned)__cvta_generic_to_shared(part) + (unsigned)(wv * Mp) * (unsigned)sizeof(double2);   // this warp's partial
    asm volatile("" : "+r"(part_w));
    RowCursor cs(sbeg, srow, r_begin, rows);
    real cost_acc = 0;
    LogAcc<real> la;
    while (cs.r < r_end) {
        const int sp = cs.sp, t = cs.t, an = cs.an;
        const int seg_end = sbeg[sp + 1];
        const int r_stop = min(min(r_end, srow[sp + 1]), cs.r + 64);      // pieces of <= 64 rows: <= 64 terms per thread in `real`
        const bool need = (((fixed >> t) & (fixed >> an)) & 1u) == 0u;    // both blocks constant: only H_ll, g_l, cost
        FrameR<real> F;
        real bt[3];                   // Rwc_t^T (c_an - c_t): the segment's baseline in the target camera
        {
            const double *Ft = Fs + t * 12, *Fa = Fs + an * 12;
            const real *Rt = Rs + t * 12;
#pragma unroll
            for (int i = 0; i < 9; ++i) { F.Rwc[i] = Ft[i]; F.R[i] = Rt[i]; }
#pragma unroll
            for (int i = 0; i < 3; ++i) F.c[i] = Ft[9 + i];
            const double d0 = Fa[9] - Ft[9], d1 = Fa[10] - Ft[10], d2 = Fa[11] - Ft[11];
#pragma unroll
            for (int j = 0; j < 3; ++j) bt[j] = (real)(Ft[j] * d0 + Ft[3 + j] * d1 + Ft[6 + j] * d2);
        }
        const unsigned tM = (unsigned)t * (unsigned)a.Mcap;       // this segment's slice of the record arrays
        real2 q[15];
#pragma unroll
        for (int i = 0; i < 15; ++i) q[i] = mk2((real)0, (real)0);
        // one reduction per (warp, segment piece); the cross-lane sum runs in fp64: lane e ends up with entry e of the 30 sums
        auto flush_q = [&]() {
            double qq[32];
#pragma unroll
            for (int i = 0; i < 15; ++i) { qq[2 * i] = (double)q[i].x; qq[2 * i + 1] = (double)q[i].y; q[i] = mk2((real)0, (real)0); }
            qq[30] = 0.0; qq[31] = 0.0;
            const double tot = transpose_reduce<double>(qq, lane);
            const int e = kQSlot[lane];
            if (e >= 0) atomicAdd(&Dta[sp * kDta + e], tot);          // +sum Y^T Y, Y^T r; the epilogue applies the signs
        };
        // what one linearised block of landmark l adds, in row order: the cost, (j.j, j.r), h_t, Y^T Y and Y^T r
        auto emit = [&](const ObsL<real> &ol, int l) {
            if (kLoss) la.add(ol.cost); else cost_acc += ol.cost;
            const unsigned rec = tM + (unsigned)l;
            const real2 jj = mk2(ol.j0 * ol.j0 + ol.j1 * ol.j1, ol.j0 * ol.r0 + ol.j1 * ol.r1);
            if (lpart) {        // the warp's own partial; a row holds a landmark at most once: no two lanes collide
                part_add(part_w + (unsigned)l * (unsigned)sizeof(double2), make_double2((double)jj.x, (double)jj.y));
            } else {
                jr[rec] = jj;
            }
            if (need) {
                real2 h[3];
#pragma unroll
                for (int p = 0; p < 3; ++p) h[p] = bfma(ol.j1, ol.Y1[p], bmul(ol.j0, ol.Y0[p]));
                real2 *dst = reinterpret_cast<real2 *>(hs) + (size_t)rec * 3;
                dst[0] = h[0]; dst[1] = h[1]; dst[2] = h[2];
                const real y0[6] = {ol.Y0[0].x, ol.Y0[0].y, ol.Y0[1].x, ol.Y0[1].y, ol.Y0[2].x, ol.Y0[2].y};
                const real y1[6] = {ol.Y1[0].x, ol.Y1[0].y, ol.Y1[1].x, ol.Y1[1].y, ol.Y1[2].x, ol.Y1[2].y};
                // upper triangle of Y^T Y by column pairs, then Y^T r
                q[0] = bfma(y1[0], ol.Y1[0], bfma(y0[0], ol.Y0[0], q[0]));
                q[1] = bfma(y1[0], ol.Y1[1], bfma(y0[0], ol.Y0[1], q[1]));
                q[2] = bfma(y1[0], ol.Y1[2], bfma(y0[0], ol.Y0[2], q[2]));
                q[3] = bfma(y1[1], ol.Y1[0], bfma(y0[1], ol.Y0[0], q[3]));
                q[4] = bfma(y1[1], ol.Y1[1], bfma(y0[1], ol.Y0[1], q[4]));
                q[5] = bfma(y1[1], ol.Y1[2], bfma(y0[1], ol.Y0[2], q[5]));
                q[6] = bfma(y1[2], ol.Y1[1], bfma(y0[2], ol.Y0[1], q[6]));
                q[7] = bfma(y1[2], ol.Y1[2], bfma(y0[2], ol.Y0[2], q[7]));
                q[8] = bfma(y1[3], ol.Y1[1], bfma(y0[3], ol.Y0[1], q[8]));
                q[9] = bfma(y1[3], ol.Y1[2], bfma(y0[3], ol.Y0[2], q[9]));
                q[10] = bfma(y1[4], ol.Y1[2], bfma(y0[4], ol.Y0[2], q[10]));
                q[11] = bfma(y1[5], ol.Y1[2], bfma(y0[5], ol.Y0[2], q[11]));
                q[12] = bfma(ol.r1, ol.Y1[0], bfma(ol.r0, ol.Y0[0], q[12]));
                q[13] = bfma(ol.r1, ol.Y1[1], bfma(ol.r0, ol.Y0[1], q[13]));
                q[14] = bfma(ol.r1, ol.Y1[2], bfma(ol.r0, ol.Y0[2], q[14]));
            }
        };
        // the table entries of the NEXT row (kRows = 2: the next two rows) are requested before the current ones are evaluated
        int k = cs.k0() + lane;
        const float2 *pz = fz + k;
        const FLm *pl = flm + k;
        float2 z_nx = make_float2(0.f, 0.f);
        int l_nx = 0;
        if (k < seg_end) { z_nx = *pz; l_nx = *pl; }
        const int nrow = r_stop - cs.r;
        if constexpr (kRows == 1) {
            for (int i = 0; i < nrow; ++i) {
                const float2 z = z_nx;
                const int l = l_nx;
                const bool valid = k < seg_end;
                k += 32; pz += 32; pl += 32;
                if (i + 1 < nrow && k < seg_end) { z_nx = *pz; l_nx = *pl; }
                if (valid) {
                    if (!(vo && skip[l])) {
                        ObsL<real> ol;
                        double x[3];
                        real xf[3], ir[3];             // ir = (1 / rho, 0, 0)
                        lm_sm_load(recs_a + (unsigned)l * kLmSm, x, xf, ir);
                        linearize_blk<kLoss, real>(F, x[0], x[1], x[2], xf[0], xf[1], xf[2], ir[0], bt, z.x, z.y, W,
                                                   diag_w, inv_cb, ol);
                        emit(ol, l);
                    }
                }
                if (kLoss && (i & 3) == 3) la.fold();
            }
        } else {
            // rows i and i + 1 per iteration: two independent linearisations in flight per lane, then their
            // contributions in row order, so every sum sees the terms of the one-row loop in the same order.  Both blocks
            // are evaluated unconditionally (a lane past the segment's end, or past an odd piece's last row, works on
            // the record of a landmark it read earlier, or record 0) and only the live ones are emitted.
            float2 z_nx1 = make_float2(0.f, 0.f);
            int l_nx1 = 0;
            if (nrow > 1 && k + 32 < seg_end) { z_nx1 = fz[k + 32]; l_nx1 = flm[k + 32]; }
            for (int i = 0; i < nrow; i += 2) {
                const float2 z0 = z_nx, z1 = z_nx1;
                const int l0 = l_nx, l1 = l_nx1;
                const bool has1 = i + 1 < nrow;
                const bool live0 = k < seg_end && !(vo && skip[l0]);
                const bool live1 = has1 && k + 32 < seg_end && !(vo && skip[l1]);
                k += 64;                  // the table is addressed from k (no running pointers: registers)
                if (i + 2 < nrow && k < seg_end) { z_nx = fz[k]; l_nx = flm[k]; }
                if (i + 3 < nrow && k + 32 < seg_end) { z_nx1 = fz[k + 32]; l_nx1 = flm[k + 32]; }
                ObsL<real> o0, o1;
                double x0[3], x1[3];
                real xf0[3], ir0[3], xf1[3], ir1[3];
                lm_sm_load(recs_a + (unsigned)l0 * kLmSm, x0, xf0, ir0);
                lm_sm_load(recs_a + (unsigned)l1 * kLmSm, x1, xf1, ir1);
                linearize_blk<kLoss, real>(F, x0[0], x0[1], x0[2], xf0[0], xf0[1], xf0[2], ir0[0], bt, z0.x, z0.y, W,
                                           diag_w, inv_cb, o0);
                linearize_blk<kLoss, real>(F, x1[0], x1[1], x1[2], xf1[0], xf1[1], xf1[2], ir1[0], bt, z1.x, z1.y, W,
                                           diag_w, inv_cb, o1);
                if (live0) emit(o0, l0);
                if (live1) emit(o1, l1);
                if (kLoss && has1 && (i & 3) == 2) la.fold();     // after rows 3, 7, 11, ... as in the one-row loop
            }
        }
        if (kLoss && (nrow & 3)) la.fold();         // never more than 4 factors in the product
        cs.r = r_stop; cs.seek();
        if (need) flush_q();
    }

    // ---- epilogue
    if (kLoss) cost_acc = (real)0.5 * (real)(wc.cauchy_a * wc.cauchy_a) * la.total();
    double cd = (double)cost_acc;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) cd += __shfl_xor_sync(0xffffffffu, cd, off);
    if (lane == 0) atomicAdd(&cost_sm[0], cd);
    __syncthreads();
    const bool exclusive = (gridDim.x == 1);
    if (exclusive) {       // this CTA wrote every record of the window: complete the landmarks here
        const double mu = pipe_mu(a, w);
        const int compute_scale = a.loop ? (a.ctrl[w].have_scale == 0) : a.compute_scale;
        const int Mq = (M + 3) & ~3;
        for (int l0 = tid; l0 < Mq; l0 += kLmBatch * kThreads) {
            LmRec lr[kLmBatch] = {};
#pragma unroll
            for (int j = 0; j < kLmBatch; ++j)
                if (l0 + j * kThreads < M) lr[j] = lms[l0 + j * kThreads];
#pragma unroll
            for (int j = 0; j < kLmBatch; ++j)
                if (l0 + j * kThreads < Mq)
                    lm_finish<real>(a, w, l0 + j * kThreads, N, M, fixed, mu, compute_scale, lpart ? part : nullptr, kWarps, Mp, &lr[j]);
        }
    }
    // direct part of the reduced system (schur_kernel subtracts the Schur sum from Hred / gred).  D(t, a) enters the
    // off-diagonal block (t, a) with a minus sign and BOTH diagonal blocks with a plus sign; its gradient part enters
    // g[t] with a plus and g[a] with a minus sign: first the per-frame sums (thread per (frame, entry)), then the copies
    for (int e = tid; e < N * kDta; e += kThreads) {
        const int f = e / kDta, v = e - f * kDta;
        double d = 0.0;
        for (int g = 0; g < f; ++g) d += Dta[spair(f, g) * kDta + v];                       // f is the target
        for (int g = f + 1; g < N; ++g) { const double x = Dta[spair(g, f) * kDta + v]; d += v < 21 ? x : -x; }   // f is the anchor
        Ddg[e] = d;
    }
    __syncthreads();
    const int npairs_cap = a.Ncap * (a.Ncap + 1) / 2;
    double *Hred_o = a.Hred + (size_t)w * npairs_cap * 36;
    double *Hdd_o = a.Hdd + (size_t)w * a.Ncap * 36;
    double *gdir_o = a.gdir + (size_t)w * a.Ncap * 6;
    double *gred_o = a.gred + (size_t)w * a.Ncap * 6;
    for (int e = tid; e < N * 36; e += kThreads) {                  // diagonal blocks
        const int f = e / 36, ij = e - f * 36, i = ij / 6, j = ij - i * 6;
        const double d = Ddg[f * kDta + (i <= j ? sym6(i, j) : sym6(j, i))];
        if (exclusive) { Hdd_o[e] = d; Hred_o[pair_idx(f, f) * 36 + ij] = d; }
        else if (d != 0.0) { atomicAdd(&Hdd_o[e], d); atomicAdd(&Hred_o[pair_idx(f, f) * 36 + ij], d); }
    }
    int fo = 1;                                                     // sq grows with e: fo only moves on (at most N - 2 steps)
    for (int e = tid; e < nsp * 36; e += kThreads) {                // off-diagonal blocks (f > g): -D(f, g)
        const int sq = e / 36, ij = e - sq * 36, i = ij / 6, j = ij - i * 6;
        while ((fo + 1) * fo / 2 <= sq) ++fo;
        const int g = sq - fo * (fo - 1) / 2;
        const double v = -Dta[sq * kDta + (i <= j ? sym6(i, j) : sym6(j, i))];
        if (exclusive) Hred_o[pair_idx(fo, g) * 36 + ij] = v; else if (v != 0.0) atomicAdd(&Hred_o[pair_idx(fo, g) * 36 + ij], v);
    }
    for (int e = tid; e < N * 6; e += kThreads) {                   // gradients
        const double d = Ddg[(e / 6) * kDta + 21 + e % 6];
        if (exclusive) { gdir_o[e] = d; gred_o[e] = d; }
        else if (d != 0.0) { atomicAdd(&gdir_o[e], d); atomicAdd(&gred_o[e], d); }
    }
    if (tid == 0) {
        if (exclusive) a.cost_vis[w] = cost_sm[0]; else atomicAdd(&a.cost_vis[w], cost_sm[0]);
    }
}

}  // namespace pvio
