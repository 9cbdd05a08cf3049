// The F-matrix outlier rejection of OpenCvImage::track_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:121-129):
//
//     findFundamentalMat(p, q, cv::FM_RANSAC, 1.0, 0.99, mask)
//
// OpenCV (absent from /root/reference; the published algorithm of calib3d/fundam.cpp + ptsetreg.cpp, restated and pinned
// against cv2 4.13.0 in oracle/fm_oracle.py) runs a SERIAL loop: draw 7 matches, 7-point solve (1..3 models), count the
// inliers of each model over all matches, keep a model with more inliers than the best so far and shrink the iteration
// budget from the new outlier ratio.  Nothing in an iteration depends on the previous ones except that budget.
//
// Here: SPECULATIVE evaluation + serial-equivalent replay.
//   host     the sample schedule: cv::RNG((uint64)-1) and getSubset (7 distinct indices, the collinearity test of the
//            last point) restated, so the schedule IS OpenCV's -- or the schedule the caller injects (the batched
//            tracker draws the same schedule on the device, fm_schedule_kernel)
//   device   fm_hypotheses_kernel: one warp per iteration of the schedule, ALL max_iters of them at once (1000 warps):
//            lane 0 solves the 7-point problem (Hartley normalisation, null space of the 7 x 9 system by a Householder
//            QR of its transpose, the cubic det(lambda f1 + (1 - lambda) f2) = 0 with cv::solveCubic's branches and
//            root order, de-normalisation), every lane then takes matches lane, lane + 32, ...: the symmetric epipolar
//            error of computeError in double, rounded to float, compared with (float) threshold^2; inlier bit masks by
//            ballot, counts by popc.  For 8 <= n < 15 OpenCV switches to LMedS: the same kernel returns the median error
//            (element n / 2 in the order of the float bit patterns, as std::nth_element on int sees them)
//   host     the replay: walk the iterations in order with OpenCV's acceptance rule and RANSACUpdateNumIters (the
//            host's own log / pow, as OpenCV's) and stop where the serial loop would have stopped; the mask of the
//            winning (iteration, model) is the result.  12 KB of counts come back, then 128 bytes of mask.
// The result is the one the serial loop produces for that schedule, whatever the inlier ratio; the device does at most
// 1000 x 3 x n error evaluations (0.4 GFLOP at n = 400) in one wave.
//
// Compiled with -fmad=false: OpenCV's scalar double code is not contracted.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"

namespace pvio {
namespace {

// ---- host and device: OpenCV's sample schedule ----------------------------------------------------------------------
// One implementation for both sides: the single call draws it on the host, the batched tracker on the device (one
// thread per frame pair, fm_schedule_kernel).  Integer RNG and unfused double arithmetic: the two draw the same subsets.
struct CvRng {                       // cv::RNG (core/operations.hpp): multiply-with-carry
    uint64_t state;
    __host__ __device__ explicit CvRng(uint64_t s) : state(s ? s : 0xffffffffULL) {}
    __host__ __device__ unsigned next() {
        state = (uint64_t)(unsigned)state * 4164903690U + (unsigned)(state >> 32);
        return (unsigned)state;
    }
    __host__ __device__ int uniform(int a, int b) { return a == b ? a : (int)(next() % (unsigned)(b - a) + a); }
};

// fundam.cpp haveCollinearPoints: the LAST of `count` points against every pair before it
__host__ __device__ __forceinline__ bool last_point_collinear(const float *pts, const int *idx, int count) {
    const int i = count - 1;
    const float xi = pts[2 * idx[i]], yi = pts[2 * idx[i] + 1];
    for (int j = 0; j < i; ++j) {
        const double dx1 = pts[2 * idx[j]] - xi, dy1 = pts[2 * idx[j] + 1] - yi;
        for (int k = 0; k < j; ++k) {
            const double dx2 = pts[2 * idx[k]] - xi, dy2 = pts[2 * idx[k] + 1] - yi;
            if (fabs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (fabs(dx1) + fabs(dy1) + fabs(dx2) + fabs(dy2)))
                return true;
        }
    }
    return false;
}

// ptsetreg.cpp getSubset for every iteration the loop could run: iteration `it` always consumes exactly one subset.
// Returns the number of iterations that have a subset (getSubset giving up ends the loop; its row holds the last try).
// The subset is drawn in a local array, which the unrolled loops keep in registers on the device: the serial chain of
// draws and collinearity tests then never waits on a load of its own subset from global memory.
__host__ __device__ int cv_schedule(const float *p, const float *q, int n, int iters, int max_attempts, int *sched) {
    CvRng rng((uint64_t)-1);
    for (int it = 0; it < iters; ++it) {
        int idx[7];
        int attempt = 0;
        for (; attempt < max_attempts; ++attempt) {
#pragma unroll
            for (int i = 0; i < 7; ++i) {
                int v;
                bool dup;
                do {
                    v = rng.uniform(0, n);
                    dup = false;
#pragma unroll
                    for (int j = 0; j < i; ++j) dup |= idx[j] == v;
                } while (dup);
                idx[i] = v;
            }
            if (!last_point_collinear(p, idx, 7) && !last_point_collinear(q, idx, 7)) break;
        }
        for (int i = 0; i < 7; ++i) sched[7 * it + i] = idx[i];
        if (attempt == max_attempts) return it;
    }
    return iters;
}

// ptsetreg.cpp RANSACUpdateNumIters
int ransac_update_num_iters(double p, double ep, int model_points, int max_iters) {
    p = std::fmax(p, 0.); p = std::fmin(p, 1.);
    ep = std::fmax(ep, 0.); ep = std::fmin(ep, 1.);
    double num = std::fmax(1. - p, DBL_MIN);
    double denom = 1. - std::pow(1. - ep, model_points);
    if (denom < DBL_MIN) return 0;
    num = std::log(num);
    denom = std::log(denom);
    return denom >= 0 || -num >= max_iters * (-denom) ? max_iters : (int)std::nearbyint(num / denom);   // cvRound
}

// ---- device ---------------------------------------------------------------------------------------------------------
// cv::solveCubic (core/mathfuncs.cpp) for double coefficients; roots in OpenCV's order
__device__ int solve_cubic(double a0, double a1, double a2, double a3, double *x) {
    const double kPi = 3.1415926535897932384626433832795;
    if (a0 == 0) {
        if (a1 == 0) {
            if (a2 == 0) return a3 == 0 ? -1 : 0;
            x[0] = -a3 / a2;
            return 1;
        }
        double d = a2 * a2 - 4 * a1 * a3;
        if (d < 0) return 0;
        d = sqrt(d);
        const double q1 = (-a2 + d) * 0.5, q2 = (a2 + d) * -0.5;
        if (fabs(q1) > fabs(q2)) { x[0] = q1 / a1; x[1] = a3 / q1; }
        else { x[0] = q2 / a1; x[1] = a3 / q2; }
        return d > 0 ? 2 : 1;
    }
    a0 = 1. / a0;
    a1 *= a0; a2 *= a0; a3 *= a0;
    const double Q = (a1 * a1 - 3 * a2) * (1. / 9);
    const double R = (2 * a1 * a1 * a1 - 9 * a1 * a2 + 27 * a3) * (1. / 54);
    const double Qcubed = Q * Q * Q;
    double d = Qcubed - R * R;
    if (d > 0) {
        const double theta = acos(R / sqrt(Qcubed));
        const double sqrtQ = sqrt(Q);
        const double t0 = -2 * sqrtQ, t1 = theta * (1. / 3), t2 = a1 * (1. / 3);
        x[0] = t0 * cos(t1) - t2;
        x[1] = t0 * cos(t1 + (2. * kPi / 3)) - t2;
        x[2] = t0 * cos(t1 + (4. * kPi / 3)) - t2;
        return 3;
    }
    if (d == 0) {
        if (R >= 0) { x[0] = -2 * pow(R, 1. / 3) - a1 / 3; x[1] = pow(R, 1. / 3) - a1 / 3; }
        else { x[0] = 2 * pow(-R, 1. / 3) - a1 / 3; x[1] = -pow(-R, 1. / 3) - a1 / 3; }
        return x[0] == x[1] ? 1 : 2;
    }
    d = sqrt(-d);
    double e = pow(d + fabs(R), 1. / 3);
    if (R > 0) e = -e;
    x[0] = (e + Q / e) - a1 * (1. / 3);
    return 1;
}

// fundam.cpp run7Point on the 7 matches idx[0..6]; models row-major into F[k][9].  Returns the model count (<= 0: none).
__device__ int seven_point(const float2 *p, const float2 *q, const int *idx, double (*F)[9]) {
    double px[7], py[7], qx[7], qy[7];
    double c1x = 0, c1y = 0, c2x = 0, c2y = 0;
    for (int i = 0; i < 7; ++i) {
        const float2 a = p[idx[i]], b = q[idx[i]];
        px[i] = a.x; py[i] = a.y; qx[i] = b.x; qy[i] = b.y;
        c1x += px[i]; c1y += py[i]; c2x += qx[i]; c2y += qy[i];
    }
    const double t = 1. / 7;
    c1x *= t; c1y *= t; c2x *= t; c2y *= t;
    double scale1 = 0, scale2 = 0;
    for (int i = 0; i < 7; ++i) {
        const double ax = px[i] - c1x, ay = py[i] - c1y, bx = qx[i] - c2x, by = qy[i] - c2y;
        scale1 += sqrt(ax * ax + ay * ay);
        scale2 += sqrt(bx * bx + by * by);
    }
    scale1 *= t; scale2 *= t;
    if (scale1 < (double)FLT_EPSILON || scale2 < (double)FLT_EPSILON) return 0;
    scale1 = sqrt(2.) / scale1;
    scale2 = sqrt(2.) / scale2;

    // M = A^T (9 x 7): column i is the equation (m2_i, 1)^T F (m1_i, 1) = 0 of match i
    double M[9][7];
    for (int i = 0; i < 7; ++i) {
        const double x0 = (px[i] - c1x) * scale1, y0 = (py[i] - c1y) * scale1;
        const double x1 = (qx[i] - c2x) * scale2, y1 = (qy[i] - c2y) * scale2;
        M[0][i] = x1 * x0; M[1][i] = x1 * y0; M[2][i] = x1;
        M[3][i] = y1 * x0; M[4][i] = y1 * y0; M[5][i] = y1;
        M[6][i] = x0; M[7][i] = y0; M[8][i] = 1;
    }
    // Householder QR of M; the null space of A is spanned by the last two columns of Q = H_0 ... H_6
    double V[7][9], beta[7];
    for (int k = 0; k < 7; ++k) {
        double nrm = 0;
        for (int r = k; r < 9; ++r) nrm += M[r][k] * M[r][k];
        nrm = sqrt(nrm);
        const double x0 = M[k][k];
        const double alpha = x0 >= 0 ? -nrm : nrm;
        double vv = 0;
        for (int r = k; r < 9; ++r) {
            const double v = r == k ? x0 - alpha : M[r][k];
            V[k][r] = v;
            vv += v * v;
        }
        beta[k] = vv > 0 ? 2. / vv : 0.;
        for (int c = k; c < 7; ++c) {
            double s = 0;
            for (int r = k; r < 9; ++r) s += V[k][r] * M[r][c];
            s *= beta[k];
            for (int r = k; r < 9; ++r) M[r][c] -= s * V[k][r];
        }
    }
    double f1[9], f2[9];
    for (int r = 0; r < 9; ++r) { f1[r] = r == 7; f2[r] = r == 8; }
    for (int k = 6; k >= 0; --k) {
        double s1 = 0, s2 = 0;
        for (int r = k; r < 9; ++r) { s1 += V[k][r] * f1[r]; s2 += V[k][r] * f2[r]; }
        s1 *= beta[k]; s2 *= beta[k];
        for (int r = k; r < 9; ++r) { f1[r] -= s1 * V[k][r]; f2[r] -= s2 * V[k][r]; }
    }

    // f ~ lambda f1 + (1 - lambda) f2, det f = 0: the cubic in lambda (run7Point's expansion)
    for (int i = 0; i < 9; ++i) f1[i] -= f2[i];
    double t0 = f2[4] * f2[8] - f2[5] * f2[7];
    double t1 = f2[3] * f2[8] - f2[5] * f2[6];
    double t2 = f2[3] * f2[7] - f2[4] * f2[6];
    double c[4];
    c[3] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2;
    c[2] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2 -
           f1[3] * (f2[1] * f2[8] - f2[2] * f2[7]) + f1[4] * (f2[0] * f2[8] - f2[2] * f2[6]) -
           f1[5] * (f2[0] * f2[7] - f2[1] * f2[6]) + f1[6] * (f2[1] * f2[5] - f2[2] * f2[4]) -
           f1[7] * (f2[0] * f2[5] - f2[2] * f2[3]) + f1[8] * (f2[0] * f2[4] - f2[1] * f2[3]);
    t0 = f1[4] * f1[8] - f1[5] * f1[7];
    t1 = f1[3] * f1[8] - f1[5] * f1[6];
    t2 = f1[3] * f1[7] - f1[4] * f1[6];
    c[0] = f1[0] * t0 - f1[1] * t1 + f1[2] * t2;
    c[1] = f2[0] * t0 - f2[1] * t1 + f2[2] * t2 -
           f2[3] * (f1[1] * f1[8] - f1[2] * f1[7]) + f2[4] * (f1[0] * f1[8] - f1[2] * f1[6]) -
           f2[5] * (f1[0] * f1[7] - f1[1] * f1[6]) + f2[6] * (f1[1] * f1[5] - f1[2] * f1[4]) -
           f2[7] * (f1[0] * f1[5] - f1[2] * f1[3]) + f2[8] * (f1[0] * f1[4] - f1[1] * f1[3]);
    double roots[3] = {0, 0, 0};
    const int n = solve_cubic(c[0], c[1], c[2], c[3], roots);
    if (n < 1 || n > 3) return n;

    for (int k = 0; k < n; ++k) {
        double lambda = roots[k], mu = 1.;
        const double s = f1[8] * roots[k] + f2[8];
        double f[9];
        if (fabs(s) > DBL_EPSILON) { mu = 1. / s; lambda *= mu; f[8] = 1.; }
        else f[8] = 0.;
        for (int i = 0; i < 8; ++i) f[i] = f1[i] * lambda + f2[i] * mu;
        // F = T2^T f T1, T = [s 0 -s cx; 0 s -s cy; 0 0 1]
        double G[9];                                    // G = f T1
        for (int r = 0; r < 3; ++r) {
            G[3 * r + 0] = f[3 * r + 0] * scale1;
            G[3 * r + 1] = f[3 * r + 1] * scale1;
            G[3 * r + 2] = f[3 * r + 0] * (-scale1 * c1x) + f[3 * r + 1] * (-scale1 * c1y) + f[3 * r + 2];
        }
        double *o = F[k];
        for (int cc = 0; cc < 3; ++cc) {
            o[0 + cc] = scale2 * G[0 + cc];
            o[3 + cc] = scale2 * G[3 + cc];
            o[6 + cc] = (-scale2 * c2x) * G[0 + cc] + (-scale2 * c2y) * G[3 + cc] + G[6 + cc];
        }
        if (fabs(o[8]) > (double)FLT_EPSILON) {
            const double inv = 1. / o[8];
            for (int i = 0; i < 9; ++i) o[i] *= inv;
        }
    }
    return n;
}

// FMEstimatorCallback::computeError for one match
__device__ __forceinline__ float fm_error(const double *F, float2 m1, float2 m2) {
    double a = F[0] * m1.x + F[1] * m1.y + F[2];
    double b = F[3] * m1.x + F[4] * m1.y + F[5];
    double c = F[6] * m1.x + F[7] * m1.y + F[8];
    const double s2 = 1. / (a * a + b * b);
    const double d2 = m2.x * a + m2.y * b + c;
    a = F[0] * m2.x + F[3] * m2.y + F[6];
    b = F[1] * m2.x + F[4] * m2.y + F[7];
    c = F[2] * m2.x + F[5] * m2.y + F[8];
    const double s1 = 1. / (a * a + b * b);
    const double d1 = m1.x * a + m1.y * b + c;
    return (float)fmax(d1 * d1 * s1, d2 * d2 * s2);        // std::max(a, b): b if a < b (NaN handling as OpenCV's is not reproduced)
}

constexpr int kWarpsPerCta = 4;

// One warp per iteration of the schedule of problem probs[blockIdx.y], whose match and iteration counts are P.surv (the
// schedule kernel's or the single call's).  RANSAC (n >= 15): counts[it] = {nmodels, inliers of model 0, 1, 2},
// masks[it][k][nw]; LMedS (n < 15): counts[it] = {nmodels, float bits of the median error of model 0, 1, 2}.
__global__ void __launch_bounds__(32 * kWarpsPerCta) fm_hypotheses_kernel(float thr2, const FmBatchProblem *probs) {
    __shared__ double sF[kWarpsPerCta][3][9];
    __shared__ int sN[kWarpsPerCta];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int it = blockIdx.x * kWarpsPerCta + warp;
    const FmBatchProblem &P = probs[blockIdx.y];
    const int n = P.surv[0], iters = P.surv[1], lmeds = n < 15 ? 1 : 0, nw = (n + 31) / 32;    // iters == 0 below 8 survivors
    const float2 *p = P.p, *q = P.q;
    const int *sched = P.sched;
    int *counts = P.counts;
    double *Fout = P.F;
    unsigned *masks = P.masks;
    if (it >= iters) return;
    if (lane == 0) {
        int idx[7];
        for (int i = 0; i < 7; ++i) idx[i] = sched[7 * it + i];
        int nm = 0;
        if (idx[0] >= 0) nm = seven_point(p, q, idx, sF[warp]);
        sN[warp] = nm;
        counts[4 * it] = nm;
        for (int k = 0; k < 3; ++k)
            for (int i = 0; i < 9; ++i) Fout[(size_t)(3 * it + k) * 9 + i] = k < nm ? sF[warp][k][i] : 0.;
    }
    __syncwarp();
    const int nm = sN[warp];
    for (int k = 0; k < 3; ++k) {
        if (k >= nm) {
            if (lane == 0) counts[4 * it + 1 + k] = lmeds ? 0x7f800000 : 0;
            continue;
        }
        double F[9];
        for (int i = 0; i < 9; ++i) F[i] = sF[warp][k][i];
        if (!lmeds) {
            int good = 0;
            for (int w = 0; w < nw; ++w) {
                const int i = 32 * w + lane;
                bool in = false;
                if (i < n) in = fm_error(F, p[i], q[i]) <= thr2;
                const unsigned b = __ballot_sync(0xffffffffu, in);
                good += __popc(b);
                if (lane == 0) masks[((size_t)(3 * it + k)) * nw + w] = b;
            }
            if (lane == 0) counts[4 * it + 1 + k] = good;
        } else {
            // std::nth_element(int bit patterns)[n / 2]: rank by (bits, index)
            const int mine = lane < n ? __float_as_int(fm_error(F, p[lane], q[lane])) : 0x7fffffff;
            int rank = 0;
            for (int j = 0; j < 32; ++j) {
                const int other = __shfl_sync(0xffffffffu, mine, j);
                rank += (other < mine) || (other == mine && j < lane);
            }
            if (lane < n && rank == n / 2) counts[4 * it + 1 + k] = mine;
        }
    }
}

// the mask of the job jobs[blockIdx.y]: LMedS, the inliers of the best model under sigma; RANSAC, a copy of the mask
// fm_hypotheses_kernel stored (n == 7: not needed)
__global__ void fm_mask_kernel(const FmMaskJob *jobs) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const FmMaskJob &J = jobs[blockIdx.y];
    if ((i >> 5) * 32 >= J.n) return;       // whole warps
    unsigned *mask = J.out;
    if (J.src) {
        if ((threadIdx.x & 31) == 0) mask[i >> 5] = J.src[i >> 5];
        return;
    }
    const float2 *p = J.p, *q = J.q;
    const double *Fm = J.F;
    const float thr2 = J.thr2;
    const int n = J.n;
    double F[9];
    for (int k = 0; k < 9; ++k) F[k] = Fm[k];
    bool in = false;
    if (i < n) in = fm_error(F, p[i], q[i]) <= thr2;
    const unsigned b = __ballot_sync(0xffffffffu, in);
    if ((threadIdx.x & 31) == 0) mask[i >> 5] = b;
}

// The batched tracker's step between LK and the hypotheses, one warp per frame pair (opencv_image.cpp:112-121): the
// warp compacts the pair's surviving matches in order, then lane 0 draws OpenCV's schedule over them when there are at
// least 8 -- one serial RNG chain per pair, as cv_schedule on the host.  surv = {survivors, iterations with a subset}.
__global__ void __launch_bounds__(32) fm_schedule_kernel(const FmBatchProblem *probs, int max_iters, int lmeds_iters) {
    const FmBatchProblem &P = probs[blockIdx.x];
    const int lane = threadIdx.x;
    int s = 0;
    for (int base = 0; base < P.n_pts; base += 32) {
        const int i = base + lane;
        const bool keep = i < P.n_pts && P.status[i];
        const unsigned b = __ballot_sync(0xffffffffu, keep);
        if (keep) {
            const int r = s + __popc(b & ((1u << lane) - 1u));
            P.p[r] = make_float2(P.prev_pts[2 * i], P.prev_pts[2 * i + 1]);
            P.q[r] = make_float2(P.next_pts[2 * i], P.next_pts[2 * i + 1]);
        }
        s += __popc(b);
    }
    __syncwarp();
    if (lane != 0) return;
    int have = 0;
    if (s >= 8) {
        const bool ransac = s >= 15;
        have = cv_schedule(reinterpret_cast<const float *>(P.p), reinterpret_cast<const float *>(P.q), s,
                           ransac ? max_iters : lmeds_iters, ransac ? 10000 : 1000, P.sched);
    }
    P.surv[0] = s; P.surv[1] = have;
}

}  // namespace

// host-only: the subsets OpenCV would draw (exported as pvio_b200_fm_sample_schedule)
int fm_cv_schedule(int n, const float *p, const float *q, int iters, int32_t *schedule) {
    return cv_schedule(p, q, n, iters, n >= 15 ? 10000 : 1000, schedule);
}

// findFundamentalMat's defaults for out-of-range options
void fm_options(double &threshold, double &confidence, int &max_iters) {
    if (threshold <= 0) threshold = 3;
    if (confidence < DBL_EPSILON || confidence > 1 - DBL_EPSILON) confidence = 0.99;
    if (max_iters < 1) max_iters = 1;
}

// the iteration budget of the LMedS branch (8 <= n < 15): RANSACUpdateNumIters at the outlier ratio OpenCV assumes
int fm_lmeds_iters(double confidence, int max_iters) { return ransac_update_num_iters(confidence, 0.45, 7, max_iters); }

// The serial loop OpenCV runs over the evaluated iterations counts[have][4] of n matches (7: the 7-point solve, 8..14:
// LMedS, >= 15: RANSAC with at most max_iters iterations), with the host's own log / pow as OpenCV's.  Sets
// inf = {iterations run, winning iteration (-1: none), winning model, method}; returns the threshold of the LMedS
// winner's mask (sigma^2), 0 otherwise.
float fm_replay(const int *counts, int n, int have, int max_iters, double confidence, int *inf) {
    int best_it = -1, best_k = -1, it = 0;
    float thr2 = 0.f;
    if (n == 7) {
        inf[3] = 3;
        if (counts[0] >= 1) { best_it = 0; best_k = 0; }
        it = 1;
    } else if (n >= 15) {
        inf[3] = 1;
        int niters = max_iters, max_good = 0;
        for (; it < niters && it < have; ++it) {
            const int nm = counts[4 * it];
            for (int k = 0; k < nm && k < 3; ++k) {
                const int good = counts[4 * it + 1 + k];
                if (good > std::max(max_good, 6)) {
                    max_good = good; best_it = it; best_k = k;
                    niters = ransac_update_num_iters(confidence, (double)(n - good) / n, 7, niters);
                }
            }
        }
    } else {
        inf[3] = 2;
        double min_median = DBL_MAX;
        for (; it < have; ++it) {
            const int nm = counts[4 * it];
            for (int k = 0; k < nm && k < 3; ++k) {
                float med;
                std::memcpy(&med, &counts[4 * it + 1 + k], 4);
                if ((double)med < min_median) { min_median = med; best_it = it; best_k = k; }
            }
        }
        if (best_it >= 0) {
            double sigma = 2.5 * 1.4826 * (1 + 5. / (n - 7)) * std::sqrt(min_median);
            sigma = std::fmax(sigma, 0.001);
            thr2 = (float)(sigma * sigma);
        }
    }
    inf[0] = it; inf[1] = best_it; inf[2] = best_k;
    return thr2;
}

int fm_ransac_impl(Handle *h, int n, const float *p, const float *q, double threshold, double confidence, int max_iters,
                   const int32_t *schedule, int n_schedule, uint8_t *mask, double *F_out, int32_t *info) {
    int inf[4] = {0, -1, -1, 0};              // iterations run, winning iteration, winning model, method (1 RANSAC, 2 LMedS, 3 seven points)
    auto finish = [&](int rc) { if (info) std::memcpy(info, inf, sizeof(inf)); return rc; };
    if (F_out) std::memset(F_out, 0, 9 * sizeof(double));
    if (n < 7) {                              // findFundamentalMat returns an empty matrix and leaves the mask alone
        if (n > 0) std::memset(mask, 0, n);
        return finish(0);
    }
    fm_options(threshold, confidence, max_iters);
    const bool seven = n == 7, ransac = n >= 15;
    const int budget = seven ? 1 : ransac ? max_iters : fm_lmeds_iters(confidence, max_iters);
    // staging: the problem, its survivor and iteration counts, the matches p[n], q[n] and the schedule [budget][7]
    // (uploaded) | counts [budget][4], the winning model and its mask (downloaded) | the mask job, written after the replay
    // and read in place; device scratch: the models [budget][3][9] and masks [budget][3][words] of every iteration
    const int nw = (n + 31) / 32;
    Stage S(h->fm.stage, &h->fm.scratch);
    S.pow2 = true;
    const auto prob = S.add<FmBatchProblem>(Stage::kUp, 1);
    const auto surv = S.add<int>(Stage::kUp, 2);
    const auto pq = S.add<float2>(Stage::kUp, 2 * (size_t)n);
    const auto sched = S.add<int>(Stage::kUp, 7 * (size_t)budget);
    const auto counts = S.add<int>(Stage::kDown, 4 * (size_t)budget);
    const auto win_F = S.add<double>(Stage::kDown, 9);
    const auto win_mask = S.add<unsigned>(Stage::kDown, nw);
    const auto job = S.add<FmMaskJob>(Stage::kMapped, 1);
    const auto F = S.add<double>(Stage::kScratch, 27 * (size_t)budget);
    const auto masks = S.add<unsigned>(Stage::kScratch, 3 * (size_t)budget * nw);
    TRY(S.place(h));
    float *hp = reinterpret_cast<float *>(S.host(pq));
    int *hs = S.host(sched);
    std::memcpy(hp, p, sizeof(float) * 2 * n);
    std::memcpy(hp + 2 * n, q, sizeof(float) * 2 * n);
    int have = budget;                        // iterations that have a subset
    if (seven) {
        for (int i = 0; i < 7; ++i) hs[i] = i;
    } else if (schedule) {
        if (n_schedule < 1) return fail(h, PVIO_B200_EINVAL, "find_fundamental_mask: empty schedule");
        have = std::min(budget, n_schedule);
        for (int it = 0; it < have; ++it) {
            if (schedule[7 * it] < 0) { have = it; break; }          // a row starting with -1: getSubset gave up there
            for (int i = 0; i < 7; ++i) {
                const int v = schedule[7 * it + i];
                if (v < 0 || v >= n) return fail(h, PVIO_B200_EINVAL, "find_fundamental_mask: schedule index out of range");
                hs[7 * it + i] = v;
            }
        }
    } else {
        have = cv_schedule(p, q, n, budget, ransac ? 10000 : 1000, hs);
    }
    if (have == 0) {                          // getSubset failed at iteration 0: run() returns false, the mask stays as created
        std::memset(mask, 0, n);
        return finish(0);
    }
    // the problem as the batched tracker's kernel reads it: n matches, `have` iterations.  The kernel runs the LMedS
    // branch for n == 7 too (the call draws no schedule then); the replay of n == 7 reads counts[0] only, which both
    // branches write alike, and its mask is all ones.
    cudaStream_t st = h->stream;
    float2 *dp = S.dev(pq), *dq = dp + n;
    *S.host(prob) = FmBatchProblem{nullptr, nullptr, nullptr, dp, dq, S.dev(sched), S.dev(counts), S.dev(F), S.dev(masks),
                                   S.dev(surv), n, have};
    S.host(surv)[0] = n; S.host(surv)[1] = have;
    TRY(S.upload(h));
    fm_hypotheses_kernel<<<(have + kWarpsPerCta - 1) / kWarpsPerCta, 32 * kWarpsPerCta, 0, st>>>((float)(threshold * threshold), S.dev(prob));
    h->launches++;
    CK(h, cudaGetLastError());
    TRY(S.download(h, counts, counts));
    CK(h, cudaStreamSynchronize(st));

    const float thr_lmeds = fm_replay(S.host(counts), n, have, max_iters, confidence, inf);
    const int best_it = inf[1], best_k = inf[2];
    if (seven) std::memset(mask, 1, n);       // fundam.cpp: the mask of the 7-point / 8-point call is all ones
    if (best_it < 0) {
        if (!seven) std::memset(mask, 0, n);
        return finish(0);
    }
    const double *best_F = S.dev(F) + (size_t)(3 * best_it + best_k) * 9;
    if (!ransac && !seven) {
        *S.host(job) = FmMaskJob{dp, dq, best_F, nullptr, S.dev(masks), thr_lmeds, n};
        FmMaskJob *d_job = nullptr;           // read in place from the pinned staging (mapped: unified addressing)
        CK(h, cudaHostGetDevicePointer(reinterpret_cast<void **>(&d_job), S.host(job), 0));
        fm_mask_kernel<<<nw, 32, 0, st>>>(d_job);
        h->launches++;
        CK(h, cudaGetLastError());
    }
    CK(h, cudaMemcpyAsync(S.host(win_F), best_F, sizeof(double) * 9, cudaMemcpyDeviceToHost, st));
    if (!seven) {
        const unsigned *src = ransac ? S.dev(masks) + (size_t)(3 * best_it + best_k) * nw : S.dev(masks);
        CK(h, cudaMemcpyAsync(S.host(win_mask), src, sizeof(unsigned) * nw, cudaMemcpyDeviceToHost, st));
    }
    CK(h, cudaStreamSynchronize(st));
    if (!seven)
        for (int i = 0; i < n; ++i) mask[i] = (S.host(win_mask)[i >> 5] >> (i & 31)) & 1u;
    if (F_out) std::memcpy(F_out, S.host(win_F), 9 * sizeof(double));
    return finish(0);
}

// ---- the batched tracker's launches (klt.cu: batch_track_impl) -----------------------------------------------------
void fm_batch_schedule(Handle *h, const FmBatchProblem *probs, int n, int max_iters, int lmeds_iters) {
    fm_schedule_kernel<<<n, 32, 0, h->stream>>>(probs, max_iters, lmeds_iters);
    h->launches++;
}

// every iteration of every pair in one launch: blockIdx.y is the pair, warps beyond its schedule exit at once
void fm_batch_hypotheses(Handle *h, const FmBatchProblem *probs, int n, int max_budget, float thr2) {
    fm_hypotheses_kernel<<<dim3((max_budget + kWarpsPerCta - 1) / kWarpsPerCta, n), 32 * kWarpsPerCta, 0, h->stream>>>(thr2, probs);
    h->launches++;
}

// every winner's mask in one launch: one warp per mask word, blockIdx.y the pair
void fm_batch_masks(Handle *h, const FmMaskJob *jobs, int n, int max_words) {
    fm_mask_kernel<<<dim3((max_words + 3) / 4, n), 128, 0, h->stream>>>(jobs);
    h->launches++;
}

}  // namespace pvio
