// Frame marginalisation: BundleAdjustor::marginalize_frame (estimation/bundle_adjustor.cpp:348-599).
//
//   prior J^T J                                   :369-413   marg_assemble_kernel
//   IMU factors adjacent to the victim            :416-450   marg_assemble_kernel
//   reprojection factors of victim-seen tracks    :453-533   lin_obs_kernel<false, double> (no loss, quirk Q3; ba_linearize.cuh)
//   landmark Schur (1/mat, isfinite skip)         :536-545   schur_kernel<double> (ba_schur.cuh)
//   frame Schur with the explicit 15x15 inverse   :547-581   marg_reduce_kernel
//   eigen factorisation, clamp lambda <= 1e-8     :583-590   marg_eig_kernel (Householder tridiagonalisation + implicit QL)
// All dense algebra is fp64.  Runs once per keyframe (not per iteration): latency, not bandwidth.
// Each of the three dense kernels runs one CTA per window: CTA c of a launch works on window w0 + c, with the dense
// scratch block c of the chunk (MargLayout).  A single window is a grid of 1.
#include <algorithm>
#include <cstring>
#include <vector>
#include "api_internal.h"
#include "ba_factors.cuh"

namespace pvio {

// Dense fp64 scratch of one window (offsets in doubles from the window's block, sized from the handle's frame capacity;
// ncap = 15 Ncap, dcap = ncap - 15) and the stride between the blocks of a chunk.
struct MargLayout {
    size_t H;                          // [ncap^2] information matrix, row-major with leading dimension 15 N, full symmetric
    size_t b;                          // [ncap]
    size_t Hk, bk;                     // [dcap^2], [dcap] after the frame Schur complement (leading dimension 15 (N - 1))
    size_t S, e;                       // [dcap^2], [dcap] the new prior, when it does not go to the window's prior arrays
    size_t scr;                        // >= 2048 + 64 Ncap doubles: IMU factor blocks, prior residual / Jacobian
    size_t stride;
};

struct MargArgs : BatchArrays {        // Hred, gred: set 0 of the vision part (xi coordinates) from the linearise + Schur stage
    int index;                         // victim frame
    int w0;                            // window of CTA 0
    double *buf;                       // chunk scratch: block c belongs to window w0 + c
    MargLayout L;
    const int32_t *slots;              // may be NULL: block c belongs to window slots[w0 + c] instead
};

__global__ void __launch_bounds__(256) marg_assemble_kernel(MargArgs a) {
    const int w = a.slots ? a.slots[a.w0 + blockIdx.x] : a.w0 + blockIdx.x;
    const WinHdr &Hh = a.hdr[w];
    const WinConst &wc = a.cst[w];
    const int N = Hh.N, n = 15 * N;
    const int tid = threadIdx.x, nt = blockDim.x;
    const size_t Nc = a.Ncap;
    const double *frames = a.frames + (size_t)w * Nc * kFrameStride;
    const WinFactors F(a, w);
    double *const blk = a.buf + blockIdx.x * a.L.stride;
    double *const Hm = blk + a.L.H, *const bv = blk + a.L.b, *const scratch = blk + a.L.scr;
    const double *Hred = a.Hred + (size_t)w * (Nc * (Nc + 1) / 2) * 36, *gred = a.gred + (size_t)w * Nc * 6;
    __shared__ double T[kMaxFrames * 36];
    for (int i = tid; i < n * n; i += nt) Hm[i] = 0.0;
    for (int i = tid; i < n; i += nt) bv[i] = 0.0;
    if (tid < N) frame_T(frames + tid * kFrameStride, wc, T + tid * 36);
    __syncthreads();
    // ---- vision: H_delta[f,g] = T_f^T X T_g  (reprojection + landmark Schur, :453-545)
    const int npairs = N * (N + 1) / 2;
    for (int e = tid; e < npairs * 36; e += nt) {
        const int p = e / 36, ij = e - p * 36, i = ij / 6, j = ij - i * 6;
        int f = 0;
        while ((f + 1) * (f + 2) / 2 <= p) ++f;
        const int gf = p - f * (f + 1) / 2;
        const double *X = Hred + p * 36;
        const double *Tf = T + f * 36, *Tg = T + gf * 36;
        double s = 0.0;
        for (int aa = 0; aa < 6; ++aa) {
            double t = 0.0;
            for (int bb = 0; bb < 6; ++bb) t += X[aa * 6 + bb] * Tg[bb * 6 + j];
            s += Tf[aa * 6 + i] * t;
        }
        const int gi = f * 15 + i, gj = gf * 15 + j;
        Hm[(size_t)gi * n + gj] = s;
        if (f != gf) Hm[(size_t)gj * n + gi] = s;
    }
    for (int e = tid; e < N * 6; e += nt) {
        const int f = e / 6, i = e - f * 6;
        double s = 0.0;
        for (int aa = 0; aa < 6; ++aa) s += T[f * 36 + aa * 6 + i] * gred[f * 6 + aa];
        bv[f * 15 + i] = s;
    }
    __syncthreads();
    // ---- prior :369-413  (H += E^T Lambda E, b += E^T S^T (S r0 + e))
    if (F.n_prior() > 0) {
        const int d = F.d();
        const int32_t *pfr = F.prior_frames();
        double *r0 = scratch, *rr = r0 + d, *vv = rr + d, *Ji = vv + d;
        if (tid < F.n_prior())
            prior_frame_raw(frames + pfr[tid] * kFrameStride, F.prior_x0() + tid * kFrameStride, r0 + 15 * tid, Ji + 9 * tid);
        __syncthreads();
        prior_residual(F.prior_S(), F.prior_e(), r0, d, [=](int i, double r) { rr[i] = r; });
        __syncthreads();
        for (int i = tid; i < d; i += nt) {
            double s = 0.0;
            for (int k = 0; k < d; ++k) s += F.prior_S()[(size_t)k * d + i] * rr[k];
            vv[i] = s;
        }
        __syncthreads();
        prior_grad(Ji, vv, d, pfr, [=](int gi, double s) { bv[gi] += s; });
        const double *L = F.prior_L();
        for (int e = tid; e < d * d; e += nt) {
            const int i = e / d, j = e - i * d;
            const int fi = i / 15, ci = i - fi * 15, fj = j / 15, cj = j - fj * 15;
            double s = 0.0;
            if (ci < 3 && cj < 3) {
                for (int k = 0; k < 3; ++k)
                    for (int m = 0; m < 3; ++m)
                        s += Ji[9 * fi + 3 * k + ci] * L[(size_t)(15 * fi + k) * d + 15 * fj + m] * Ji[9 * fj + 3 * m + cj];
            } else if (ci < 3) {
                for (int k = 0; k < 3; ++k) s += Ji[9 * fi + 3 * k + ci] * L[(size_t)(15 * fi + k) * d + j];
            } else if (cj < 3) {
                for (int m = 0; m < 3; ++m) s += L[(size_t)i * d + 15 * fj + m] * Ji[9 * fj + 3 * m + cj];
            } else {
                s = L[(size_t)i * d + j];
            }
            Hm[(size_t)(pfr[fi] * 15 + ci) * n + pfr[fj] * 15 + cj] += s;
        }
        __syncthreads();
    }
    // ---- IMU factors with j == index or j == index + 1  :416-450.  The functor reads the bias
    // linearisation point from the very memory passed as the parameter, so dbg = dba = 0.
    for (int m = 0; m < F.n_imu(); ++m) {
        const int fi = F.imu_idx()[2 * m], fj = F.imu_idx()[2 * m + 1];
        if (fj != a.index && fj != a.index + 1) continue;
        double *Jraw = scratch, *rraw = Jraw + 450, *Jw = rraw + 16, *rw = Jw + 450;
        const double *rec = F.imu_rec() + (size_t)m * kImuStride;
        if (tid == 0) imu_factor_raw(frames + fi * kFrameStride, frames + fj * kFrameStride, rec, wc, 1, rraw, Jraw);
        __syncthreads();
        for (int e = tid; e < 15 * 31; e += nt) {
            const int row = e / 31, col = e - row * 31;
            const double *Wm = rec + 11 + row * 15;
            double s = 0.0;
            if (col < 30) { for (int k = 0; k < 15; ++k) s += Wm[k] * Jraw[k * 30 + col]; Jw[row * 30 + col] = s; }
            else { for (int k = 0; k < 15; ++k) s += Wm[k] * rraw[k]; rw[row] = s; }
        }
        __syncthreads();
        for (int e = tid; e < 30 * 31; e += nt) {
            const int ra = e / 31, cb_ = e - ra * 31;
            const int ga = (ra < 15 ? fi * 15 + ra : fj * 15 + ra - 15);
            double s = 0.0;
            if (cb_ < 30) {
                const int gb = (cb_ < 15 ? fi * 15 + cb_ : fj * 15 + cb_ - 15);
                for (int k = 0; k < 15; ++k) s += Jw[k * 30 + ra] * Jw[k * 30 + cb_];
                Hm[(size_t)ga * n + gb] += s;
            } else {
                for (int k = 0; k < 15; ++k) s += Jw[k * 30 + ra] * rw[k];
                bv[ga] += s;
            }
        }
        __syncthreads();
    }
}

// Frame Schur complement :547-581.  inv = H[vv]^-1 by Gauss-Jordan with partial pivoting
// (Eigen's dynamic .inverse() is PartialPivLU based), then Hk = H[kk] - H[kv] inv H[vk].
__global__ void __launch_bounds__(256) marg_reduce_kernel(const WinHdr *hdr, int w0, int index, double *buf, MargLayout L,
                                                          const int32_t *slots) {
    double *const blk = buf + blockIdx.x * L.stride;
    const double *H = blk + L.H, *b = blk + L.b;
    double *Hk = blk + L.Hk, *bk = blk + L.bk;
    const int n = 15 * hdr[slots ? slots[w0 + blockIdx.x] : w0 + blockIdx.x].N, dk = n - 15, v0 = 15 * index;
    const int tid = threadIdx.x, nt = blockDim.x;
    __shared__ double M[15][31];
    __shared__ int piv_sm;
    for (int e = tid; e < 15 * 30; e += nt) {
        const int i = e / 30, j = e - i * 30;
        M[i][j] = (j < 15) ? H[(size_t)(v0 + i) * n + v0 + j] : ((j - 15 == i) ? 1.0 : 0.0);
    }
    __syncthreads();
    for (int c = 0; c < 15; ++c) {
        if (tid == 0) {
            int p = c;
            double best = fabs(M[c][c]);
            for (int i = c + 1; i < 15; ++i) if (fabs(M[i][c]) > best) { best = fabs(M[i][c]); p = i; }
            piv_sm = p;
        }
        __syncthreads();
        const int p = piv_sm;
        if (p != c && tid < 30) { const double t = M[c][tid]; M[c][tid] = M[p][tid]; M[p][tid] = t; }
        __syncthreads();
        const double ip = 1.0 / M[c][c];
        __syncthreads();
        if (tid < 30) M[c][tid] *= ip;
        __syncthreads();
        // eliminate column c from the other rows (compute, barrier, write: no read/write race)
        double newv[2] = {0.0, 0.0};
        int cnt = 0;
        for (int e = tid; e < 15 * 30; e += nt, ++cnt) {
            const int i = e / 30, jx = e - i * 30;
            newv[cnt] = (i != c) ? M[i][jx] - M[i][c] * M[c][jx] : M[i][jx];
        }
        __syncthreads();
        cnt = 0;
        for (int e = tid; e < 15 * 30; e += nt, ++cnt) M[e / 30][e % 30] = newv[cnt];
        __syncthreads();
    }
    // keep index list: all coordinates except the victim's 15
    // W = H[kv] * inv  (dk x 15) streamed through registers per thread
    for (int e = tid; e < dk * (dk + 1); e += nt) {
        const int i = e / (dk + 1), j = e - i * (dk + 1);
        const int gi = i < v0 ? i : i + 15;
        // row vector H[gi, v] * inv
        double acc = 0.0;
        if (j < dk) {
            const int gj = j < v0 ? j : j + 15;
            for (int k = 0; k < 15; ++k) {
                double wk = 0.0;
                for (int m = 0; m < 15; ++m) wk += H[(size_t)gi * n + v0 + m] * M[m][15 + k];
                acc += wk * H[(size_t)(v0 + k) * n + gj];
            }
            Hk[(size_t)i * dk + j] = H[(size_t)gi * n + gj] - acc;
        } else {
            for (int k = 0; k < 15; ++k) {
                double wk = 0.0;
                for (int m = 0; m < 15; ++m) wk += H[(size_t)gi * n + v0 + m] * M[m][15 + k];
                acc += wk * b[v0 + k];
            }
            bk[i] = b[gi] - acc;
        }
    }
}

// Symmetric eigen-decomposition for the factorisation :583-590 (Eigen::SelfAdjointEigenSolver in the reference): Householder
// tridiagonalisation + implicit QL with eigenvector accumulation (the EISPACK tred2 / tql2 pair), one CTA, the matrix
// in SHARED memory (odd leading dimension: conflict-free rows and columns).  Every O(n^2) inner loop is spread over the
// CTA; the scalar QL recurrence runs on one thread, which hands a batch of rotations to the CTA (thread k owns row k of
// the eigenvector matrix and applies the batch in order: no barrier inside a sweep).
// Then S = sqrt(max(lambda, 0 if <= 1e-8)) V^T and e = sqrt(1 / lambda) V^T b.
__device__ __forceinline__ double block_sum(double v, double *red, int tid, int nt) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((tid & 31) == 0) red[tid >> 5] = v;
    __syncthreads();
    double s = 0.0;
    for (int k = 0; k < (nt >> 5); ++k) s += red[k];
    return s;
}

#ifdef PVIO_MARG_STAMPS            // tuning builds of tools/ only: phase times of the eigen-solver
__device__ long long g_marg_stamps[8];
#define MARG_STAMP(k) do { __syncthreads(); if (threadIdx.x == 0) g_marg_stamps[k] = clock64(); } while (0)
#else
#define MARG_STAMP(k) do { } while (0)
#endif

// Per window (CTA c: window w0 + c): S [c * S_stride] dense n x n row-major, evec [c * e_stride]; x0 (may be NULL): the
// linearisation point of the new prior, frames 1 .. N - 1 of the window's state (frames, x0: window w0's, x_stride apart).
// slots (may be NULL): CTA c works on window w = slots[w0 + c] and its outputs are at [w * stride] instead.
__global__ void __launch_bounds__(256) marg_eig_kernel(const WinHdr *hdr, int w0, const double *buf, MargLayout L, int ring,
                                                       double *S_all, size_t S_stride, double *e_all, size_t e_stride,
                                                       const double *frames, double *x0, size_t x_stride,
                                                       const int32_t *slots) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int tid = threadIdx.x, nt = blockDim.x;
    const int c = blockIdx.x, w = slots ? slots[w0 + c] : w0 + c, N = hdr[w].N, n = 15 * (N - 1);
    const size_t o = slots ? (size_t)w : (size_t)c;
    const double *Ain = buf + c * L.stride + L.Hk, *bvec = buf + c * L.stride + L.bk;
    double *S = S_all + o * S_stride, *evec = e_all + o * e_stride;
    const int ld = n | 1;
    double *a = reinterpret_cast<double *>(smem_raw);       // [n][ld]: matrix -> eigenvectors (columns)
    double *d = a + (size_t)n * ld;                         // [n]
    double *e = d + n;                                      // [n]
    double *rot = e + n;                                    // [ring][2][n] rotation cosines / sines of the QL sweeps in flight
    __shared__ double red[8];
    __shared__ double sc_sm[4];
    __shared__ int ctl[2 + 2 * 4];                          // produced, consumed, index range of each ring slot
    for (int idx = tid; idx < n * n; idx += nt) a[(idx / n) * ld + idx % n] = Ain[idx];
    __syncthreads();
    MARG_STAMP(0);
    // ---- tred2
    for (int i = n - 1; i > 0; --i) {
        const int l = i - 1;
        double *ai = a + (size_t)i * ld;
        if (l > 0) {
            double sa = 0.0;
            for (int k = tid; k <= l; k += nt) sa += fabs(ai[k]);
            const double scale = block_sum(sa, red, tid, nt);
            if (scale == 0.0) {
                if (tid == 0) { e[i] = ai[l]; d[i] = 0.0; }
                __syncthreads();
                continue;
            }
            double sh = 0.0;
            for (int k = tid; k <= l; k += nt) { const double v = ai[k] / scale; ai[k] = v; sh += v * v; }
            double h = block_sum(sh, red, tid, nt);
            if (tid == 0) {
                const double f = ai[l], g = f >= 0 ? -sqrt(h) : sqrt(h);
                e[i] = scale * g;
                sc_sm[0] = h - f * g;
                ai[l] = f - g;
            }
            __syncthreads();
            h = sc_sm[0];
            double sf = 0.0;
            for (int j = tid; j <= l; j += nt) {             // e[j] = (A u)_j / h, u = row i
                a[(size_t)j * ld + i] = ai[j] / h;
                double g = 0.0;
                const double *aj = a + (size_t)j * ld;
                for (int k = 0; k <= j; ++k) g += aj[k] * ai[k];
                for (int k = j + 1; k <= l; ++k) g += a[(size_t)k * ld + j] * ai[k];
                e[j] = g / h;
                sf += e[j] * ai[j];
            }
            const double f = block_sum(sf, red, tid, nt);
            const double hh = f / (h + h);
            for (int j = tid; j <= l; j += nt) e[j] -= hh * ai[j];
            __syncthreads();
            const int tri = (l + 1) * (l + 2) / 2;          // rank-2 update of the lower triangle
            for (int idx = tid; idx < tri; idx += nt) {
                int j = (int)((sqrtf(8.0f * idx + 1.0f) - 1.0f) * 0.5f);
                while ((j + 1) * (j + 2) / 2 <= idx) ++j;
                while (j * (j + 1) / 2 > idx) --j;
                const int k = idx - j * (j + 1) / 2;
                a[(size_t)j * ld + k] -= ai[j] * e[k] + e[j] * ai[k];
            }
            if (tid == 0) d[i] = h;
        } else if (tid == 0) { e[i] = ai[l]; d[i] = 0.0; }
        __syncthreads();
    }
    if (tid == 0) { d[0] = 0.0; e[0] = 0.0; }
    __syncthreads();
    MARG_STAMP(1);
    for (int i = 0; i < n; ++i) {                            // accumulate the transformations
        const int l = i - 1;
        double *ai = a + (size_t)i * ld;
        if (d[i] != 0.0) {
            for (int j = tid; j <= l; j += nt) {
                double g = 0.0;
                for (int k = 0; k <= l; ++k) g += ai[k] * a[(size_t)k * ld + j];
                for (int k = 0; k <= l; ++k) a[(size_t)k * ld + j] -= g * a[(size_t)k * ld + i];
            }
        }
        __syncthreads();
        if (tid == 0) { d[i] = ai[i]; ai[i] = 1.0; }
        for (int j = tid; j <= l; j += nt) { a[(size_t)j * ld + i] = 0.0; ai[j] = 0.0; }
        __syncthreads();
    }
    MARG_STAMP(2);
    // ---- tql2, producer / consumer: the scalar recurrence of the implicit QL sweeps touches only d and e -- it does not
    // depend on the eigenvector matrix -- so ONE thread (lane 0 of warp 0) runs ahead through all sweeps, publishing each
    // sweep's rotations (cosines, sines, index range) in a ring of `ring` slots, while warps 1..7 apply the batches in
    // order, row k of the matrix per thread.  The sweep time was scalar chain + application + three CTA barriers
    // (13 K cycles per sweep, ~220 sweeps at n = 120); it is now the longer of the two.
    if (tid == 0) { for (int i = 1; i < n; ++i) e[i - 1] = e[i]; e[n - 1] = 0.0; }
    volatile int *vctl = ctl;                                // [0] batches produced, [1] batches consumed
    if (tid == 0) { vctl[0] = 0; vctl[1] = 0; }
    int *rng = ctl + 2;                                      // [ring][2] index range of each slot (i_hi, i_lo); i_hi = -2: the end
    __syncthreads();
    if (tid < 32) {
        if (tid == 0) {
            int prod = 0;
            for (int l = 0; l < n; ++l) {
                for (int iter = 0; iter < 64; ++iter) {
                    int m = l;
                    for (; m < n - 1; ++m) { const double dd = fabs(d[m]) + fabs(d[m + 1]); if (fabs(e[m]) <= 2.3e-16 * dd) break; }
                    if (m == l) break;
                    while (prod - vctl[1] >= ring) __nanosleep(40);       // every slot still in use
                    double *rc = rot + (size_t)(prod % ring) * 2 * n, *rs = rc + n;
                    // (sqrt(f^2 + g^2) instead of hypot, one reciprocal instead of two divisions: this scalar chain is the
                    // critical path of the kernel -- ~60 dependent rotations per sweep, ~200 sweeps; the magnitudes here
                    // (<= 1e15 from the gauge prior) are far from the range where hypot's rescaling matters)
                    double g = (d[l + 1] - d[l]) / (2.0 * e[l]), r = sqrt(g * g + 1.0);
                    g = d[m] - d[l] + e[l] / (g + (g >= 0 ? fabs(r) : -fabs(r)));
                    double s = 1.0, c = 1.0, p = 0.0;
                    int i = m - 1;
                    bool broke = false;
                    // e[i] and d[i] of the NEXT rotation are loaded ahead (they are untouched originals: off the dependent
                    // chain s, c, g, p), and d[i + 1] is the d[i] of the rotation before
                    double e_i = e[i], d_i = d[i], d_i1 = d[m];
                    for (; i >= l; --i) {
                        const double e_nx = i > l ? e[i - 1] : 0.0, d_nx = i > l ? d[i - 1] : 0.0;
                        const double f = s * e_i, b = c * e_i;
                        const double q2 = f * f + g * g;
                        if (q2 == 0.0) { e[i + 1] = 0.0; d[i + 1] -= p; e[m] = 0.0; broke = true; break; }
                        const double ir = rsqrt(q2);            // one reciprocal square root gives both r and 1 / r
                        e[i + 1] = r = q2 * ir;
                        s = f * ir; c = g * ir; g = d_i1 - p; r = (d_i - g) * s + 2.0 * c * b; p = s * r; d[i + 1] = g + p; g = c * r - b;
                        rc[i] = c; rs[i] = s;
                        d_i1 = d_i; e_i = e_nx; d_i = d_nx;
                    }
                    if (!broke) { d[l] -= p; e[l] = g; e[m] = 0.0; }
                    rng[2 * (prod % ring)] = m - 1;                      // rotations i = m - 1 .. i_lo, in this order
                    rng[2 * (prod % ring) + 1] = broke ? i + 1 : l;
                    __threadfence_block();
                    vctl[0] = ++prod;
                }
            }
            while (prod - vctl[1] >= ring) __nanosleep(40);
            rng[2 * (prod % ring)] = -2;
            __threadfence_block();
            vctl[0] = prod + 1;
        }
    } else {
        const int ct = tid - 32, nct = nt - 32;
        for (int k = 0;; ++k) {
            while (vctl[0] <= k) __nanosleep(20);
            __threadfence_block();
            const int i_hi = rng[2 * (k % ring)], i_lo = rng[2 * (k % ring) + 1];
            if (i_hi == -2) break;
            const double *rc = rot + (size_t)(k % ring) * 2 * n, *rs = rc + n;
            for (int row = ct; row < n; row += nct) {        // row `row` of the eigenvector matrix takes the whole batch
                double *zk = a + (size_t)row * ld;
                double zi1 = zk[i_hi + 1];
                for (int i = i_hi; i >= i_lo; --i) {
                    const double zi = zk[i], c = rc[i], s = rs[i];
                    zk[i + 1] = s * zi + c * zi1;
                    zi1 = c * zi - s * zi1;
                }
                zk[i_lo] = zi1;
            }
            asm volatile("bar.sync 1, %0;" ::"r"(nct) : "memory");       // the consumers are done with the slot
            if (ct == 0) { vctl[1] = k + 1; }
        }
    }
    __syncthreads();
    MARG_STAMP(3);
    // S = sqrt(lambda_clamped) V^T ; e = sqrt(1 / lambda) V^T b
    for (int i = tid; i < n; i += nt) {
        const double lam = d[i];
        const bool pos = lam > 1.0e-8;
        const double sl = pos ? sqrt(lam) : 0.0, il = pos ? sqrt(1.0 / lam) : 0.0;
        double dot = 0.0;
        for (int k = 0; k < n; ++k) {
            const double v = a[(size_t)k * ld + i];
            S[(size_t)i * n + k] = sl * v;
            dot += v * bvec[k];
        }
        evec[i] = il * dot;
    }
    if (x0)
        for (int i = tid; i < (N - 1) * kFrameStride; i += nt) x0[o * x_stride + i] = frames[o * x_stride + kFrameStride + i];
    MARG_STAMP(4);
}

#ifdef PVIO_MARG_STAMPS
extern "C" int pvio_b200_debug_marg_stamps(long long *out) {
    return cudaMemcpyFromSymbol(out, g_marg_stamps, sizeof(long long) * 8) == cudaSuccess ? 0 : -1;
}
#endif

// Windows per pass of the dense kernels.  Their scratch blocks (about 0.4 MB each at N = 9, Handle::marg) are allocated
// for the largest pass a handle has run and reused by every pass: the marginaliser runs at every keyframe, and nothing
// is allocated in the steady state.  Two per SM: at D = 135 the eigen-solver's shared memory admits one CTA
// per SM, so the second half of a pass queues behind the first; at N = 6 several CTAs share an SM.
constexpr int kMargChunkPerSm = 2;
constexpr size_t kEigSmemMax = 226 * 1024;

static MargLayout marg_layout(const Handle *h) {
    const size_t ncap = 15 * (size_t)h->Ncap, dcap = ncap - 15;
    MargLayout L;
    L.H = 0; L.b = L.H + ncap * ncap;
    L.Hk = L.b + ncap; L.bk = L.Hk + dcap * dcap;
    L.S = L.bk + dcap; L.e = L.S + dcap * dcap;
    L.scr = L.e + dcap;
    L.stride = L.scr + 2048 + 64 * (size_t)h->Ncap;
    return L;
}

// dynamic shared memory of the eigen-solver: matrix + d, e + the ring of rotation batches
static size_t eig_smem(int dk, int ring) { return sizeof(double) * ((size_t)dk * (dk | 1) + (2 + 2 * (size_t)ring) * dk); }
static bool eig_fits(int dk) { return eig_smem(dk, 2) <= kEigSmemMax; }      // 15 (N - 1) <= 165

// The launch shape of marg_eig_kernel for a grid whose largest matrix is dk_max: a ring of 4 rotation batches, or 2 when
// the matrix leaves no room for 4.  Every CTA of the launch gets the ring and the shared memory of the largest.  Every
// accepted size takes 4: at dk = 165 the 4-slot ring needs 231000 bytes of the 231424 opted in.
struct EigLaunch { int ring; size_t smem; };
static EigLaunch eig_launch(int dk_max) {
    const int ring = eig_smem(dk_max, 4) <= kEigSmemMax ? 4 : 2;
    return {ring, eig_smem(dk_max, ring)};
}

// once per handle, for the handle's device (pvio_b200_create): function attributes belong to the current device
int marg_opt_in(Handle *h) {
    CK(h, cudaFuncSetAttribute(marg_eig_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEigSmemMax));
    return 0;
}

// The marginaliser of n uploaded windows at their device states: the vision part of all n windows, then the dense tail
// chunk by chunk (assemble -> frame Schur complement -> eigen-solver; a window's three kernels stay in one chunk, so its
// old prior is consumed before its new one overwrites it).  eig = false stops after the Schur complement.
// The windows are [0, n), or the list h_slots / d_slots (host / device copies of one list; every kernel, the vision
// sweeps included, then works on the listed windows only).
// to_slots: S, e and the linearisation point (the CURRENT states of frames 1 .. N - 1) go straight into each window's own
// prior arrays, where a later pack of the shifted window names them with prior_S == NULL or a resident slot's next solve
// reads them; otherwise (n == 1, no list) into the scratch block of window 0.
int run_marg(Handle *h, int n, int index, bool eig, bool to_slots, const int32_t *h_slots, const int32_t *d_slots) {
    const int chunk = std::min(n, kMargChunkPerSm * h->sm_count);
    const MargLayout L = marg_layout(h);
    TRY(reserve(h, h->marg, L.stride * chunk, kDevice));
    // vision part: no loss, victim-seen landmarks only, mu = 0, fp64 (lin_obs_kernel<false, double> + schur_kernel<double>)
    TRY(run_marg_vision(h, n, h_slots, d_slots));
    double *buf = h->marg.d;
    MargArgs m = launch_args<MargArgs>(h);
    m.index = index; m.buf = buf; m.L = L; m.slots = d_slots;
    for (int w0 = 0; w0 < n; w0 += chunk) {
        const int cn = std::min(chunk, n - w0);
        m.w0 = w0;
        marg_assemble_kernel<<<cn, 256, 0, h->stream>>>(m);
        marg_reduce_kernel<<<cn, 256, 0, h->stream>>>(h->hdr.d, w0, index, buf, L, d_slots);
        h->launches += 2;
        if (!eig) continue;
        int dk = 0;
        for (int i = w0; i < w0 + cn; ++i) dk = std::max(dk, 15 * (h->hdr.h[h_slots ? h_slots[i] : i].N - 1));
        const EigLaunch el = eig_launch(dk);
        if (to_slots) {        // with a list the kernel offsets each output by its slot, without one CTA c writes w0 + c
            const int o = d_slots ? 0 : w0;
            marg_eig_kernel<<<cn, 256, el.smem, h->stream>>>(h->hdr.d, w0, buf, L, el.ring,
                h->prior_S.dslot(o), h->prior_S.per, h->prior_e.dslot(o), h->prior_e.per, h->frames.dslot(o),
                h->prior_x0.dslot(o), h->prior_x0.per, d_slots);
        } else {
            marg_eig_kernel<<<cn, 256, el.smem, h->stream>>>(h->hdr.d, w0, buf, L, el.ring,
                buf + L.S, L.stride, buf + L.e, L.stride, nullptr, nullptr, 0, nullptr);
        }
        ++h->launches;
    }
    CK(h, cudaGetLastError());
    return 0;
}

int marginalize_impl(Handle *h, const pvio_b200_window *w, const pvio_b200_state *s, int index,
                     double *S_out, double *e_out, double *H_out, double *b_out) {
    const int N = w->n_frames;
    if (index < 0 || index >= N || N < 2) return fail(h, PVIO_B200_EINVAL, "marginalize: bad frame index");
    if (!w->use_inertial) return fail(h, PVIO_B200_EINVAL, "marginalize: the window must carry motion states");
    const int dk = 15 * (N - 1);
    const bool eig = S_out || e_out;
    if (eig && !eig_fits(dk))
        return fail(h, PVIO_B200_EINVAL, "marginalize: window too large for the shared-memory eigen-solver (15 (N - 1) <= 165)");
    TRY(pack_and_upload(h, w, s));
    TRY(run_marg(h, 1, index, eig, false));
    const MargLayout L = marg_layout(h);
    const double *blk = h->marg.d;
    if (H_out) CK(h, cudaMemcpyAsync(H_out, blk + L.Hk, sizeof(double) * dk * dk, cudaMemcpyDeviceToHost, h->stream));
    if (b_out) CK(h, cudaMemcpyAsync(b_out, blk + L.bk, sizeof(double) * dk, cudaMemcpyDeviceToHost, h->stream));
    if (S_out) CK(h, cudaMemcpyAsync(S_out, blk + L.S, sizeof(double) * dk * dk, cudaMemcpyDeviceToHost, h->stream));
    if (e_out) CK(h, cudaMemcpyAsync(e_out, blk + L.e, sizeof(double) * dk, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaGetLastError());
    return 0;
}

bool marg_eig_fits(int dk) { return eig_fits(dk); }

// pvio_b200_batch_marginalize: every window is checked before anything is launched, so a rejected call changes nothing.
int batch_marginalize_impl(Handle *h, int n, double *S_out, int64_t S_stride, double *e_out, int64_t e_stride) {
    if (n < 1 || n > h->n_uploaded) return fail(h, PVIO_B200_EINVAL, "batch_marginalize: windows not uploaded");
    for (int i = 0; i < n; ++i) {
        const WinHdr &H = h->hdr.h[i];
        const int dk = 15 * (H.N - 1);
        if (!H.use_inertial) return fail(h, PVIO_B200_EINVAL, "batch_marginalize: every window must carry motion states");
        if (H.N < 2) return fail(h, PVIO_B200_EINVAL, "batch_marginalize: a window needs at least two frames");
        if (!eig_fits(dk))
            return fail(h, PVIO_B200_EINVAL, "batch_marginalize: window too large for the shared-memory eigen-solver (15 (N - 1) <= 165)");
        if ((S_out && S_stride < (int64_t)dk * dk) || (e_out && e_stride < dk))
            return fail(h, PVIO_B200_EINVAL, "batch_marginalize: output stride smaller than a window's prior");
    }
    TRY(run_marg(h, n, 0, true, true));
    for (int i = 0; i < n; ++i) {          // slot i's prior arrays hold the dense dk x dk S and e at their start
        const size_t dk = 15 * (size_t)(h->hdr.h[i].N - 1);
        if (S_out) CK(h, cudaMemcpyAsync(S_out + i * S_stride, h->prior_S.dslot(i), sizeof(double) * dk * dk,
                                         cudaMemcpyDeviceToHost, h->stream));
        if (e_out) CK(h, cudaMemcpyAsync(e_out + i * e_stride, h->prior_e.dslot(i), sizeof(double) * dk,
                                         cudaMemcpyDeviceToHost, h->stream));
    }
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaGetLastError());
    for (int i = 0; i < n; ++i) h->slots[i].prior_resident = h->hdr.h[i].N - 1;
    return 0;
}

// pvio_b200_selftest_eig: the unchanged marg_eig_kernel in one launch over n given symmetric matrices, so that tests can
// pin the eigen-solver against a reference on spectra no window produces.  Problem c is staged as block c of a
// MargLayout-shaped scratch (Hk, bk; the kernel reads nothing else) with a WinHdr of its own whose N = dk_c / 15 + 1 (the
// only field the kernel reads); the launch shape is the marginaliser's, eig_launch of the largest dk.  A, b, S_out and
// e_out hold the problems back to back: dk_c x dk_c row-major matrices, dk_c vectors.
int selftest_eig_impl(Handle *h, int n, const int32_t *dk, const double *A, const double *b, double *S_out, double *e_out) {
    if (n < 1) return fail(h, PVIO_B200_EINVAL, "selftest_eig: n < 1");
    int dmax = 0;
    for (int c = 0; c < n; ++c) {
        if (dk[c] < 15 || dk[c] % 15 != 0 || !eig_fits(dk[c]))
            return fail(h, PVIO_B200_EINVAL, "selftest_eig: every dk must be a multiple of 15 in [15, 165]");
        dmax = std::max(dmax, (int)dk[c]);
    }
    MargLayout L{};
    L.Hk = 0; L.bk = (size_t)dmax * dmax; L.stride = L.bk + dmax;
    DevBuf<double> buf;                    // n input blocks, then n output blocks (S at the block's start, e at its bk)
    DevBuf<WinHdr> hdr;
    TRY(alloc(h, buf, 2 * n * L.stride, kBoth));
    TRY(alloc(h, hdr, n, kBoth));
    size_t oa = 0, ob = 0;
    for (int c = 0; c < n; ++c) {
        const size_t d = dk[c];
        memcpy(buf.h + c * L.stride + L.Hk, A + oa, sizeof(double) * d * d);
        memcpy(buf.h + c * L.stride + L.bk, b + ob, sizeof(double) * d);
        hdr.h[c].N = dk[c] / 15 + 1;
        oa += d * d; ob += d;
    }
    double *out = buf.d + n * L.stride;
    CK(h, cudaMemcpyAsync(buf.d, buf.h, sizeof(double) * n * L.stride, cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(hdr.d, hdr.h, sizeof(WinHdr) * n, cudaMemcpyHostToDevice, h->stream));
    const EigLaunch el = eig_launch(dmax);
    marg_eig_kernel<<<n, 256, el.smem, h->stream>>>(hdr.d, 0, buf.d, L, el.ring, out, L.stride, out + L.bk, L.stride,
                                                   nullptr, nullptr, 0, nullptr);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(buf.h, out, sizeof(double) * n * L.stride, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    oa = ob = 0;
    for (int c = 0; c < n; ++c) {
        const size_t d = dk[c];
        memcpy(S_out + oa, buf.h + c * L.stride, sizeof(double) * d * d);
        memcpy(e_out + ob, buf.h + c * L.stride + L.bk, sizeof(double) * d);
        oa += d * d; ob += d;
    }
    return 0;
}

}  // namespace pvio
