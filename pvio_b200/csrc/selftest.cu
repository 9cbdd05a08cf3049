// Device self-tests: the Lie-group helpers (ba_math.cuh), so that the GPU tests sweep expmap / logmap / right_jacobian
// across the Taylor thresholds of geometry/lie_algebra.cpp:35-55 and angles near pi against the NumPy oracle
// (oracle/lie.py); and the reduced-system Cholesky solve (ba_chol.cuh), judged against an exact-residual reference
// (oracle/chol_oracle.py).  Not part of the reference interface.
#include <algorithm>
#include <cstring>
#include "api_internal.h"
#include "ba_chol.cuh"
#include "ba_math.cuh"

namespace pvio {

// in: w[n][3]; out[n][32]: expmap(w) (4), logmap(expmap(w)) (3), right_jacobian(w) (9), right_jacobian(w)^-1 (9),
// quat_plus((0,0,0,1) rotated by w, w) (4), 3 spare
__global__ void selftest_lie_kernel(int n, const double *w, double *out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const double v[3] = {w[3 * i], w[3 * i + 1], w[3 * i + 2]};
    double *o = out + (size_t)i * 32;
    double q[4], l[3], J[9], Ji[9], p[4];
    expmap(v, q);
    logmap(q, l);
    right_jacobian(v, J);
    mat3_inv(J, Ji);
    quat_plus(q, v, p);
    for (int k = 0; k < 4; ++k) o[k] = q[k];
    for (int k = 0; k < 3; ++k) o[4 + k] = l[k];
    for (int k = 0; k < 9; ++k) { o[7 + k] = J[k]; o[16 + k] = Ji[k]; }
    for (int k = 0; k < 4; ++k) o[25 + k] = p[k];
    o[29] = o[30] = o[31] = 0.0;
}

int selftest_lie_impl(Handle *h, int n, const double *w_in, double *out) {
    DevBuf<double> buf;
    TRY(alloc(h, buf, (size_t)n * 35, kDevice));
    double *d = buf.d;
    CK(h, cudaMemcpyAsync(d, w_in, sizeof(double) * 3 * n, cudaMemcpyHostToDevice, h->stream));
    selftest_lie_kernel<<<(n + 127) / 128, 128, 0, h->stream>>>(n, d, d + 3 * (size_t)n);
    ++h->launches;
    CK(h, cudaMemcpyAsync(out, d + 3 * (size_t)n, sizeof(double) * 32 * n, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// pvio_b200_selftest_chol: the factorisations of solve_kernel / solve_kernel_visual on caller-given systems, so that
// tests can judge them at fp64 level on their own (the GN step's parity tests see them only through the fp32 records).
// One CTA per system, of the production kernel's width and launch bounds.  System c (Ds[c] unknowns, row-major matrix and
// right-hand side at off[2c], off[2c + 1]) is packed as solve_body packs a reduced system: the lower 4 x 4 tiles of kTP
// doubles, padding rows up to Dp = 4 nb with an identity diagonal, the right-hand side in the solution vector.
enum CholMode { kCholNarrow = 0, kCholWide = 1, kCholWideTiled = 2 };

static size_t chol_selftest_smem(int D) {
    const size_t nb = (D + 3) / 4;
    return sizeof(double) * ((nb + 1) * (nb + 2) / 2 * kTP + 4 * nb);
}

template <int kMode>
static __device__ __forceinline__ void chol_selftest_body(const int32_t *Ds, const long long *off, const double *Ain,
                                                          const double *bin, double *xout, int32_t *okout) {
    const int c = blockIdx.x, D = Ds[c], nb = (D + 3) >> 2, Dp = nb * 4, tid = threadIdx.x, nt = blockDim.x;
    const double *Ac = Ain + off[2 * c], *bc = bin + off[2 * c + 1];
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int nA = (nb + 1) * (nb + 2) / 2 * kTP;
    double *A = reinterpret_cast<double *>(smem_raw), *x = A + nA;
    __shared__ int flag_sm;
    for (int i = tid; i < nA; i += nt) A[i] = 0.0;
    __syncthreads();
    for (int e = tid; e < Dp * Dp; e += nt) {
        const int i = e / Dp, j = e - i * Dp;
        if (j <= i) A[tri(i, j)] = i < D ? Ac[(size_t)i * D + j] : (i == j ? 1.0 : 0.0);
    }
    for (int i = tid; i < Dp; i += nt) x[i] = i < D ? bc[i] : 0.0;
    __syncthreads();
    const bool ok = kMode == kCholWideTiled ? chol_solve_tiled<true>(A, x, nb, &flag_sm)
                                            : chol_solve<kMode == kCholWide>(A, x, nb, &flag_sm);
    for (int i = tid; i < D; i += nt) xout[off[2 * c + 1] + i] = ok ? x[i] : 0.0;   // solve_body's dx of a failed solve
    if (tid == 0) okout[c] = ok ? 1 : 0;
}

static __global__ void __launch_bounds__(64, 10) selftest_chol_narrow_kernel(const int32_t *Ds, const long long *off,
                                                                             const double *A, const double *b, double *x,
                                                                             int32_t *ok) {
    chol_selftest_body<kCholNarrow>(Ds, off, A, b, x, ok);
}
static __global__ void __launch_bounds__(256) selftest_chol_wide_kernel(const int32_t *Ds, const long long *off,
                                                                        const double *A, const double *b, double *x,
                                                                        int32_t *ok) {
    chol_selftest_body<kCholWide>(Ds, off, A, b, x, ok);
}
static __global__ void __launch_bounds__(256) selftest_chol_wide_tiled_kernel(const int32_t *Ds, const long long *off,
                                                                              const double *A, const double *b, double *x,
                                                                              int32_t *ok) {
    chol_selftest_body<kCholWideTiled>(Ds, off, A, b, x, ok);
}

// the dynamic shared memory run_solve's kernels opt in to, once per process (see pvio_b200_create)
int selftest_chol_opt_in(Handle *h) {
    CK(h, cudaFuncSetAttribute(selftest_chol_narrow_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 48 * 1024));
    CK(h, cudaFuncSetAttribute(selftest_chol_wide_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    CK(h, cudaFuncSetAttribute(selftest_chol_wide_tiled_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    return 0;
}

int selftest_chol_impl(Handle *h, int n, int mode, const int32_t *Ds, const double *A, const double *b, double *x_out,
                       int32_t *ok_out) {
    if (n < 1) return fail(h, PVIO_B200_EINVAL, "selftest_chol: n < 1");
    if (mode < kCholNarrow || mode > kCholWideTiled) return fail(h, PVIO_B200_EINVAL, "selftest_chol: unknown mode");
    // the shared memory run_solve gives the kernel whose factorisation the mode runs
    const size_t cap = mode == kCholNarrow ? 48 * 1024 : 220 * 1024;
    size_t smax = 0, na = 0, nx = 0;
    for (int c = 0; c < n; ++c) {
        if (Ds[c] < 1) return fail(h, PVIO_B200_EINVAL, "selftest_chol: every D must be >= 1");
        if (chol_selftest_smem(Ds[c]) > cap)
            return fail(h, PVIO_B200_EINVAL, "selftest_chol: system too large for the mode's shared memory");
        if (mode == kCholWide && (Ds[c] + 3) / 4 > 64)
            return fail(h, PVIO_B200_EINVAL, "selftest_chol: more than 64 block rows for the register factorisation");
        smax = std::max(smax, chol_selftest_smem(Ds[c]));
        na += (size_t)Ds[c] * Ds[c];
        nx += Ds[c];
    }
    DevBuf<double> buf;                    // A, b, x back to back
    DevBuf<long long> off;                 // per system: offset of its matrix in A, of its vector in b and x
    DevBuf<int32_t> iv;                    // Ds, then ok
    TRY(alloc(h, buf, na + 2 * nx, kBoth));
    TRY(alloc(h, off, 2 * (size_t)n, kBoth));
    TRY(alloc(h, iv, 2 * (size_t)n, kBoth));
    memcpy(buf.h, A, sizeof(double) * na);
    memcpy(buf.h + na, b, sizeof(double) * nx);
    size_t oa = 0, ob = 0;
    for (int c = 0; c < n; ++c) {
        off.h[2 * c] = (long long)oa; off.h[2 * c + 1] = (long long)ob;
        oa += (size_t)Ds[c] * Ds[c]; ob += Ds[c];
    }
    memcpy(iv.h, Ds, sizeof(int32_t) * n);
    CK(h, cudaMemcpyAsync(buf.d, buf.h, sizeof(double) * (na + nx), cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(off.d, off.h, sizeof(long long) * 2 * n, cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(iv.d, iv.h, sizeof(int32_t) * n, cudaMemcpyHostToDevice, h->stream));
    const double *dA = buf.d, *db = buf.d + na;
    double *dx = buf.d + na + nx;
    if (mode == kCholNarrow) selftest_chol_narrow_kernel<<<n, 64, smax, h->stream>>>(iv.d, off.d, dA, db, dx, iv.d + n);
    else if (mode == kCholWide) selftest_chol_wide_kernel<<<n, 256, smax, h->stream>>>(iv.d, off.d, dA, db, dx, iv.d + n);
    else selftest_chol_wide_tiled_kernel<<<n, 256, smax, h->stream>>>(iv.d, off.d, dA, db, dx, iv.d + n);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(x_out, dx, sizeof(double) * nx, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(ok_out, iv.d + n, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // namespace pvio
