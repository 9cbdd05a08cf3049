// Device self-test of the Lie-group helpers (ba_math.cuh): lets the GPU tests sweep expmap / logmap /
// right_jacobian across the Taylor thresholds of geometry/lie_algebra.cpp:35-55 and angles near pi against the
// NumPy oracle (oracle/lie.py).  Not part of the reference interface.
#include "api_internal.h"
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

}  // namespace pvio
