// IMU pre-integration on the device: PreIntegrator::integrate / increment / compute_sqrt_inv_cov
// (pvio/src/pvio/estimation/preintegrator.cpp:39-102) for a batch of independent factors, one warp each (the warp body
// is imu.cuh's, which the resident slots' re-integration before a solve shares, batch_window.cu).  The reference
// re-integrates every IMU factor of the window at each solve (bundle_adjustor.cpp:226-231) and each new frame's factor
// before PnP (sliding_window_tracker.cpp:74-78); this kernel produces the same per-factor record the BA and PnP
// kernels consume (PVIO_B200_IMU_* layout).
#include "api_internal.h"
#include "imu.cuh"

namespace pvio {

struct ImuArgs {
    int n;
    const int32_t *begin;     // [n + 1] CSR into samples
    const double *samples;    // [total][7]: t, w xyz, a xyz
    const double *t_end;      // [n]
    const double *bias;       // [n][6]: bg, ba
    const double *noise;      // [4][9]: cov_w, cov_a, cov_bg, cov_ba (row major 3x3)
    double *rec;              // [n][kImuStride]
};

// factor f of a call (imu_integrate_warp's Factor)
struct ImuCallFactor {
    const ImuArgs &a;
    int f;
    const double *samples, *noise;
    __device__ int begin() const { return a.begin[f]; }
    __device__ int end() const { return a.begin[f + 1]; }
    __device__ double t_end() const { return a.t_end[f]; }
    __device__ double *rec() const { return a.rec + (size_t)f * kImuStride; }
};

__global__ void __launch_bounds__(128) preintegrate_kernel(ImuArgs a) {
    __shared__ ImuWarpSm sm[4];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int f = blockIdx.x * 4 + wv;
    if (f >= a.n) return;                                    // whole warps leave together
    const double *bias = a.bias + 6 * f;
    const double bg[3] = {bias[0], bias[1], bias[2]}, ba[3] = {bias[3], bias[4], bias[5]};
    imu_integrate_warp(sm[wv], lane, ImuCallFactor{a, f, a.samples, a.noise}, bg, ba);
}

}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_preintegrate(pvio_b200_handle hh, int n_factors, const int32_t *begin, const double *samples,
                                      const double *t_end, const double *bias, const double *noise_cov, double *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n_factors < 1 || !begin || !samples || !t_end || !bias || !noise_cov || !records)
        return fail(h, PVIO_B200_EINVAL, "preintegrate: bad argument");
    for (int i = 0; i < n_factors; ++i)
        if (begin[i + 1] <= begin[i])
            return fail(h, PVIO_B200_EINVAL, "preintegrate: a factor without IMU samples (integrate() returns false, preintegrator.cpp:86)");
    cudaSetDevice(h->device);
    const size_t total = (size_t)begin[n_factors];
    const size_t nd = total * 7 + (size_t)n_factors * 7 + 36 + (size_t)n_factors * kImuStride;
    DevBuf<double> d;
    DevBuf<int32_t> db;
    TRY(alloc(h, d, nd, kDevice));
    TRY(alloc(h, db, n_factors + 1, kDevice));
    ImuArgs a;
    a.n = n_factors; a.begin = db.d;
    double *ds = d.d, *dt = ds + total * 7, *dbias = dt + n_factors, *dn = dbias + (size_t)n_factors * 6, *dr = dn + 36;
    a.samples = ds; a.t_end = dt; a.bias = dbias; a.noise = dn; a.rec = dr;
    cudaStream_t st = h->stream;
    CK(h, cudaMemcpyAsync(db.d, begin, sizeof(int32_t) * (n_factors + 1), cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(ds, samples, sizeof(double) * total * 7, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(dt, t_end, sizeof(double) * n_factors, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(dbias, bias, sizeof(double) * n_factors * 6, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(dn, noise_cov, sizeof(double) * 36, cudaMemcpyHostToDevice, st));
    preintegrate_kernel<<<(n_factors + 3) / 4, 128, 0, st>>>(a);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(records, dr, sizeof(double) * (size_t)n_factors * kImuStride, cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    return PVIO_B200_OK;
}
