// Multi-view DLT triangulation of new tracks: Track::triangulate (pvio/src/pvio/map/track.cpp:83-106) with
// triangulate_point / triangulate_point_scored (pvio/src/pvio/geometry/stereo.h:67-75, 104-128); the arithmetic of one
// track is tri_point_scored (tri.cuh).
#include "api_internal.h"
#include "tri.cuh"

namespace pvio {

struct TriArgs {
    int n_tracks;
    const double *P;          // [n_frames][12] row-major 3x4 camera matrices [R | T] (track.cpp:90-95)
    const int32_t *begin;     // [n_tracks + 1]
    const int32_t *frame;     // [total]
    const double *z;          // [total][2] normalised keypoints
    double *p_out;            // [n_tracks][3]
    double *score;            // [n_tracks]
    uint8_t *valid;           // [n_tracks]
};

// the views of the tracks: observation o of the CSR list
struct TriViews {
    const TriArgs &a;
    __device__ const double *P(int o) const { return a.P + (size_t)a.frame[o] * 12; }
    __device__ const double *z(int o) const { return a.z + 2 * o; }
};

__global__ void triangulate_kernel(TriArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_tracks) return;
    const int b0 = a.begin[t], b1 = a.begin[t + 1];
    double p[3], score;
    const bool ok = tri_point_scored(TriViews{a}, b0, b1, p, score);
    for (int k = 0; k < 3; ++k) a.p_out[3 * t + k] = p[k];
    a.score[t] = score;
    a.valid[t] = ok ? 1 : 0;
}

}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_triangulate(pvio_b200_handle hh, int n_frames, const double *P, int n_tracks, const int32_t *begin,
                                     const int32_t *obs_frame, const double *obs_z, double *points, uint8_t *valid, double *score) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    if (n_frames < 1 || n_tracks < 1 || !P || !begin || !obs_frame || !obs_z || !points || !valid || !score)
        return fail(h, PVIO_B200_EINVAL, "triangulate: bad argument");
    const int total = begin[n_tracks];
    for (int i = 0; i < n_tracks; ++i)
        if (begin[i + 1] - begin[i] < 2) return fail(h, PVIO_B200_EINVAL, "triangulate: a track needs at least two views (stereo.h:106)");
    for (int i = 0; i < total; ++i)
        if (obs_frame[i] < 0 || obs_frame[i] >= n_frames) return fail(h, PVIO_B200_EINVAL, "triangulate: frame index out of range");
    cudaSetDevice(h->device);
    const size_t szP = sizeof(double) * 12 * n_frames, szB = sizeof(int32_t) * (n_tracks + 1), szF = sizeof(int32_t) * total,
                 szZ = sizeof(double) * 2 * total, szO = sizeof(double) * 3 * n_tracks, szS = sizeof(double) * n_tracks, szV = n_tracks;
    auto al = [](size_t x) { return (x + 15) & ~(size_t)15; };
    const size_t oP = 0, oZ = oP + al(szP), oO = oZ + al(szZ), oS = oO + al(szO), oB = oS + al(szS), oF = oB + al(szB), oV = oF + al(szF);
    DevBuf<unsigned char> buf;
    TRY(alloc(h, buf, oV + al(szV), kDevice));
    unsigned char *d = buf.d;
    cudaStream_t st = h->stream;
    CK(h, cudaMemcpyAsync(d + oP, P, szP, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(d + oZ, obs_z, szZ, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(d + oB, begin, szB, cudaMemcpyHostToDevice, st));
    CK(h, cudaMemcpyAsync(d + oF, obs_frame, szF, cudaMemcpyHostToDevice, st));
    TriArgs a;
    a.n_tracks = n_tracks; a.P = reinterpret_cast<double *>(d + oP); a.z = reinterpret_cast<double *>(d + oZ);
    a.begin = reinterpret_cast<int32_t *>(d + oB); a.frame = reinterpret_cast<int32_t *>(d + oF);
    a.p_out = reinterpret_cast<double *>(d + oO); a.score = reinterpret_cast<double *>(d + oS); a.valid = d + oV;
    triangulate_kernel<<<(n_tracks + 127) / 128, 128, 0, st>>>(a);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(points, d + oO, szO, cudaMemcpyDeviceToHost, st));
    CK(h, cudaMemcpyAsync(score, d + oS, szS, cudaMemcpyDeviceToHost, st));
    CK(h, cudaMemcpyAsync(valid, d + oV, szV, cudaMemcpyDeviceToHost, st));
    CK(h, cudaStreamSynchronize(st));
    return PVIO_B200_OK;
}
