// Multi-view DLT triangulation of new tracks: Track::triangulate (pvio/src/pvio/map/track.cpp:83-106) with
// triangulate_point / triangulate_point_scored (pvio/src/pvio/geometry/stereo.h:67-75, 104-128).
// The reference takes the last right singular vector of the 2n x 4 matrix A (JacobiSVD); here one thread per
// track accumulates the 4 x 4 Gram matrix A^T A in fp64 and takes its eigenvector of smallest eigenvalue by
// cyclic Jacobi rotations -- the same vector up to sign (every use below is sign invariant); sigma_4^2 against
// sigma_1^2 costs half the digits, which leaves ~1e-10 of the direction in fp64 for pixel-level residuals.
#include "api_internal.h"

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

__device__ __forceinline__ void jacobi_eig4_smallest(double G[16], double q[4]) {
    double V[16] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1};
    for (int sweep = 0; sweep < 30; ++sweep) {
        double off = 0.0, dg = 0.0;
        for (int i = 0; i < 4; ++i) { dg += G[i * 5] * G[i * 5]; for (int j = i + 1; j < 4; ++j) off += G[i * 4 + j] * G[i * 4 + j]; }
        if (off <= 1e-60 * dg || off == 0.0) break;
        for (int p = 0; p < 3; ++p)
            for (int r = p + 1; r < 4; ++r) {
                const double apq = G[p * 4 + r];
                if (apq == 0.0) continue;
                const double th = (G[r * 5] - G[p * 5]) / (2.0 * apq);
                const double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
                for (int k = 0; k < 4; ++k) {                   // columns p, r of G
                    const double gp = G[k * 4 + p], gr = G[k * 4 + r];
                    G[k * 4 + p] = c * gp - s * gr; G[k * 4 + r] = s * gp + c * gr;
                }
                for (int k = 0; k < 4; ++k) {                   // rows p, r
                    const double gp = G[p * 4 + k], gr = G[r * 4 + k];
                    G[p * 4 + k] = c * gp - s * gr; G[r * 4 + k] = s * gp + c * gr;
                }
                for (int k = 0; k < 4; ++k) {
                    const double vp = V[k * 4 + p], vr = V[k * 4 + r];
                    V[k * 4 + p] = c * vp - s * vr; V[k * 4 + r] = s * vp + c * vr;
                }
            }
    }
    int m = 0;
    for (int i = 1; i < 4; ++i) if (G[i * 5] < G[m * 5]) m = i;
    for (int k = 0; k < 4; ++k) q[k] = V[k * 4 + m];
}

__global__ void triangulate_kernel(TriArgs a) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= a.n_tracks) return;
    const int b0 = a.begin[t], b1 = a.begin[t + 1];
    double G[16];
    for (int i = 0; i < 16; ++i) G[i] = 0.0;
    for (int o = b0; o < b1; ++o) {                               // stereo.h:69-72
        const double *P = a.P + (size_t)a.frame[o] * 12;
        const double zx = a.z[2 * o], zy = a.z[2 * o + 1];
        double r0[4], r1[4];
        for (int k = 0; k < 4; ++k) { r0[k] = zx * P[8 + k] - P[k]; r1[k] = zy * P[8 + k] - P[4 + k]; }
        for (int i = 0; i < 4; ++i)
            for (int j = 0; j < 4; ++j) G[i * 4 + j] += r0[i] * r0[j] + r1[i] * r1[j];
    }
    double q[4];
    jacobi_eig4_smallest(G, q);
    bool ok = true;                                               // stereo.h:104-128
    double score = 0.0;
    for (int o = b0; o < b1; ++o) {
        const double *P = a.P + (size_t)a.frame[o] * 12;
        double qi[3];
        for (int r = 0; r < 3; ++r) qi[r] = P[4 * r] * q[0] + P[4 * r + 1] * q[1] + P[4 * r + 2] * q[2] + P[4 * r + 3] * q[3];
        if (!(qi[2] * q[3] > 0)) ok = false;
        if (!(qi[2] / q[3] < 100)) ok = false;
        const double ex = qi[0] / qi[2] - a.z[2 * o], ey = qi[1] / qi[2] - a.z[2 * o + 1];
        score += ex * ex + ey * ey;
    }
    score /= (double)(b1 - b0);
    double s = ok ? q[3] : sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    for (int k = 0; k < 3; ++k) a.p_out[3 * t + k] = q[k] / s;
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
