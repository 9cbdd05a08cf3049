// Multi-view DLT triangulation of one track (stereo.h:67-75, 104-128), shared by pvio_b200_triangulate (tri.cu) and the
// triangulation of new tracks in pvio_b200_batch_window_localize (bw_frame.cu).
// The reference takes the last right singular vector of the 2n x 4 matrix A (JacobiSVD); here one thread per
// track accumulates the 4 x 4 Gram matrix A^T A in fp64 and takes its eigenvector of smallest eigenvalue by
// cyclic Jacobi rotations -- the same vector up to sign (every use below is sign invariant); sigma_4^2 against
// sigma_1^2 costs half the digits, which leaves ~1e-10 of the direction in fp64 for pixel-level residuals.
#pragma once

namespace pvio {

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

// triangulate_point_scored over views b0 .. b1 - 1: views.P(o) the row-major 3x4 camera matrix [R | T] of view o,
// views.z(o) its normalised keypoint [2].  p: q.hnormalized() when valid, otherwise the unit direction; returns
// has_parallax.
template <typename Views>
__device__ __forceinline__ bool tri_point_scored(const Views &views, int b0, int b1, double p[3], double &score_out) {
    double G[16];
    for (int i = 0; i < 16; ++i) G[i] = 0.0;
    for (int o = b0; o < b1; ++o) {                               // stereo.h:69-72
        const double *P = views.P(o);
        const double zx = views.z(o)[0], zy = views.z(o)[1];
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
        const double *P = views.P(o);
        double qi[3];
        for (int r = 0; r < 3; ++r) qi[r] = P[4 * r] * q[0] + P[4 * r + 1] * q[1] + P[4 * r + 2] * q[2] + P[4 * r + 3] * q[3];
        if (!(qi[2] * q[3] > 0)) ok = false;
        if (!(qi[2] / q[3] < 100)) ok = false;
        const double ex = qi[0] / qi[2] - views.z(o)[0], ey = qi[1] / qi[2] - views.z(o)[1];
        score += ex * ex + ey * ey;
    }
    score_out = score / (double)(b1 - b0);
    const double s = ok ? q[3] : sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]);
    for (int k = 0; k < 3; ++k) p[k] = q[k] / s;
    return ok;
}

}  // namespace pvio
