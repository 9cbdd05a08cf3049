// The two-view step of Initializer::init_sfm (pvio/src/pvio/core/initializer.cpp:102-161) for many sequences at once
// (pvio_b200_batch_two_view): the match-count and parallax gates, find_homography_matrix and find_essential_matrix
// (geometry/stereo.cpp:36-80: Ransac<> of utility/ransac.h over solve_homography_4pt / solve_essential_5pt), both
// decompositions (homography.cpp:22-91, essential.cpp:213-276, the SVD form), and the scored triangulation of the 8
// pose candidates (stereo.cpp:149-171).  All fp64.
//
// The RANSAC loops follow fmat.cu's pattern (DESIGN 4.7c): every iteration is evaluated speculatively, and the serial
// acceptance rule is replayed on the host over the counts.
//   device  tv_schedule_kernel: one thread per problem draws Ransac::solve's sample schedule -- a LotBox (random.h) of
//           n lots seeded with `seed`, refilled every iteration, the lots' permutation carried over -- for H (4 draws
//           per iteration) and for E (5), each from a fresh LotBox
//   device  tv_homography_kernel: one warp per (problem, iteration); lane 0 solves the normalised 4-point DLT (null
//           vector of the 8 x 9 system by a Householder QR of its transpose), the lanes count the matches whose
//           symmetric transfer error is within the threshold
//   device  tv_essential_kernel: one warp per (problem, iteration); the 4-dimensional null space of the 5 x 9 system,
//           the 10 x 20 constraint polynomials (one row per lane), the Gauss-Jordan elimination with the reference's
//           pivot order (columns over lanes), the 10 x 10 action matrix; lane 0 finds its real eigenpairs (Hessenberg
//           reduction, Francis double-shift QR, inverse iteration); up to 10 models, each counted by the lanes
//   host    the replay of Ransac::solve's loop over the counts, with the host's log and pow
//   device  tv_finish_kernel: one CTA per problem: the winners' masks, the parallax, both decompositions, the 8 x n
//           scored triangulations, the selection, the winner's points
//
// Model order: Ransac::solve keeps the first model of an iteration that beats the best count.  The reference orders an
// iteration's E models by Eigen's real-Schur eigenvalue order; here they are ordered by ascending eigenvalue.  The two
// differ only when two models of one iteration tie on the winning count.
//
// Compiled with -fmad=false: the host arithmetic of the reference is not contracted.
#include <cfloat>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "ransac.cuh"
#include "tri.cuh"

namespace pvio {
namespace {

// ---- small dense helpers --------------------------------------------------------------------------------------------
__device__ __forceinline__ void mul3(const double *A, const double *B, double *C) {   // row-major C = A B
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
}
__device__ __forceinline__ double det3(const double *m) {
    return m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
}
__device__ __forceinline__ double dot3(const double *a, const double *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// 3 x 3 inverse by cofactors: inv(i, j) = cof(j, i) / det, det along column 0
__device__ void inverse3(const double *m, double *r) {
    double c[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
            c[3 * i + j] = m[3 * i1 + j1] * m[3 * i2 + j2] - m[3 * i1 + j2] * m[3 * i2 + j1];
        }
    const double det = (c[0] * m[0] + c[3] * m[3]) + c[6] * m[6];
    const double inv = 1.0 / det;
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) r[3 * i + j] = c[3 * j + i] * inv;
}

// columns C .. 8 of Q for the Householder QR of the 9 x C matrix M (row-major [9][C]): the null space of M^T.
// out[k - C][r], r < 9.
template <int C>
__device__ void householder_null(double (*M)[C], double (*out)[9]) {
    double V[C][9], beta[C];
    for (int k = 0; k < C; ++k) {
        double nrm = 0;
        for (int r = k; r < 9; ++r) nrm += M[r][k] * M[r][k];
        nrm = sqrt(nrm);
        const double x0 = M[k][k], alpha = x0 >= 0 ? -nrm : nrm;
        double vv = 0;
        for (int r = k; r < 9; ++r) {
            const double v = r == k ? x0 - alpha : M[r][k];
            V[k][r] = v;
            vv += v * v;
        }
        beta[k] = vv > 0 ? 2. / vv : 0.;
        for (int c = k; c < C; ++c) {
            double s = 0;
            for (int r = k; r < 9; ++r) s += V[k][r] * M[r][c];
            s *= beta[k];
            for (int r = k; r < 9; ++r) M[r][c] -= s * V[k][r];
        }
    }
    for (int q = C; q < 9; ++q) {
        double *f = out[q - C];
        for (int r = 0; r < 9; ++r) f[r] = r == q;
        for (int k = C - 1; k >= 0; --k) {
            double s = 0;
            for (int r = k; r < 9; ++r) s += V[k][r] * f[r];
            s *= beta[k];
            for (int r = k; r < 9; ++r) f[r] -= s * V[k][r];
        }
    }
}

// ---- homography (homography.cpp:99-166) -----------------------------------------------------------------------------
// solve_homography_4pt on the matches idx[0..3]; H row-major, p2 ~ H p1
__device__ void homography_4pt(const double2 *p1, const double2 *p2, const int *idx, double *H) {
    double ax[4], ay[4], bx[4], by[4];
    double ma0 = 0, ma1 = 0, mb0 = 0, mb1 = 0;
    for (int i = 0; i < 4; ++i) {
        const double2 a = p1[idx[i]], b = p2[idx[i]];
        ax[i] = a.x; ay[i] = a.y; bx[i] = b.x; by[i] = b.y;
        ma0 += a.x; ma1 += a.y; mb0 += b.x; mb1 += b.y;
    }
    ma0 /= 4; ma1 /= 4; mb0 /= 4; mb1 /= 4;
    double sa = 0, sb = 0;
    for (int i = 0; i < 4; ++i) {
        const double dax = ax[i] - ma0, day = ay[i] - ma1, dbx = bx[i] - mb0, dby = by[i] - mb1;
        sa += sqrt(dax * dax + day * day);
        sb += sqrt(dbx * dbx + dby * dby);
    }
    const double sqrt2 = sqrt(2.0);
    sa = 1.0 / (sqrt2 * sa);
    sb = 1.0 / (sqrt2 * sb);
    // M = A^T (9 x 8), A the 8 x 9 system of the normalised matches in the unknowns h, H(k, j) = h[3 j + k]
    double M[9][8];
    for (int r = 0; r < 9; ++r)
        for (int c = 0; c < 8; ++c) M[r][c] = 0;
    for (int i = 0; i < 4; ++i) {
        const double a0 = (ax[i] - ma0) * sa, a1 = (ay[i] - ma1) * sa, b0 = (bx[i] - mb0) * sb, b1 = (by[i] - mb1) * sb;
        const int e = 2 * i, o = 2 * i + 1;
        M[1][e] = -a0; M[2][e] = a0 * b1; M[4][e] = -a1; M[5][e] = a1 * b1; M[7][e] = -1; M[8][e] = b1;
        M[0][o] = a0; M[2][o] = -a0 * b0; M[3][o] = a1; M[5][o] = -a1 * b0; M[6][o] = 1; M[8][o] = -b0;
    }
    double h[1][9];
    householder_null<8>(M, h);
    double NH[9];
    for (int k = 0; k < 3; ++k)
        for (int j = 0; j < 3; ++j) NH[3 * k + j] = h[0][3 * j + k];
    const double Nb[9] = {1 / sb, 0, mb0, 0, 1 / sb, mb1, 0, 0, 1};
    const double Na[9] = {sa, 0, -sa * ma0, 0, sa, -sa * ma1, 0, 0, 1};
    double T[9];
    mul3(Nb, NH, T);
    mul3(T, Na, H);
}

// homography_geometric_error: |p2 - hnormalized(H p1)|^2
__device__ __forceinline__ double h_error(const double *H, double x1, double y1, double x2, double y2) {
    const double u = (H[0] * x1 + H[1] * y1) + H[2], v = (H[3] * x1 + H[4] * y1) + H[5], w = (H[6] * x1 + H[7] * y1) + H[8];
    const double dx = x2 - u / w, dy = y2 - v / w;
    return dx * dx + dy * dy;
}

// essential_geometric_error: (p2^T E p1)^2 / |(E p1)_xy|^2
__device__ __forceinline__ double e_error(const double *E, double x1, double y1, double x2, double y2) {
    const double a = (E[0] * x1 + E[1] * y1) + E[2], b = (E[3] * x1 + E[4] * y1) + E[5], c = (E[6] * x1 + E[7] * y1) + E[8];
    const double r = (x2 * a + y2 * b) + c;
    return r * r / (a * a + b * b);
}

// ---- the 5-point solver (essential.cpp:114-288) ---------------------------------------------------------------------
// Polynomials in x, y, z of degree <= 3 over the graded reverse-lexicographic monomials
//   xxx xxy xyy yyy xxz xyz yyz xzz yzz zzz | xx xy yy xz yz zz | x y z | 1
// Products are truncated at degree 3; kPairs lists, for every product term, (output, left, right) in summation order.
struct PolyTable {
    int8_t ex[20][3];
    int n;
    int8_t pairs[200][3];
};
constexpr PolyTable make_poly_table() {
    PolyTable t{};
    const int8_t e[20][3] = {{3, 0, 0}, {2, 1, 0}, {1, 2, 0}, {0, 3, 0}, {2, 0, 1}, {1, 1, 1}, {0, 2, 1}, {1, 0, 2},
                             {0, 1, 2}, {0, 0, 3}, {2, 0, 0}, {1, 1, 0}, {0, 2, 0}, {1, 0, 1}, {0, 1, 1}, {0, 0, 2},
                             {1, 0, 0}, {0, 1, 0}, {0, 0, 1}, {0, 0, 0}};
    for (int i = 0; i < 20; ++i)
        for (int k = 0; k < 3; ++k) t.ex[i][k] = e[i][k];
    t.n = 0;
    for (int a = 0; a < 20; ++a)
        for (int b = 0; b < 20; ++b) {
            const int x = e[a][0] + e[b][0], y = e[a][1] + e[b][1], z = e[a][2] + e[b][2];
            if (x + y + z > 3) continue;
            for (int m = 0; m < 20; ++m)
                if (e[m][0] == x && e[m][1] == y && e[m][2] == z) {
                    t.pairs[t.n][0] = (int8_t)m; t.pairs[t.n][1] = (int8_t)a; t.pairs[t.n][2] = (int8_t)b;
                    ++t.n;
                }
        }
    return t;
}
__constant__ PolyTable kPoly = make_poly_table();
constexpr int kXX = 10, kX = 16, kY = 17, kZ = 18, kOne = 19;

__device__ __forceinline__ void poly_mul_add(const double *a, const double *b, double *r) {   // r += a b
    for (int t = 0; t < kPoly.n; ++t) r[kPoly.pairs[t][0]] += a[kPoly.pairs[t][1]] * b[kPoly.pairs[t][2]];
}

// Real eigenvalues (|imag| < 1e-10) of the 10 x 10 matrix A in ascending order and their eigenvectors' solutions
// (x, y, z) = (v_x, v_y, v_z) / v_1.  Hessenberg reduction by stabilised elimination, Francis double-shift QR for the
// eigenvalues, inverse iteration for the eigenvectors.  Returns the count (0 if the QR does not converge).
__device__ int real_eigen_solutions(const double (*A)[10], double (*xs)[3]) {
    constexpr int n = 10;
    double a[n][n];
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) a[i][j] = A[i][j];
    for (int m = 1; m < n - 1; ++m) {                  // Hessenberg form
        double x = 0;
        int piv = m;
        for (int j = m; j < n; ++j)
            if (fabs(a[j][m - 1]) > fabs(x)) { x = a[j][m - 1]; piv = j; }
        if (piv != m) {
            for (int j = m - 1; j < n; ++j) { const double t = a[piv][j]; a[piv][j] = a[m][j]; a[m][j] = t; }
            for (int j = 0; j < n; ++j) { const double t = a[j][piv]; a[j][piv] = a[j][m]; a[j][m] = t; }
        }
        if (x != 0) {
            for (int i = m + 1; i < n; ++i) {
                double y = a[i][m - 1];
                if (y != 0) {
                    y /= x;
                    a[i][m - 1] = y;
                    for (int j = m; j < n; ++j) a[i][j] -= y * a[m][j];
                    for (int j = 0; j < n; ++j) a[j][m] += y * a[j][i];
                }
            }
        }
    }
    for (int i = 2; i < n; ++i)
        for (int j = 0; j < i - 1; ++j) a[i][j] = 0;
    double wr[n], wi[n];
    double anorm = 0;
    for (int i = 0; i < n; ++i)
        for (int j = i > 0 ? i - 1 : 0; j < n; ++j) anorm += fabs(a[i][j]);
    int nn = n - 1;
    double t = 0;
    while (nn >= 0) {                                  // Francis double-shift QR
        int its = 0, l;
        do {
            for (l = nn; l >= 1; --l) {
                double s = fabs(a[l - 1][l - 1]) + fabs(a[l][l]);
                if (s == 0) s = anorm;
                if (fabs(a[l][l - 1]) + s == s) { a[l][l - 1] = 0; break; }
            }
            double x = a[nn][nn];
            if (l == nn) {
                wr[nn] = x + t; wi[nn] = 0; --nn;
            } else {
                double y = a[nn - 1][nn - 1], w = a[nn][nn - 1] * a[nn - 1][nn];
                if (l == nn - 1) {
                    const double p = 0.5 * (y - x), q = p * p + w;
                    double z = sqrt(fabs(q));
                    x += t;
                    if (q >= 0) {
                        z = p + (p >= 0 ? fabs(z) : -fabs(z));
                        wr[nn - 1] = wr[nn] = x + z;
                        if (z != 0) wr[nn] = x - w / z;
                        wi[nn - 1] = wi[nn] = 0;
                    } else {
                        wr[nn - 1] = wr[nn] = x + p;
                        wi[nn - 1] = -z; wi[nn] = z;
                    }
                    nn -= 2;
                } else {
                    if (its == 60) return 0;
                    if (its == 10 || its == 20 || its == 40) {   // exceptional shifts
                        t += x;
                        for (int i = 0; i <= nn; ++i) a[i][i] -= x;
                        const double s = fabs(a[nn][nn - 1]) + fabs(a[nn - 1][nn - 2]);
                        y = x = 0.75 * s;
                        w = -0.4375 * s * s;
                    }
                    ++its;
                    int m;
                    double p = 0, q = 0, r = 0, z;
                    for (m = nn - 2; m >= l; --m) {
                        z = a[m][m];
                        r = x - z;
                        double s = y - z;
                        p = (r * s - w) / a[m + 1][m] + a[m][m + 1];
                        q = a[m + 1][m + 1] - z - r - s;
                        r = a[m + 2][m + 1];
                        s = fabs(p) + fabs(q) + fabs(r);
                        p /= s; q /= s; r /= s;
                        if (m == l) break;
                        const double u = fabs(a[m][m - 1]) * (fabs(q) + fabs(r));
                        const double v = fabs(p) * (fabs(a[m - 1][m - 1]) + fabs(z) + fabs(a[m + 1][m + 1]));
                        if (u + v == v) break;
                    }
                    for (int i = m + 2; i <= nn; ++i) {
                        a[i][i - 2] = 0;
                        if (i != m + 2) a[i][i - 3] = 0;
                    }
                    for (int k = m; k <= nn - 1; ++k) {
                        if (k != m) {
                            p = a[k][k - 1];
                            q = a[k + 1][k - 1];
                            r = k != nn - 1 ? a[k + 2][k - 1] : 0;
                            x = fabs(p) + fabs(q) + fabs(r);
                            if (x != 0) { p /= x; q /= x; r /= x; }
                        }
                        const double sn = sqrt(p * p + q * q + r * r), s = p >= 0 ? sn : -sn;
                        if (s != 0) {
                            if (k == m) {
                                if (l != m) a[k][k - 1] = -a[k][k - 1];
                            } else {
                                a[k][k - 1] = -s * x;
                            }
                            p += s;
                            x = p / s; y = q / s; z = r / s; q /= p; r /= p;
                            for (int j = k; j <= nn; ++j) {
                                p = a[k][j] + q * a[k + 1][j];
                                if (k != nn - 1) { p += r * a[k + 2][j]; a[k + 2][j] -= p * z; }
                                a[k + 1][j] -= p * y;
                                a[k][j] -= p * x;
                            }
                            const int mmin = nn < k + 3 ? nn : k + 3;
                            for (int i = l; i <= mmin; ++i) {
                                p = x * a[i][k] + y * a[i][k + 1];
                                if (k != nn - 1) { p += z * a[i][k + 2]; a[i][k + 2] -= p * r; }
                                a[i][k + 1] -= p * q;
                                a[i][k] -= p;
                            }
                        }
                    }
                }
            }
        } while (l < nn - 1);
    }
    double lam[n];
    int nr = 0;
    for (int i = 0; i < n; ++i) {
        if (!(fabs(wi[i]) < 1.0e-10)) continue;
        int j = nr++;                                  // insertion in ascending order
        for (; j > 0 && lam[j - 1] > wr[i]; --j) lam[j] = lam[j - 1];
        lam[j] = wr[i];
    }
    double scale = 0;
    for (int i = 0; i < n; ++i)
        for (int j = 0; j < n; ++j) scale = fmax(scale, fabs(A[i][j]));
    const double tiny = DBL_EPSILON * (scale > 0 ? scale : 1.0);
    for (int e = 0; e < nr; ++e) {                     // inverse iteration on A - lambda I
        double L[n][n];
        int perm[n];
        for (int i = 0; i < n; ++i) {
            perm[i] = i;
            for (int j = 0; j < n; ++j) L[i][j] = A[i][j] - (i == j ? lam[e] : 0.0);
        }
        for (int k = 0; k < n; ++k) {
            int piv = k;
            for (int i = k + 1; i < n; ++i)
                if (fabs(L[i][k]) > fabs(L[piv][k])) piv = i;
            if (piv != k) {
                for (int j = 0; j < n; ++j) { const double tt = L[k][j]; L[k][j] = L[piv][j]; L[piv][j] = tt; }
                const int tp = perm[k]; perm[k] = perm[piv]; perm[piv] = tp;
            }
            if (fabs(L[k][k]) < tiny) L[k][k] = L[k][k] < 0 ? -tiny : tiny;
            for (int i = k + 1; i < n; ++i) {
                const double f = L[i][k] / L[k][k];
                L[i][k] = f;
                for (int j = k + 1; j < n; ++j) L[i][j] -= f * L[k][j];
            }
        }
        double v[n];
        for (int i = 0; i < n; ++i) v[i] = 1.0;
        for (int pass = 0; pass < 2; ++pass) {
            double b[n];
            for (int i = 0; i < n; ++i) b[i] = v[perm[i]];
            for (int i = 0; i < n; ++i)
                for (int j = 0; j < i; ++j) b[i] -= L[i][j] * b[j];
            for (int i = n - 1; i >= 0; --i) {
                for (int j = i + 1; j < n; ++j) b[i] -= L[i][j] * b[j];
                b[i] /= L[i][i];
            }
            double mx = 0;
            for (int i = 0; i < n; ++i) mx = fmax(mx, fabs(b[i]));
            for (int i = 0; i < n; ++i) v[i] = b[i] / mx;
        }
        const double w = v[kOne - kXX];
        xs[e][0] = v[kX - kXX] / w; xs[e][1] = v[kY - kXX] / w; xs[e][2] = v[kZ - kXX] / w;
    }
    return nr;
}

// ---- the one-sided Jacobi SVD of a 3 x 3 matrix ---------------------------------------------------------------------
// M = U diag(s) V^T, s descending.  U's columns are M's orthogonalised columns over their norms; with rank2 the third is
// u0 x u1 instead (the left null vector of an essential matrix, whose third column is noise).
__device__ void svd3(const double *M, bool rank2, double *s, double *U, double *V) {
    double a[3][3], v[3][3];                           // a[c][r]: column c
    for (int c = 0; c < 3; ++c)
        for (int r = 0; r < 3; ++r) { a[c][r] = M[3 * r + c]; v[c][r] = r == c; }
    for (int sweep = 0; sweep < 40; ++sweep) {
        bool rotated = false;
        for (int pq = 0; pq < 3; ++pq) {
            const int p = pq == 2 ? 1 : 0, q = pq == 0 ? 1 : 2;
            const double alpha = dot3(a[p], a[p]), beta = dot3(a[q], a[q]), gamma = dot3(a[p], a[q]);
            if (fabs(gamma) <= 1e-15 * sqrt(alpha * beta)) continue;
            rotated = true;
            const double zeta = (beta - alpha) / (2 * gamma);
            const double t = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1 + zeta * zeta));
            const double c = 1 / sqrt(1 + t * t), sn = c * t;
            for (int r = 0; r < 3; ++r) {
                const double ap = a[p][r], aq = a[q][r];
                a[p][r] = c * ap - sn * aq; a[q][r] = sn * ap + c * aq;
                const double vp = v[p][r], vq = v[q][r];
                v[p][r] = c * vp - sn * vq; v[q][r] = sn * vp + c * vq;
            }
        }
        if (!rotated) break;
    }
    double sig[3];
    for (int c = 0; c < 3; ++c) sig[c] = sqrt(dot3(a[c], a[c]));
    int o[3] = {0, 1, 2};
    for (int i = 1; i < 3; ++i)
        for (int j = i; j > 0 && sig[o[j]] > sig[o[j - 1]]; --j) { const int t = o[j]; o[j] = o[j - 1]; o[j - 1] = t; }
    double u[3][3];
    for (int i = 0; i < 3; ++i) {
        s[i] = sig[o[i]];
        for (int r = 0; r < 3; ++r) u[i][r] = a[o[i]][r] / sig[o[i]];
    }
    if (rank2) {
        u[2][0] = u[0][1] * u[1][2] - u[0][2] * u[1][1];
        u[2][1] = u[0][2] * u[1][0] - u[0][0] * u[1][2];
        u[2][2] = u[0][0] * u[1][1] - u[0][1] * u[1][0];
    }
    for (int r = 0; r < 3; ++r)
        for (int i = 0; i < 3; ++i) { U[3 * r + i] = u[i][r]; V[3 * r + i] = v[o[i]][r]; }
}

__device__ __forceinline__ void normalize3(double *t) {            // Eigen's normalized(): a zero vector stays zero
    const double q = dot3(t, t);
    if (q > 0) { const double nn = sqrt(q); for (int k = 0; k < 3; ++k) t[k] /= nn; }
}

// decompose_homography (homography.cpp:22-91), the Malis-Vargas branches in the reference's order.  Returns false for a
// pure rotation (R1 = R2 from the SVD, T = 0).
__device__ bool decompose_homography(const double *H, double *R1, double *R2, double *T1, double *T2) {
    double s[3], U[9], V[9];
    svd3(H, false, s, U, V);
    double Hn[9], S[9];
    for (int k = 0; k < 9; ++k) Hn[k] = H[k] / s[1];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j)
            S[3 * i + j] = ((Hn[i] * Hn[j] + Hn[3 + i] * Hn[3 + j]) + Hn[6 + i] * Hn[6 + j]) - (i == j ? 1.0 : 0.0);
    bool rot = true;
    for (int k = 0; k < 9; ++k)
        if (fabs(S[k]) > 1e-3) rot = false;
    if (rot) {
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) R1[3 * i + j] = (U[3 * i] * V[3 * j] + U[3 * i + 1] * V[3 * j + 1]) + U[3 * i + 2] * V[3 * j + 2];
        if (det3(R1) < 0)
            for (int k = 0; k < 9; ++k) R1[k] = -R1[k];
        for (int k = 0; k < 9; ++k) R2[k] = R1[k];
        for (int k = 0; k < 3; ++k) T1[k] = T2[k] = 0;
        return false;
    }
    const double s00 = S[0], s01 = S[1], s02 = S[2], s11 = S[4], s12 = S[5], s22 = S[8];
    const double ms00 = s12 * s12 - s11 * s22, ms11 = s02 * s02 - s00 * s22, ms22 = s01 * s01 - s00 * s11;
    const double rs00 = sqrt(ms00), rs11 = sqrt(ms11), rs22 = sqrt(ms22);
    const double tr = (s00 + s11) + s22;
    const double nu = 2.0 * sqrt(1 + tr - ms00 - ms11 - ms22);
    const double tenormsq = 2 + tr - nu;
    double n1[3], n2[3], t1[3], t2[3];
    if (s00 > s11 && s00 > s22) {
        const double e = (s01 * s02 - s00 * s12) < 0 ? -1 : 1;
        n1[0] = s00; n1[1] = s01 + rs22; n1[2] = s02 + e * rs11;
        n2[0] = s00; n2[1] = s01 - rs22; n2[2] = s02 - e * rs11;
        const double l1 = sqrt(dot3(n1, n1)), l2 = sqrt(dot3(n2, n2));
        for (int k = 0; k < 3; ++k) { t1[k] = l1 * n2[k] / s00; t2[k] = l2 * n1[k] / s00; }
    } else if (s11 > s00 && s11 > s22) {
        const double e = (s11 * s02 - s01 * s12) < 0 ? -1 : 1;
        n1[0] = s01 + rs22; n1[1] = s11; n1[2] = s12 - e * rs00;
        n2[0] = s01 - rs22; n2[1] = s11; n2[2] = s12 + e * rs00;
        const double l1 = sqrt(dot3(n1, n1)), l2 = sqrt(dot3(n2, n2));
        for (int k = 0; k < 3; ++k) { t2[k] = l2 * n1[k] / s11; t1[k] = l1 * n2[k] / s11; }
    } else {
        const double e = (s12 * s02 - s01 * s22) < 0 ? -1 : 1;
        n1[0] = s02 + e * rs11; n1[1] = s12 + rs00; n1[2] = s22;
        n2[0] = s02 - e * rs11; n2[1] = s12 - rs00; n2[2] = s22;
        const double l1 = sqrt(dot3(n1, n1)), l2 = sqrt(dot3(n2, n2));
        for (int k = 0; k < 3; ++k) { t1[k] = l1 * n2[k] / s22; t2[k] = l2 * n1[k] / s22; }
    }
    normalize3(n1);
    normalize3(n2);
    for (int k = 0; k < 3; ++k) { t1[k] -= tenormsq * n1[k]; t2[k] -= tenormsq * n2[k]; }
    double M1[9], M2[9];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) {
            M1[3 * i + j] = (i == j ? 1.0 : 0.0) - (t1[i] / nu) * n1[j];
            M2[3 * i + j] = (i == j ? 1.0 : 0.0) - (t2[i] / nu) * n2[j];
        }
    mul3(Hn, M1, R1);
    mul3(Hn, M2, R2);
    for (int k = 0; k < 3; ++k) { t1[k] *= 0.5; t2[k] *= 0.5; }
    for (int i = 0; i < 3; ++i) { T1[i] = dot3(R1 + 3 * i, t1); T2[i] = dot3(R2 + 3 * i, t2); }
    return true;
}

// decompose_essential, the SVD form (essential.cpp:259-274), with a fixed sign of T and order of R1, R2
__device__ void decompose_essential(const double *E, double *R1, double *R2, double *T) {
    double s[3], U[9], V[9], VT[9];
    svd3(E, true, s, U, V);
    if (det3(U) < 0)
        for (int k = 0; k < 9; ++k) U[k] = -U[k];
    for (int i = 0; i < 3; ++i)
        for (int j = 0; j < 3; ++j) VT[3 * i + j] = V[3 * j + i];
    if (det3(VT) < 0)
        for (int k = 0; k < 9; ++k) VT[k] = -VT[k];
    const double W[9] = {0, 1, 0, -1, 0, 0, 0, 0, 1}, Wt[9] = {0, -1, 0, 1, 0, 0, 0, 0, 1};
    double UW[9];
    mul3(U, W, UW);
    mul3(UW, VT, R1);
    mul3(U, Wt, UW);
    mul3(UW, VT, R2);
    for (int k = 0; k < 3; ++k) T[k] = U[3 * k + 2];
    // An essential matrix has two equal singular values, so the SVD's order of u0 and u1 is decided by rounding, and
    // with it the sign of T and the order of R1 and R2.  Both are fixed here: T's component of largest magnitude is
    // positive, and R1 is the rotation of larger trace (the smaller angle).
    int m = 0;
    for (int k = 1; k < 3; ++k)
        if (fabs(T[k]) > fabs(T[m])) m = k;
    if (T[m] < 0)
        for (int k = 0; k < 3; ++k) T[k] = -T[k];
    if ((R2[0] + R2[4]) + R2[8] > (R1[0] + R1[4]) + R1[8])
        for (int k = 0; k < 9; ++k) { const double t = R1[k]; R1[k] = R2[k]; R2[k] = t; }
}

// ---- the batched call -----------------------------------------------------------------------------------------------
// one problem as the kernels read it; h_it / e_it / e_k are the replay's winners (-1: none), set before the finish
struct TvProb {
    const double2 *p1, *p2;
    int n, seed, iters, off;                  // matches, seed, iterations evaluated (0 below 5 matches), match offset
    int min_matches, min_tri, h_it, e_it, e_k, pad;
    double fx, fy, min_parallax, thr_h, thr_e;
};
// one problem's results as the finish kernel writes them
struct TvOut {
    int status, candidate, triangulated, pad;
    double parallax, H[9], E[9], R[9], T[3];
};
// the device arrays of one call; problem k's iteration rows start at k * I, its matches at off (8 * off for sc, ok)
struct TvScratch {
    int I;                                    // iteration rows per problem
    int *lots, *sched_h, *sched_e, *cnt_h, *cnt_e;   // [total], [P][I][4], [P][I][5], [P][I], [P][I][11]
    double *Hm, *Em;                          // [P][I][9], [P][I][10][9]
    double *par, *sc;                         // [total], [8 total]
    uint8_t *ok;                              // [8 total]
    uint8_t *hmask, *emask, *pstat;           // [total] results
    double *pts;                              // [total][3] results
    TvOut *out;                               // [P]
};

__global__ void tv_schedule_kernel(const TvProb *probs, int n_probs, TvScratch s) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n_probs) return;
    const TvProb &P = probs[k];
    if (P.iters == 0) return;
    lotbox_schedule(P.n, P.seed, 4, P.iters, s.lots + P.off, s.sched_h + (size_t)k * s.I * 4);
    lotbox_schedule(P.n, P.seed, 5, P.iters, s.lots + P.off, s.sched_e + (size_t)k * s.I * 5);
}

constexpr int kTvWarps = 4;

__global__ void __launch_bounds__(32 * kTvWarps) tv_homography_kernel(const TvProb *probs, TvScratch s) {
    __shared__ double sH[kTvWarps][18];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int it = blockIdx.x * kTvWarps + warp, k = blockIdx.y;
    const TvProb &P = probs[k];
    if (it >= P.iters) return;
    const size_t row = (size_t)k * s.I + it;
    if (lane == 0) {
        double H[9];
        homography_4pt(P.p1, P.p2, s.sched_h + 4 * row, H);
        for (int i = 0; i < 9; ++i) { sH[warp][i] = H[i]; s.Hm[9 * row + i] = H[i]; }
        inverse3(H, sH[warp] + 9);
    }
    __syncwarp();
    double H[18];
    for (int i = 0; i < 18; ++i) H[i] = sH[warp][i];
    int good = 0;
    for (int base = 0; base < P.n; base += 32) {
        const int i = base + lane;
        bool in = false;
        if (i < P.n) {
            const double2 a = P.p1[i], b = P.p2[i];
            in = h_error(H, a.x, a.y, b.x, b.y) + h_error(H + 9, b.x, b.y, a.x, a.y) <= P.thr_h;
        }
        good += __popc(__ballot_sync(0xffffffffu, in));
    }
    if (lane == 0) s.cnt_h[row] = good;
}

// shared working set of one warp of tv_essential_kernel: 4.3 KB (17.5 KB per CTA of kTvWarps warps)
struct EssWarp {
    double basis[4][9];                       // null-space basis, basis[c][r]
    double eet[9][20];                        // E E^T, then the 10 x 20 system (rows 0 .. 9 in poly[])
    double poly[10][20];
    double act[10][10];
    double xs[10][3];
    int nm;
};

__global__ void __launch_bounds__(32 * kTvWarps) tv_essential_kernel(const TvProb *probs, TvScratch s) {
    __shared__ EssWarp sw[kTvWarps];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int it = blockIdx.x * kTvWarps + warp, k = blockIdx.y;
    const TvProb &P = probs[k];
    if (it >= P.iters) return;
    EssWarp &W = sw[warp];
    const size_t row = (size_t)k * s.I + it;
    if (lane == 0) {                          // A^T (9 x 5): A(i, 3 j + m) = p1h[j] p2h[m]
        const int *idx = s.sched_e + 5 * row;
        double M[9][5];
        for (int i = 0; i < 5; ++i) {
            const double2 a = P.p1[idx[i]], b = P.p2[idx[i]];
            const double ah[3] = {a.x, a.y, 1.0}, bh[3] = {b.x, b.y, 1.0};
            for (int j = 0; j < 3; ++j)
                for (int m = 0; m < 3; ++m) M[3 * j + m][i] = ah[j] * bh[m];
        }
        householder_null<5>(M, W.basis);
    }
    __syncwarp();
    // Epoly(i, j) = x Ex + y Ey + z Ez + Ew, E*(i, j) = basis[*][3 j + i]
    auto epoly = [&](int i, int j, double *p) {
        for (int m = 0; m < 20; ++m) p[m] = 0;
        p[kX] = W.basis[0][3 * j + i]; p[kY] = W.basis[1][3 * j + i]; p[kZ] = W.basis[2][3 * j + i]; p[kOne] = W.basis[3][3 * j + i];
    };
    if (lane < 9) {                           // (E E^T)(i, j)
        const int i = lane / 3, j = lane % 3;
        double r[20], a[20], b[20];
        for (int m = 0; m < 20; ++m) r[m] = 0;
        for (int c = 0; c < 3; ++c) { epoly(i, c, a); epoly(j, c, b); poly_mul_add(a, b, r); }
        for (int m = 0; m < 20; ++m) W.eet[lane][m] = r[m];
    }
    __syncwarp();
    if (lane < 9) {                           // (E E^T E - trace(E E^T) / 2 E)(i, j)
        const int i = lane / 3, j = lane % 3;
        double r[20], b[20], e[20], ht[20], q[20];
        for (int m = 0; m < 20; ++m) { r[m] = q[m] = 0; ht[m] = 0.5 * ((W.eet[0][m] + W.eet[4][m]) + W.eet[8][m]); }
        for (int c = 0; c < 3; ++c) { epoly(c, j, b); poly_mul_add(W.eet[3 * i + c], b, r); }
        epoly(i, j, e);
        poly_mul_add(ht, e, q);
        for (int m = 0; m < 20; ++m) W.poly[lane][m] = r[m] - q[m];
    } else if (lane == 9) {                   // det E along row 0
        double m11[20], m12[20], m21[20], m22[20], a[20], b[20], e[20], r[20];
        for (int m = 0; m < 20; ++m) r[m] = 0;
        for (int c = 0; c < 3; ++c) {
            const int c1 = (c + 1) % 3, c2 = (c + 2) % 3;
            epoly(1, c1, m11); epoly(2, c2, m22); epoly(1, c2, m12); epoly(2, c1, m21);
            for (int m = 0; m < 20; ++m) a[m] = b[m] = 0;
            poly_mul_add(m11, m22, a);
            poly_mul_add(m12, m21, b);
            for (int m = 0; m < 20; ++m) a[m] -= b[m];
            epoly(0, c, e);
            poly_mul_add(e, a, r);
        }
        for (int m = 0; m < 20; ++m) W.poly[9][m] = r[m];
    }
    __syncwarp();
    // Gauss-Jordan with the reference's row order (essential.cpp:155-176), columns over lanes 0 .. 19
    int perm[10];
    for (int i = 0; i < 10; ++i) perm[i] = i;
    for (int i = 0; i < 10; ++i) {
        for (int j = i + 1; j < 10; ++j)
            if (fabs(W.poly[perm[i]][i]) < fabs(W.poly[perm[j]][i])) { const int t = perm[i]; perm[i] = perm[j]; perm[j] = t; }
        const double piv = W.poly[perm[i]][i];
        if (piv == 0) continue;
        double f[10];
        __syncwarp();
        if (lane < 20) W.poly[perm[i]][lane] /= piv;
        __syncwarp();
        for (int j = i + 1; j < 10; ++j) f[j] = W.poly[perm[j]][i];
        __syncwarp();
        if (lane < 20)
            for (int j = i + 1; j < 10; ++j) W.poly[perm[j]][lane] -= W.poly[perm[i]][lane] * f[j];
        __syncwarp();
    }
    for (int i = 9; i > 0; --i) {
        double f[10];
        for (int j = 0; j < i; ++j) f[j] = W.poly[perm[j]][i];
        __syncwarp();
        if (lane < 20)
            for (int j = 0; j < i; ++j) W.poly[perm[j]][lane] -= W.poly[perm[i]][lane] * f[j];
        __syncwarp();
    }
    // the action matrix of multiplication by x on the basis xx xy yy xz yz zz x y z 1
    if (lane < 10) {
        const int src[6] = {0, 1, 2, 4, 5, 7};          // xxx xxy xyy xxz xyz xzz
        const int unit[4] = {0, 1, 3, 6};               // xx xy xz x
        for (int c = 0; c < 10; ++c)
            W.act[lane][c] = lane < 6 ? -W.poly[perm[src[lane]]][kXX + c] : (c == unit[lane - 6] ? 1.0 : 0.0);
    }
    __syncwarp();
    if (lane == 0) W.nm = real_eigen_solutions(W.act, W.xs);
    __syncwarp();
    const int nm = W.nm;
    int *cnt = s.cnt_e + 11 * row;
    if (lane == 0) cnt[0] = nm;
    for (int m = 0; m < 10; ++m) {
        if (m >= nm) {
            if (lane == 0) cnt[1 + m] = 0;
            continue;
        }
        double E[9], Et[9];
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) {
                const int r = 3 * j + i;
                E[3 * i + j] = ((W.basis[0][r] * W.xs[m][0] + W.basis[1][r] * W.xs[m][1]) + W.basis[2][r] * W.xs[m][2]) + W.basis[3][r];
            }
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) Et[3 * i + j] = E[3 * j + i];
        if (lane < 9) s.Em[(row * 10 + m) * 9 + lane] = E[lane];
        int good = 0;
        for (int base = 0; base < P.n; base += 32) {
            const int i = base + lane;
            bool in = false;
            if (i < P.n) {
                const double2 a = P.p1[i], b = P.p2[i];
                in = e_error(E, a.x, a.y, b.x, b.y) + e_error(Et, b.x, b.y, a.x, a.y) <= P.thr_e;
            }
            good += __popc(__ballot_sync(0xffffffffu, in));
        }
        if (lane == 0) cnt[1 + m] = good;
    }
}

// the views of one match under candidate (R, T): P1 = [I | 0], P2 = [R | T]
__constant__ double kP1[12] = {1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0};
struct TwoViews {
    const double *P2;
    double z1[2], z2[2];
    __device__ const double *P(int o) const { return o ? P2 : kP1; }
    __device__ const double *z(int o) const { return o ? z2 : z1; }
};

constexpr int kFinishThreads = 256;

__global__ void __launch_bounds__(kFinishThreads) tv_finish_kernel(const TvProb *probs, TvScratch s) {
    __shared__ double sH[18], sE[18], sP2[8][12], sScore[8];
    __shared__ int sCnt[8], sRot, sBest;
    const int k = blockIdx.x, tid = threadIdx.x;
    if (tid == 0) sRot = 0;
    const TvProb &P = probs[k];
    const int n = P.n, off = P.off;
    TvOut &O = s.out[k];
    for (int i = tid; i < n; i += kFinishThreads) {        // apply_k(p1) - apply_k(p2)
        const double2 a = P.p1[i], b = P.p2[i];
        const double dx = a.x * P.fx - b.x * P.fx, dy = a.y * P.fy - b.y * P.fy;
        s.par[off + i] = sqrt(dx * dx + dy * dy);
    }
    if (tid == 0) {
        const size_t base = (size_t)k * s.I;
        for (int i = 0; i < 9; ++i) {
            sH[i] = P.h_it >= 0 ? s.Hm[(base + P.h_it) * 9 + i] : 0.0;
            sE[i] = P.e_it >= 0 ? s.Em[((base + P.e_it) * 10 + P.e_k) * 9 + i] : 0.0;
        }
        inverse3(sH, sH + 9);
        for (int i = 0; i < 3; ++i)
            for (int j = 0; j < 3; ++j) sE[9 + 3 * i + j] = sE[3 * j + i];
        for (int i = 0; i < 9; ++i) { O.H[i] = sH[i]; O.E[i] = sE[i]; }
        if (n >= 5) {
            double RH1[9], RH2[9], TH1[3], TH2[3], RE1[9], RE2[9], TE[3];
            sRot = decompose_homography(sH, RH1, RH2, TH1, TH2) ? 0 : 1;
            normalize3(TH1);
            normalize3(TH2);
            decompose_essential(sE, RE1, RE2, TE);
            normalize3(TE);
            const double *Rs[8] = {RH1, RH1, RH2, RH2, RE1, RE1, RE2, RE2};
            const double *Ts[8] = {TH1, TH1, TH2, TH2, TE, TE, TE, TE};
            for (int c = 0; c < 8; ++c) {
                const double sg = (c & 1) ? -1.0 : 1.0;
                for (int r = 0; r < 3; ++r) {
                    for (int j = 0; j < 3; ++j) sP2[c][4 * r + j] = Rs[c][3 * r + j];
                    sP2[c][4 * r + 3] = sg * Ts[c][r];
                }
            }
        }
    }
    __syncthreads();
    if (n >= 5) {
        for (int i = tid; i < n; i += kFinishThreads) {
            const double2 a = P.p1[i], b = P.p2[i];
            s.hmask[off + i] = P.h_it >= 0 && h_error(sH, a.x, a.y, b.x, b.y) + h_error(sH + 9, b.x, b.y, a.x, a.y) <= P.thr_h;
            s.emask[off + i] = P.e_it >= 0 && e_error(sE, a.x, a.y, b.x, b.y) + e_error(sE + 9, b.x, b.y, a.x, a.y) <= P.thr_e;
        }
        for (int t = tid; t < 8 * n; t += kFinishThreads) {   // triangulate_from_rt_scored of every candidate
            const int c = t / n, i = t - c * n;
            const double2 a = P.p1[i], b = P.p2[i];
            double p[3], score;
            const bool ok = tri_point_scored(TwoViews{sP2[c], {a.x, a.y}, {b.x, b.y}}, 0, 2, p, score);
            s.sc[8 * (size_t)off + t] = score;
            s.ok[8 * (size_t)off + t] = ok;
        }
    } else {
        for (int i = tid; i < n; i += kFinishThreads) s.hmask[off + i] = s.emask[off + i] = 0;
    }
    __syncthreads();
    if (n >= 5 && tid < 8) {                   // count and mean score of candidate tid, summed in match order
        int cnt = 0;
        double sum = 0;
        for (int i = 0; i < n; ++i)
            if (s.ok[8 * (size_t)off + tid * n + i]) { sum += s.sc[8 * (size_t)off + tid * n + i]; ++cnt; }
        sCnt[tid] = cnt;
        sScore[tid] = sum / (double)(cnt > 1 ? cnt : 1);
    }
    __syncthreads();
    if (tid == 0) {
        double par = 0;
        for (int i = 0; i < n; ++i) par += s.par[off + i];
        par /= (n > 1 ? n : 1);
        int best = -1, status;
        if (n >= 5) {                          // stereo.cpp:155-163: the selection, count_threshold = min_triangulation
            best = 0;
            for (int c = 0; c < 8; ++c) {
                if (sCnt[c] > P.min_tri && sScore[c] < sScore[best]) best = c;
                else if (sCnt[c] > sCnt[best]) best = c;
            }
        }
        if (n < P.min_matches || n < 5) status = PVIO_B200_TWO_VIEW_FEW_MATCHES;
        else if (par < P.min_parallax) status = PVIO_B200_TWO_VIEW_LOW_PARALLAX;
        else if (sRot) status = PVIO_B200_TWO_VIEW_PURE_ROTATION;
        else if (sCnt[best] < P.min_tri) status = PVIO_B200_TWO_VIEW_FEW_TRIANGULATED;
        else status = PVIO_B200_TWO_VIEW_OK;
        O.status = status;
        O.parallax = par;
        O.candidate = best;
        O.triangulated = best >= 0 ? sCnt[best] : 0;
        for (int r = 0; r < 3; ++r) {
            for (int j = 0; j < 3; ++j) O.R[3 * r + j] = best >= 0 ? sP2[best][4 * r + j] : (r == j);
            O.T[r] = best >= 0 ? sP2[best][4 * r + 3] : 0.0;
        }
        sBest = best;
    }
    __syncthreads();
    const int best = sBest;
    for (int i = tid; i < n; i += kFinishThreads) {         // the winner's points (0 where it failed)
        double p[3] = {0, 0, 0};
        bool ok = false;
        if (best >= 0) {
            const double2 a = P.p1[i], b = P.p2[i];
            double score;
            ok = tri_point_scored(TwoViews{sP2[best], {a.x, a.y}, {b.x, b.y}}, 0, 2, p, score);
        }
        for (int c = 0; c < 3; ++c) s.pts[3 * (size_t)(off + i) + c] = ok ? p[c] : 0.0;
        s.pstat[off + i] = ok;
    }
}

// problems are the grid's y dimension in the hypothesis kernels; match offsets are int
constexpr int kMaxTwoViewProblems = 65535;

int tv_check(Handle *h, int n, const pvio_b200_two_view *recs) {
    if (n < 0 || (n > 0 && !recs)) return fail(h, PVIO_B200_EINVAL, "batch_two_view: bad record list");
    if (n > kMaxTwoViewProblems) return fail(h, PVIO_B200_EINVAL, "batch_two_view: more than 65535 problems");
    int64_t total = 0;
    for (int k = 0; k < n; ++k) {
        const pvio_b200_two_view &r = recs[k];
        if (r.n_matches < 0 || r.n_matches > (1 << 24)) return fail(h, PVIO_B200_EINVAL, "batch_two_view: n_matches out of range");
        if (r.n_matches > 0 && (!r.p1 || !r.p2)) return fail(h, PVIO_B200_EINVAL, "batch_two_view: NULL keypoints");
        if (!(r.fx > 0) || !(r.fy > 0)) return fail(h, PVIO_B200_EINVAL, "batch_two_view: fx and fy must be positive");
        if (!(r.confidence > 0) || r.max_iteration < 1) return fail(h, PVIO_B200_EINVAL, "batch_two_view: confidence and max_iteration must be positive");
        if (r.min_matches < 0 || r.min_triangulation < 0) return fail(h, PVIO_B200_EINVAL, "batch_two_view: negative minimum");
        total += r.n_matches;
    }
    if (total > INT32_MAX) return fail(h, PVIO_B200_EINVAL, "batch_two_view: more than 2^31 - 1 matches in one call");
    return 0;
}

}  // namespace

int batch_two_view_impl(Handle *h, int n, const pvio_b200_two_view *recs) {
    TRY(tv_check(h, n, recs));
    if (n == 0) return 0;
    cudaSetDevice(h->device);
    std::vector<int> off(n + 1, 0);
    int I = 1;
    bool want_sched = false;
    for (int k = 0; k < n; ++k) {
        off[k + 1] = off[k] + recs[k].n_matches;
        if (recs[k].n_matches >= 5) I = std::max(I, recs[k].max_iteration);
        want_sched |= recs[k].h_schedule || recs[k].e_schedule;
    }
    const size_t total = (size_t)off[n], tot1 = std::max<size_t>(total, 1), rows = (size_t)n * I;
    // staging: problems | p1 | p2 (uploaded) | schedules H, E | counts H, E | outputs | masks and point status | points
    // (downloaded); device scratch: lots | H models | E models | parallax | scores | score flags
    Stage S(h->tv.stage, &h->tv.scratch);
    const auto prob = S.add<TvProb>(Stage::kUp, n);
    const auto p1 = S.add<double>(Stage::kUp, 2 * tot1), p2 = S.add<double>(Stage::kUp, 2 * tot1);
    const auto sh = S.add<int>(Stage::kDown, 4 * rows), se = S.add<int>(Stage::kDown, 5 * rows);
    const auto ch = S.add<int>(Stage::kDown, rows), ce = S.add<int>(Stage::kDown, 11 * rows);
    const auto out = S.add<TvOut>(Stage::kDown, n);
    const auto mask = S.add<uint8_t>(Stage::kDown, 3 * tot1);
    const auto pts = S.add<double>(Stage::kDown, 3 * tot1);
    const auto lots = S.add<int>(Stage::kScratch, tot1);
    const auto hm = S.add<double>(Stage::kScratch, 9 * rows), em = S.add<double>(Stage::kScratch, 90 * rows);
    const auto par = S.add<double>(Stage::kScratch, tot1), sco = S.add<double>(Stage::kScratch, 8 * tot1);
    const auto ok = S.add<uint8_t>(Stage::kScratch, 8 * tot1);
    TRY(S.place(h));

    TvProb *hp = S.host(prob), *dp = S.dev(prob);
    double *h1 = S.host(p1), *h2 = S.host(p2);
    const double2 *d1 = reinterpret_cast<const double2 *>(S.dev(p1)), *d2 = reinterpret_cast<const double2 *>(S.dev(p2));
    for (int k = 0; k < n; ++k) {
        const pvio_b200_two_view &r = recs[k];
        const double thr = 0.7 / r.fx;
        TvProb &P = hp[k];
        P = TvProb{};
        P.p1 = d1 + off[k]; P.p2 = d2 + off[k];
        P.n = r.n_matches; P.seed = r.seed; P.iters = r.n_matches >= 5 ? r.max_iteration : 0; P.off = off[k];
        P.min_matches = r.min_matches; P.min_tri = r.min_triangulation;
        P.h_it = P.e_it = P.e_k = -1;
        P.fx = r.fx; P.fy = r.fy; P.min_parallax = r.min_parallax;
        P.thr_h = 2.0 * 5.99 * thr * thr;     // stereo.cpp:75-76 and :52-53
        P.thr_e = 2.0 * 3.84 * thr * thr;
        if (r.n_matches > 0) {
            std::memcpy(h1 + 2 * off[k], r.p1, sizeof(double) * 2 * r.n_matches);
            std::memcpy(h2 + 2 * off[k], r.p2, sizeof(double) * 2 * r.n_matches);
        }
    }
    TvScratch sc{};
    sc.I = I;
    sc.lots = S.dev(lots);
    sc.sched_h = S.dev(sh); sc.sched_e = S.dev(se); sc.cnt_h = S.dev(ch); sc.cnt_e = S.dev(ce);
    sc.Hm = S.dev(hm); sc.Em = S.dev(em);
    sc.par = S.dev(par); sc.sc = S.dev(sco); sc.ok = S.dev(ok);
    sc.out = S.dev(out);
    sc.hmask = S.dev(mask); sc.emask = S.dev(mask) + tot1; sc.pstat = S.dev(mask) + 2 * tot1;
    sc.pts = S.dev(pts);

    cudaStream_t st = h->stream;
    TRY(S.upload(h));
    tv_schedule_kernel<<<(n + 63) / 64, 64, 0, st>>>(dp, n, sc);
    const dim3 grid((I + kTvWarps - 1) / kTvWarps, n);
    tv_homography_kernel<<<grid, 32 * kTvWarps, 0, st>>>(dp, sc);
    tv_essential_kernel<<<grid, 32 * kTvWarps, 0, st>>>(dp, sc);
    h->launches += 3;
    CK(h, cudaGetLastError());
    TRY(S.download(h, want_sched ? sh : ch, ce));
    CK(h, cudaStreamSynchronize(st));

    std::vector<int> res(8 * n);
    for (int k = 0; k < n; ++k) {
        TvProb &P = hp[k];
        int *rk = &res[8 * k];
        rk[0] = rk[1] = rk[4] = rk[5] = 0; rk[2] = rk[3] = rk[6] = rk[7] = -1;
        if (P.iters == 0) continue;
        ransac_replay(S.host(ch) + (size_t)k * I, 1, true, P.n, P.iters, recs[k].confidence, rk);
        ransac_replay(S.host(ce) + (size_t)k * I * 11, 11, false, P.n, P.iters, recs[k].confidence, rk + 4);
        P.h_it = rk[2]; P.e_it = rk[6]; P.e_k = rk[7];
    }
    TRY(S.upload(h, prob));
    tv_finish_kernel<<<n, kFinishThreads, 0, st>>>(dp, sc);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h, out, pts));
    CK(h, cudaStreamSynchronize(st));

    const TvOut *ho = S.host(out);
    const uint8_t *hmk = S.host(mask);
    const double *hpts = S.host(pts);
    for (int k = 0; k < n; ++k) {
        const pvio_b200_two_view &r = recs[k];
        const TvOut &O = ho[k];
        const int *rk = &res[8 * k];
        const int nk = r.n_matches, o = off[k], Ik = hp[k].iters;
        if (r.info) {
            const int32_t info[10] = {O.status, rk[0], rk[1], rk[2], rk[4], rk[5], rk[6], rk[7], O.candidate, O.triangulated};
            std::memcpy(r.info, info, sizeof(info));
        }
        if (r.parallax) *r.parallax = O.parallax;
        if (r.H) std::memcpy(r.H, O.H, sizeof(O.H));
        if (r.E) std::memcpy(r.E, O.E, sizeof(O.E));
        if (r.R) std::memcpy(r.R, O.R, sizeof(O.R));
        if (r.T) std::memcpy(r.T, O.T, sizeof(O.T));
        if (r.h_mask && nk) std::memcpy(r.h_mask, hmk + o, nk);
        if (r.e_mask && nk) std::memcpy(r.e_mask, hmk + tot1 + o, nk);
        if (r.point_status && nk) std::memcpy(r.point_status, hmk + 2 * tot1 + o, nk);
        if (r.points && nk) std::memcpy(r.points, hpts + 3 * (size_t)o, sizeof(double) * 3 * nk);
        const size_t rb = (size_t)k * I;
        if (r.h_schedule && Ik) std::memcpy(r.h_schedule, S.host(sh) + 4 * rb, sizeof(int) * 4 * Ik);
        if (r.e_schedule && Ik) std::memcpy(r.e_schedule, S.host(se) + 5 * rb, sizeof(int) * 5 * Ik);
        if (r.h_counts && Ik) std::memcpy(r.h_counts, S.host(ch) + rb, sizeof(int) * Ik);
        if (r.e_counts && Ik) std::memcpy(r.e_counts, S.host(ce) + 11 * rb, sizeof(int) * 11 * Ik);
    }
    return 0;
}

}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_batch_two_view(pvio_b200_handle hh, int n, const pvio_b200_two_view *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_two_view_impl(h, n, records);
}
