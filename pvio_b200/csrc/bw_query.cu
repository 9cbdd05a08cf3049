// Queries on the resident slots at their current state: the joint covariance of window frames with the landmarks'
// inverse-depth variances (pvio_b200_batch_window_covariance), every landmark's world point with its covariance
// (pvio_b200_batch_window_landmarks), and the state at any time inside the window (pvio_b200_batch_window_trajectory).
#include <cmath>
#include <vector>

#include <math_constants.h>

#include "ba_cov_lm.cuh"
#include "batch_window.cuh"
#include "imu.cuh"
#include "imu_factor_cov.cuh"

namespace pvio {

// ---- pvio_b200_batch_window_landmarks: every row's world point, and for the rows the solve treats as landmarks the
// point's covariance from the covariance call's Sigma_xi and the landmark's Schur records
struct BwLmk {
    int32_t slot, n_rows, T;      // rows written; live rows of the slot
    int32_t rows_off;             // ints into the call's row list; -1: rows [0, n_rows) of the slot (every live track)
    int32_t out_off;              // rows into the call's points
    int32_t cov, cov_off, pad;    // index among the records with a covariance (-1: none); rows into its outputs
};
struct LmkArgs {
    const BwLmk *rec;             // [n]
    const int32_t *rows;          // the named rows of every record
    const int32_t *cov_rec;       // [n_cov] the record of each covariance record
    double *pts;                  // out: [rows][3]
    int32_t *role;                // out: [rows]
    int32_t *lm_of;               // scratch: [n_cov][Mcap] the packed landmark of each row of the slot, -1: none
    const int32_t *status;        // [n_cov] cov_kernel's status
    const double *sig_xi;         // [n_cov][Ncap][Ncap][36] Sigma_xi of every frame pair (cov_kernel)
    double *pcov, *var;           // out: [cov rows][9], [cov rows]
};
constexpr int kLmkWarps = 4;

// One CTA per record: Track::get_landmark_point() of every row; for a record with a covariance, the packed landmark of
// every row of its slot (bw_layout_kernel's lm_row inverted) for bw_landmark_cov_kernel
__global__ void __launch_bounds__(kBwThreads) bw_landmark_point_kernel(BwArgs a, LmkArgs L) {
    const BwLmk r = L.rec[blockIdx.x];
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    for (int k = threadIdx.x; k < r.n_rows; k += kBwThreads) {
        const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
        bw_landmark_point(a, base + row, fr, c, L.pts + 3 * ((size_t)r.out_off + k));
        L.role[r.out_off + k] = a.trole[base + row];
    }
    if (r.cov < 0) return;
    int32_t *lm = L.lm_of + (size_t)r.cov * a.Mcap;
    for (int q = threadIdx.x; q < r.T; q += kBwThreads) lm[q] = -1;
    __syncthreads();
    for (int lp = threadIdx.x; lp < a.hdr[w].M; lp += kBwThreads) lm[a.lm_row[base + lp]] = lp;
}

// row i of X_l = [[x]x, I]
__device__ __forceinline__ void lmk_xrow(const double *x, int i, double *o) {
    o[0] = i == 1 ? x[2] : (i == 2 ? -x[1] : 0.0);
    o[1] = i == 0 ? -x[2] : (i == 2 ? x[0] : 0.0);
    o[2] = i == 0 ? x[1] : (i == 1 ? -x[0] : 0.0);
    o[3] = i == 0 ? 1.0 : 0.0; o[4] = i == 1 ? 1.0 : 0.0; o[5] = i == 2 ? 1.0 : 0.0;
}

// One warp per row of a record with a covariance (grid: covariance records x row blocks).  Var(rho) as cov_lm_kernel
// forms it (ba_cov_lm.cuh), C = Cov(xi_a, rho) = -(Sigma_xi h_l)_a / H_ll from the same products, then
//   Sigma_x = X Sigma_aa X^T - X C c^T - c C^T X^T + c c^T Var(rho),  X = [[x - o]x, I], c = -(x - c_a) / rho,
// o the window's origin, about which frame_T takes xi,
// the upper triangle on six lanes, mirrored (exactly symmetric).  NaN for a row that is not a landmark of the solve and
// for every row of a record whose factorisation failed.
template <typename real>
__global__ void __launch_bounds__(32 * kLmkWarps) bw_landmark_cov_kernel(BwArgs a, LmkArgs L) {
    __shared__ double u_sm[kLmkWarps][6 * kMaxFrames];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int crec = blockIdx.x;                     // the covariance record
    const BwLmk r = L.rec[L.cov_rec[crec]];
    const int k = blockIdx.y * kLmkWarps + wv;
    if (k >= r.n_rows) return;
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
    const int lm = L.lm_of[(size_t)crec * a.Mcap + row];
    double *P = L.pcov + 9 * ((size_t)r.cov_off + k);
    double *V = L.var + r.cov_off + k;
    if (lm < 0 || L.status[crec] != PVIO_B200_OK) {
        if (lane < 9) P[lane] = CUDART_NAN;
        if (lane == 0) *V = CUDART_NAN;
        return;
    }
    const int N = a.hdr[w].N;
    const unsigned fixed = (unsigned)a.hdr[w].fixed_mask & ((1u << N) - 1u);
    const real *hs = reinterpret_cast<const real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    double *u = u_sm[wv];
    cov_lm_h(hs, a.Mcap, lm, N, fixed, lane, u);
    __syncwarp();
    const double *X = L.sig_xi + (size_t)crec * a.Ncap * a.Ncap * 36;
    const int an = __ffs(a.tmask[base + row]) - 1;
    double srow = 0.0;
    const double q = cov_lm_quad<true>(u, X, N, lane, an, srow);
    const double hll = a.lm_aux[base + lm].hll;
    const double var = cov_lm_var(hll, q);
    double C[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) C[i] = -__shfl_sync(0xffffffffu, srow, (6 * an + i) & 31) / hll;
    const double2 z = a.tz[(base + row) * a.Ncap + an];
    const double rho = a.trho[base + row];
    double qc[4], pc[3], x[3];
    bw_cam_pose(a.frames + ((size_t)w * a.Ncap + an) * kFrameStride, a.cst[w], qc, pc);
    bw_world_point(qc, pc, z.x, z.y, rho, x);
    const double cl[3] = {-(x[0] - pc[0]) / rho, -(x[1] - pc[1]) / rho, -(x[2] - pc[2]) / rho};
    const double *o = a.cst[w].origin;                  // xi is taken about the window's origin (frame_T)
    const double xo[3] = {x[0] - o[0], x[1] - o[1], x[2] - o[2]};
    if (lane < 6) {
        const int i = lane < 3 ? 0 : (lane < 5 ? 1 : 2), j = lane < 3 ? lane : (lane < 5 ? lane - 2 : 2);
        double Xi[6], Xj[6];
        lmk_xrow(xo, i, Xi);
        lmk_xrow(xo, j, Xj);
        const double *S = X + ((size_t)an * N + an) * 36;
        double s = 0.0, bi = 0.0, bj = 0.0;
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            double t = 0.0;
#pragma unroll
            for (int n = 0; n < 6; ++n) t += S[m * 6 + n] * Xj[n];
            s += Xi[m] * t;
            bi += Xi[m] * C[m];
            bj += Xj[m] * C[m];
        }
        const double cli = i == 0 ? cl[0] : (i == 1 ? cl[1] : cl[2]), clj = j == 0 ? cl[0] : (j == 1 ? cl[1] : cl[2]);
        const double v = s - bi * clj - cli * bj + cli * clj * var;
        P[3 * i + j] = v;
        P[3 * j + i] = v;
    }
    if (lane == 0) *V = var;
}

// ---- pvio_b200_batch_window_trajectory: the state at any time inside the window, forward from the preceding frame
// through the part of its IMU factor's kept samples up to that time, and its covariance
struct BwTraj {
    int32_t slot, N, n_times, cov;    // cov: index among the records with a covariance (-1: none asked; -2: asked, but
                                      // no factor holds samples)
    int64_t t_off;                    // rows into the call's times, states and frames
    int64_t cov_off;                  // doubles into the covariance scratch: the joint block of the frames that own a
                                      // factor with samples (CovRec::cov_off)
    int64_t scov_off;                 // rows into the call's state covariances
    int32_t ns[kMaxFrames];           // samples of factor k (frames k, k + 1), 0: none
};
static_assert(sizeof(BwTraj) % sizeof(double) == 0, "records are staged as whole 8-byte words");
struct TrajArgs {
    const BwTraj *rec;                // [n]
    const double *times;              // [rows]
    double *states;                   // out: [rows][16]
    int32_t *frame;                   // out: [rows]
    double *scov;                     // out: [cov rows][225]
    const double *jcov;               // cov_kernel's joint blocks (scratch)
    const int32_t *status;            // [n_cov] cov_kernel's status
    int covs;                         // 1: the per-warp covariance scratch is laid out
};
// per warp of bw_trajectory_kernel: the chain, the emitted copy, then (with covariances) four 15 x 15 matrices
__host__ __device__ constexpr size_t traj_warp_bytes(bool covs) { return 2 * sizeof(ImuWarpSm) + (covs ? 4 * 225 * 8 : 0); }

// the first of the n sorted times t[i] that is >= x (upper: > x)
__device__ __forceinline__ int traj_bound(const double *t, int n, double x, bool upper) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (upper ? t[m] <= x : t[m] < x) lo = m + 1;
        else hi = m;
    }
    return lo;
}

// queries [q0, q1) of record r, which no factor takes: frame -1, a zero state, a NaN covariance.  One warp.
__device__ __forceinline__ void none_rows(const TrajArgs &T, const BwTraj &r, int lane, int q0, int q1, bool cov) {
    for (int q = q0; q < q1; ++q) {
        const size_t row = r.t_off + q;
        if (lane < 16) T.states[16 * row + lane] = 0.0;
        if (lane == 0) T.frame[row] = -1;
        if (cov)
            for (int e = lane; e < 225; e += 32) T.scov[225 * ((size_t)r.scov_off + q) + e] = CUDART_NAN;
    }
}

// The factor k one warp serves and its queries, shared by both trajectory kernels: the times t >= s_0.t of factor k
// and below s_0.t of the next factor with samples (so k is the largest such factor whose s_0.t <= t), found by binary
// search; it takes those at most its t_end, or all of them when factor k + 1 holds samples.  The warp writes the rows
// past its t_end that no factor takes (frame -1), and with `first` those before the earliest s_0.t.  False: the warp
// has no queries.
struct TrajFac {
    int k, m, q0, q2;                 // factor, samples, queries [q0, q2)
    size_t F;                         // frame k of the slot
    const double *x, *smp, *noise;    // frame k's state, the samples, the noise [4][9]
    double t_end, bg[3], ba[3];
};
__device__ __forceinline__ bool traj_factor(const BwArgs &a, const TrajArgs &T, const BwTraj &r, int k, bool first,
                                            int lane, bool cov, TrajFac &f) {
    const int nf = r.N - 1, nq = r.n_times;
    const double *tq = T.times + r.t_off;
    const size_t F0 = (size_t)r.slot * a.Ncap;
    auto s0 = [&](int j) { return a.imu_s[(F0 + j) * a.Scap * 7]; };
    if (first) {
        double lo = CUDART_INF;
        for (int j = 0; j < nf; ++j)
            if (r.ns[j] > 0) lo = fmin(lo, s0(j));
        none_rows(T, r, lane, 0, traj_bound(tq, nq, lo, false), cov);
    }
    if (k >= nf || r.ns[k] == 0) return false;
    f.k = k; f.m = r.ns[k]; f.F = F0 + k;
    const double lo = s0(k);
    double hi = CUDART_INF;
    for (int j = k + 1; j < nf; ++j)
        if (r.ns[j] > 0) hi = fmin(hi, s0(j));
    const double *aux = a.imu_aux + f.F * kImuAux;
    f.t_end = aux[0];
    f.noise = aux + 1;
    f.q0 = traj_bound(tq, nq, lo, false);
    const int q1 = max(f.q0, traj_bound(tq, nq, hi, false));
    f.q2 = (k + 1 < nf && r.ns[k + 1] > 0) ? q1 : min(q1, max(f.q0, traj_bound(tq, nq, f.t_end, true)));
    none_rows(T, r, lane, f.q2, q1, cov);
    f.x = a.frames + f.F * kFrameStride;
    f.smp = a.imu_s + f.F * a.Scap * 7;
    for (int c = 0; c < 3; ++c) { f.bg[c] = f.x[10 + c]; f.ba[c] = f.x[13 + c]; }
    return f.q0 < f.q2;
}

// The forward walk of a factor's samples, as imu_integrate_warp walks them (imu_step_warp), emitting each query as the
// walk passes it: the increment of the last sample at or before t, over t - s_j.t, goes onto a copy E of the chain S,
// which is what imu_integrate_warp gives for the samples at or before t with t_end = t; then emit(q).  knot(j) sees
// the chain at s_j.t before sample j is stepped.  ToEnd: walk every sample, leaving the full re-integration in S;
// otherwise stop after the last query.
template <bool ToEnd, typename Knot, typename Emit>
__device__ __forceinline__ void traj_walk(ImuWarpSm &S, ImuWarpSm &E, const TrajFac &f, const double *tq, int lane,
                                          Knot knot, Emit emit) {
    imu_reset_warp(S, lane);
    int q = f.q0;
    for (int j = 0; j < f.m && (ToEnd || q < f.q2); ++j) {
        const double *d = f.smp + (size_t)j * 7;
        const bool last = j + 1 == f.m;
        const double t_next = last ? f.t_end : f.smp[(size_t)(j + 1) * 7];
        knot(j);
        for (; q < f.q2 && (last || tq[q] < t_next); ++q) {   // the queries whose last sample is s_j
            imu_copy_warp(S, E, lane);
            imu_step_warp(E, lane, d, tq[q] - d[0], f.bg, f.ba, f.noise);
            emit(q);
        }
        if (ToEnd || (!last && q < f.q2)) imu_step_warp(S, lane, d, t_next - d[0], f.bg, f.ba, f.noise);
    }
}

// One CTA per record, one warp per factor k with samples (warp k), each walking its samples once (traj_factor,
// traj_walk).  Each query's state is PreIntegrator::predict from frame k's state, and with a covariance Phi Sigma_k
// Phi^T + Psi Sigma_delta Psi^T (imu_factor_propagate), Sigma_delta the partial increment's covariance itself.  Times
// no warp takes (before the first sample, past a factor's t_end, over a factor without samples) get frame -1, a zero
// state and a NaN covariance: warp 0 writes those before the earliest s_0.t, each warp those past its t_end.
__global__ void __launch_bounds__(32 * (kMaxFrames - 1)) bw_trajectory_kernel(BwArgs a, TrajArgs T) {
    extern __shared__ __align__(16) unsigned char traj_sm[];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const BwTraj &r = T.rec[blockIdx.x];
    const int nf = r.N - 1;
    const double *tq = T.times + r.t_off;
    const bool cov = r.cov != -1;                           // -2: covariances asked, no factor holds samples
    const bool cov_ok = r.cov >= 0 && T.status[r.cov] == PVIO_B200_OK;
    TrajFac f;
    if (!traj_factor(a, T, r, wv, wv == 0, lane, cov, f)) return;
    const int k = f.k;
    unsigned char *base = traj_sm + (size_t)wv * traj_warp_bytes(T.covs);
    ImuWarpSm &S = *reinterpret_cast<ImuWarpSm *>(base), &E = *reinterpret_cast<ImuWarpSm *>(base + sizeof(ImuWarpSm));
    double *A = reinterpret_cast<double *>(base + 2 * sizeof(ImuWarpSm)), *B = A + 225, *C = B + 225, *D = C + 225;
    const double *x = f.x;
    // Sigma_k: frame k's diagonal block of the joint covariance of the frames that own a factor with samples
    unsigned has = 0;
    for (int j = 0; j < nf; ++j) has |= (r.ns[j] > 0 ? 1u : 0u) << j;
    const int K15 = 15 * __popc(has), p15 = 15 * __popc(has & ((1u << k) - 1u));
    const double *Sk = T.jcov + r.cov_off + (size_t)p15 * K15 + p15;
    traj_walk<false>(S, E, f, tq, lane, [](int) {}, [&](int q) {
        const size_t row = r.t_off + q;
        if (lane == 0) {
            bw_imu_predict(x, E.tsum, E.q, E.p, E.v, T.states + 16 * row);
            T.frame[row] = k;
        }
        if (!cov) return;
        double *out = T.scov + 225 * (size_t)(r.scov_off + q);
        if (!cov_ok) {
            for (int e = lane; e < 225; e += 32) out[e] = CUDART_NAN;
            return;
        }
        for (int e = lane; e < 225; e += 32) {
            const int i = e / 15, c = e % 15;
            A[e] = 0.5 * (Sk[(size_t)i * K15 + c] + Sk[(size_t)c * K15 + i]);
            D[e] = (i < 9 && c < 9) ? E.C[i * 9 + c]
                 : (i >= 9 && i < 12 && c >= 9 && c < 12) ? E.cbg[(i - 9) * 3 + c - 9]
                 : (i >= 12 && c >= 12) ? E.cba[(i - 12) * 3 + c - 12] : 0.0;
        }
        __syncwarp();
        double Rs[9], dR[9];
        quat_to_mat(x, Rs);
        quat_to_mat(E.q, dR);
        const ImuFactorJac fj{E.tsum, E.p, E.v, E.dq_dbg, E.dp_dbg, E.dp_dba, E.dv_dbg, E.dv_dba};
        imu_factor_propagate(A, B, C, D, fj, Rs, dR, lane);
        for (int e = lane; e < 225; e += 32) {
            const int i = e / 15, c = e % 15;
            out[e] = 0.5 * ((A[e] + D[e]) + (A[c * 15 + i] + D[c * 15 + i]));
        }
        __syncwarp();
    });
}

// ---- pvio_b200_batch_window_smoothed_trajectory: the state at t conditioned on both frames around it (the header's
// definition).  Per query the forward walk keeps the partial increment Delta(t) in global scratch (kTrajSnap doubles:
// C, cbg, cba, the five bias Jacobians, q, p, v, dt), and per knot the chain's rotation at s_j (4 doubles).
constexpr int kTrajSnap = 156;
struct TrajSmooth {
    double *snap;                     // [rows][kTrajSnap]
    double *knot;                     // [records][kMaxFrames - 1][Scap][4]
};

// one step's transition A = [[Ri, 0, 0], [-dt^2/2 M, I, dt I], [-dt M, 0, I]] over dt of sample d from rotation q, as
// imu_step_warp forms Ri and M.  Lane 0.
struct TrajA { double Ri[9], M[9], dt; };
__device__ __forceinline__ void traj_a(TrajA &A, const double *d, const double *q, double dt, const double *bg,
                                       const double *ba) {
    const double th[3] = {(d[1] - bg[0]) * dt, (d[2] - bg[1]) * dt, (d[3] - bg[2]) * dt};
    const double acc[3] = {d[4] - ba[0], d[5] - ba[1], d[6] - ba[2]};
    double qi[4], qc[4], Rd[9], Ha[9];
    expmap(th, qi);
    quat_conj(qi, qc);
    quat_to_mat(qc, A.Ri);
    quat_to_mat(q, Rd);
    hat(acc, Ha);
    mat3_mul(Rd, Ha, A.M);
    A.dt = dt;
}
// entry (r, c) of A^T X (xt: of A^T X^T), X 9 x 9 row-major
__device__ __forceinline__ double traj_at(const TrajA &A, const double *X, int r, int c, bool xt) {
    auto x = [&](int i, int j) { return xt ? X[j * 9 + i] : X[i * 9 + j]; };
    const double dt = A.dt;
    if (r >= 6) return dt * x(r - 3, c) + x(r, c);
    if (r >= 3) return x(r, c);
    double s = 0.0, m = 0.0;
    for (int k = 0; k < 3; ++k) {
        s += A.Ri[k * 3 + r] * x(k, c);
        m += A.M[k * 3 + r] * (0.5 * dt * dt * x(3 + k, c) + dt * x(6 + k, c));
    }
    return s - m;
}
// Y = A^T X (xt: A^T X^T), by the warp's lanes; Y must not alias X
__device__ __forceinline__ void traj_at_warp(const TrajA &A, const double *X, double *Y, bool xt, int lane) {
    for (int e = lane; e < 81; e += 32) Y[e] = traj_at(A, X, e / 9, e % 9, xt);
    __syncwarp();
}
// y = A^T v (9).  One lane.
__device__ __forceinline__ void traj_at_vec(const TrajA &A, const double *v, double *y) {
    const double dt = A.dt;
    for (int r = 0; r < 3; ++r) {
        double s = 0.0, m = 0.0;
        for (int k = 0; k < 3; ++k) {
            s += A.Ri[k * 3 + r] * v[k];
            m += A.M[k * 3 + r] * (0.5 * dt * dt * v[3 + k] + dt * v[6 + k]);
        }
        y[r] = s - m;
    }
    for (int r = 3; r < 6; ++r) y[r] = v[r];
    for (int r = 6; r < 9; ++r) y[r] = dt * v[r - 3] + v[r];
}
// C = A B (n x n, row-major; A, B with leading dimension n), by the warp's lanes
__device__ __forceinline__ void traj_mm(const double *A, const double *B, double *C, int n, int lane) {
    for (int e = lane; e < n * n; e += 32) {
        const int i = e / n, j = e % n;
        double s = 0.0;
        for (int m = 0; m < n; ++m) s += A[i * n + m] * B[m * n + j];
        C[e] = s;
    }
    __syncwarp();
}

// per warp of bw_smoothed_trajectory_kernel
struct TrajSmSm {
    ImuWarpSm S, E;                   // the chain (after the walk: Delta(T)), a query's partial increment
    TrajA A;                          // the step the backward pass is at
    double r[15], lam[15];            // the residual; Sigma(T)^-1 r carried back to the pass's knot (bias parts fixed)
    double u[15], Gu[9], Eu[9];       // a query's K r; Jr(u_theta) and R(exp(u_theta))
    double U9[81], Ub[18];            // sqrt_inv_block of C(T), cbg(T), cba(T)
    double Rk[9], Jri[9];             // R(q_k), Jr(r_theta)^-1
    double dqs[4], dps[3], dvs[3], dqdbg[9];      // a query's Delta_s, its dq_dbg carried through exp(u_theta)
    int pd;                           // Sigma(T) positive definite
};
struct TrajSmCov {                    // with covariances
    double L[81], W[81];              // Phi^T C(T)^-1 and Phi^T C(T)^-1 Phi at the pass's knot
    double Cb[18];                    // cbg(T)^-1, cba(T)^-1
    double X[4][81];                  // 9 x 9 scratch
    double Dk[225], P[4][225];        // dr/dx_k; 15 x 15 scratch
};
__host__ __device__ constexpr size_t traj_smooth_bytes(bool covs) {
    return sizeof(TrajSmSm) + (covs ? sizeof(TrajSmCov) : 0);
}

// rows 0-2 of the 15 x 15 P by G (null: unchanged), rows 3-5 and 6-8 by R: P <- diag(G, R, R, I, I) P.  Lane per column.
__device__ __forceinline__ void traj_rows(double *P, const double *G, const double *R, int lane) {
    if (lane < 15) {
        double t[9];
        for (int i = 0; i < 9; ++i) t[i] = P[i * 15 + lane];
        for (int b = G ? 0 : 1; b < 3; ++b) {
            const double *X = b == 0 ? G : R;
            for (int i = 0; i < 3; ++i)
                P[(3 * b + i) * 15 + lane] = X[3 * i] * t[3 * b] + X[3 * i + 1] * t[3 * b + 1] + X[3 * i + 2] * t[3 * b + 2];
        }
    }
    __syncwarp();
}
// columns 0-2 of the 15 x 15 P by G (null: unchanged), columns 3-5 and 6-8 by R^T: P <- P diag(G, R^T, R^T, I, I).
// Lane per row.
__device__ __forceinline__ void traj_cols(double *P, const double *G, const double *R, int lane) {
    if (lane < 15) {
        double t[9];
        double *row = P + lane * 15;
        for (int i = 0; i < 9; ++i) t[i] = row[i];
        for (int b = G ? 0 : 1; b < 3; ++b)
            for (int c = 0; c < 3; ++c)
                row[3 * b + c] = b == 0 ? t[0] * G[c] + t[1] * G[3 + c] + t[2] * G[6 + c]
                                        : t[3 * b] * R[3 * c] + t[3 * b + 1] * R[3 * c + 1] + t[3 * b + 2] * R[3 * c + 2];
    }
    __syncwarp();
}

// One CTA of one warp per (record, factor k with samples): grid (records, factors).  The forward walk of
// bw_trajectory_kernel runs to t_end (traj_walk<true>), keeping each query's partial increment and each knot's
// rotation in global scratch; then r and sqrt_inv_block of Sigma(T) (frame -2 for every query when Sigma(T) is not
// positive definite), and a backward adjoint pass over the knots that carries lam = Phi^T Sigma(T)^-1 r, and with
// covariances L = Phi^T C(T)^-1 and W = Phi^T C(T)^-1 Phi, one step per sample, emitting each query as it reaches it:
//   K r = C(t) A_t^T lam,  K = C(t) A_t^T L,  Sigma_c = C(t) - C(t) A_t^T W A_t C(t)
// with A_t the rest of the query's sample from t (bias blocks: cbg(t) cbg(T)^-1); past t_end K = A the last sample
// from t_end on to t.  Then the state is predict(x_k, Delta(t) (+) K r) with the bias part of K r added, and the
// covariance J Sigma_{k,k+1} J^T + Psi Sigma_c Psi^T (the header's definition), exactly symmetric.  Linear in samples
// plus queries; shared memory does not grow with either.
__global__ void __launch_bounds__(32) bw_smoothed_trajectory_kernel(BwArgs a, TrajArgs T, TrajSmooth Z) {
    extern __shared__ __align__(16) unsigned char traj_sm[];
    const int lane = threadIdx.x;
    const BwTraj &r = T.rec[blockIdx.x];
    const int nf = r.N - 1;
    const double *tq = T.times + r.t_off;
    const bool cov = r.cov != -1;
    const bool cov_ok = r.cov >= 0 && T.status[r.cov] == PVIO_B200_OK;
    TrajFac f;
    if (!traj_factor(a, T, r, blockIdx.y, blockIdx.y == 0, lane, cov, f)) return;
    TrajSmSm &W = *reinterpret_cast<TrajSmSm *>(traj_sm);
    TrajSmCov &V = *reinterpret_cast<TrajSmCov *>(traj_sm + sizeof(TrajSmSm));
    ImuWarpSm &S = W.S, &E = W.E;
    const int k = f.k;
    const double *x = f.x, *x1 = x + kFrameStride;
    double *kq = Z.knot + ((size_t)blockIdx.x * (kMaxFrames - 1) + k) * a.Scap * 4;
    traj_walk<true>(S, E, f, tq, lane, [&](int j) { if (lane < 4) kq[4 * j + lane] = S.q[lane]; }, [&](int q) {
        double *z = Z.snap + (size_t)(r.t_off + q) * kTrajSnap;
        for (int e = lane; e < 81; e += 32) z[e] = E.C[e];
        if (lane < 9) {
            z[81 + lane] = E.cbg[lane]; z[90 + lane] = E.cba[lane]; z[99 + lane] = E.dq_dbg[lane];
            z[108 + lane] = E.dp_dbg[lane]; z[117 + lane] = E.dp_dba[lane]; z[126 + lane] = E.dv_dbg[lane];
            z[135 + lane] = E.dv_dba[lane];
        }
        if (lane < 4) z[144 + lane] = E.q[lane];
        if (lane < 3) { z[148 + lane] = E.p[lane]; z[151 + lane] = E.v[lane]; }
        if (lane == 0) z[154] = E.tsum;
        __syncwarp();
    });
    // ---- r = Delta* (-) Delta(T) and the factors of Sigma(T)
    const double Tt = S.tsum;
    double dsp[3], dsv[3], dsq[4];                           // Delta* (lane 0)
    if (lane == 0) {
        const double g[3] = {0.0, 0.0, -9.80665};            // as bw_imu_predict
        double qc[4], qe[4], y[3];
        quat_to_mat(x, W.Rk);
        quat_conj(x, qc);
        quat_mul(qc, x1, dsq);
        quat_conj(S.q, qc);
        quat_mul(qc, dsq, qe);
        logmap(qe, W.r);
        for (int c = 0; c < 3; ++c) y[c] = x1[4 + c] - x[4 + c] - x[7 + c] * Tt - 0.5 * g[c] * Tt * Tt;
        mat3_tvec(W.Rk, y, dsp);
        for (int c = 0; c < 3; ++c) y[c] = x1[7 + c] - x[7 + c] - g[c] * Tt;
        mat3_tvec(W.Rk, y, dsv);
        for (int c = 0; c < 3; ++c) {
            W.r[3 + c] = dsp[c] - S.p[c];
            W.r[6 + c] = dsv[c] - S.v[c];
            W.r[9 + c] = x1[10 + c] - x[10 + c];
            W.r[12 + c] = x1[13 + c] - x[13 + c];
        }
        sqrt_inv_block(S.C, 9, 9, W.U9, 9);
    } else if (lane == 1) {
        sqrt_inv_block(S.cbg, 3, 3, W.Ub, 3);
    } else if (lane == 2) {
        sqrt_inv_block(S.cba, 3, 3, W.Ub + 9, 3);
    }
    __syncwarp();
    if (lane == 0) {            // every pivot R_jj^2 = U_jj^-2 above 1e-10 C_jj (a one-sample factor's C(T) has rank 6)
        bool pd = true;
        for (int j = 0; j < 15; ++j) {
            const double u = j < 9 ? W.U9[j * 10] : W.Ub[(j - 9) / 3 * 9 + (j % 3) * 4];
            const double c = j < 9 ? S.C[j * 10] : (j < 12 ? S.cbg : S.cba)[(j % 3) * 4];
            pd = pd && u > 0.0 && u < CUDART_INF && u * u * c * 1e-10 < 1.0;
        }
        W.pd = pd;
    }
    __syncwarp();
    if (!W.pd) {                                             // no smoother: frame -2
        for (int q = f.q0; q < f.q2; ++q) {
            const size_t row = r.t_off + q;
            if (lane < 16) T.states[16 * row + lane] = 0.0;
            if (lane == 0) T.frame[row] = -2;
            if (cov)
                for (int e = lane; e < 225; e += 32) T.scov[225 * ((size_t)r.scov_off + q) + e] = CUDART_NAN;
        }
        return;
    }
    const bool cv = cov && cov_ok;
    if (lane == 0) {                                         // lam = Sigma(T)^-1 r
        double y[9];
        for (int i = 0; i < 9; ++i) {
            double s = 0.0;
            for (int j = i; j < 9; ++j) s += W.U9[i * 9 + j] * W.r[j];
            y[i] = s;
        }
        for (int i = 0; i < 9; ++i) {
            double s = 0.0;
            for (int j = 0; j <= i; ++j) s += W.U9[j * 9 + i] * y[j];
            W.lam[i] = s;
        }
        for (int b = 0; b < 2; ++b) {
            const double *U = W.Ub + 9 * b, *rb = W.r + 9 + 3 * b;
            for (int i = 0; i < 3; ++i) {
                double s = 0.0;
                for (int j = i; j < 3; ++j) s += U[i * 3 + j] * rb[j];
                y[i] = s;
            }
            for (int i = 0; i < 3; ++i) {
                double s = 0.0;
                for (int j = 0; j <= i; ++j) s += U[j * 3 + i] * y[j];
                W.lam[9 + 3 * b + i] = s;
            }
        }
        double J[9];
        right_jacobian(W.r, J);
        mat3_inv(J, W.Jri);
    }
    __syncwarp();
    if (cv) {
        for (int e = lane; e < 81; e += 32) {                // L = W = C(T)^-1 = U^T U
            const int i = e / 9, j = e % 9;
            double s = 0.0;
            for (int m = 0; m <= min(i, j); ++m) s += W.U9[m * 9 + i] * W.U9[m * 9 + j];
            V.L[e] = s;
            V.W[e] = s;
        }
        if (lane < 18) {
            const double *U = W.Ub + 9 * (lane / 9);
            const int i = (lane % 9) / 3, j = lane % 3;
            double s = 0.0;
            for (int m = 0; m <= min(i, j); ++m) s += U[m * 3 + i] * U[m * 3 + j];
            V.Cb[lane] = s;
        }
        for (int e = lane; e < 225; e += 32) V.Dk[e] = 0.0;
        __syncwarp();
        if (lane == 0) {                                     // dr/dx_k
            double Er[9], Rq[9], X[9], Y[9], qe[4];
            expmap(W.r, qe);
            quat_to_mat(qe, Er);
            quat_to_mat(dsq, Rq);
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) Y[3 * i + j] = Rq[3 * j + i];
            mat3_mul(W.Jri, Y, X);
            put_block(V.Dk, 0, 0, X, -1.0);
            mat3_mul_tn(Er, S.dq_dbg, Y);
            mat3_mul(W.Jri, Y, X);
            put_block(V.Dk, 0, 3, X, -1.0);
            for (int i = 0; i < 3; ++i)
                for (int j = 0; j < 3; ++j) Y[3 * i + j] = W.Rk[3 * j + i];
            hat(dsp, X);
            put_block(V.Dk, 1, 0, X);
            put_block(V.Dk, 1, 1, Y, -1.0);
            put_block(V.Dk, 1, 2, Y, -Tt);
            put_block(V.Dk, 1, 3, S.dp_dbg, -1.0);
            put_block(V.Dk, 1, 4, S.dp_dba, -1.0);
            hat(dsv, X);
            put_block(V.Dk, 2, 0, X);
            put_block(V.Dk, 2, 2, Y, -1.0);
            put_block(V.Dk, 2, 3, S.dv_dbg, -1.0);
            put_block(V.Dk, 2, 4, S.dv_dba, -1.0);
            put_block(V.Dk, 3, 3, nullptr, -1.0);
            put_block(V.Dk, 4, 4, nullptr, -1.0);
        }
        __syncwarp();
    }
    // Sigma_{k,k+1}: frames k and k + 1 in the joint block of the frames {k, k + 1 : factor k holds samples}
    unsigned has = 0;
    for (int j = 0; j < nf; ++j) has |= (r.ns[j] > 0 ? 3u : 0u) << j;
    const int K15 = 15 * __popc(has), p15 = 15 * __popc(has & ((1u << k) - 1u));
    const double *Sj = T.jcov + r.cov_off + (size_t)p15 * K15 + p15;
    auto sjoint = [&](int i, int c) { return 0.5 * (Sj[(size_t)i * K15 + c] + Sj[(size_t)c * K15 + i]); };

    // one query: row q, its partial increment z; gap: past t_end
    auto emit = [&](int q, bool gap) {
        const size_t row = r.t_off + q;
        const double *z = Z.snap + row * kTrajSnap, *Ct = z;
        if (lane == 0) {
            double *u = W.u;
            if (gap) {                                       // K r = A r (bias part r)
                double mr[3];
                mat3_vec(W.A.M, W.r, mr);
                mat3_vec(W.A.Ri, W.r, u);
                const double dt = W.A.dt;
                for (int c = 0; c < 3; ++c) {
                    u[3 + c] = -0.5 * dt * dt * mr[c] + W.r[3 + c] + dt * W.r[6 + c];
                    u[6 + c] = -dt * mr[c] + W.r[6 + c];
                    u[9 + c] = W.r[9 + c];
                    u[12 + c] = W.r[12 + c];
                }
            } else {                                         // K r = C(t) A_t^T lam, cbg(t) lam_bg, cba(t) lam_ba
                double lt[9];
                traj_at_vec(W.A, W.lam, lt);
                for (int i = 0; i < 9; ++i) {
                    double s = 0.0;
                    for (int j = 0; j < 9; ++j) s += Ct[i * 9 + j] * lt[j];
                    u[i] = s;
                }
                for (int i = 0; i < 6; ++i) {
                    const double *Cb = z + 81 + 9 * (i / 3);
                    const int ib = i % 3;
                    u[9 + i] = Cb[ib * 3] * W.lam[9 + i - ib] + Cb[ib * 3 + 1] * W.lam[10 + i - ib] +
                               Cb[ib * 3 + 2] * W.lam[11 + i - ib];
                }
            }
            // Delta_s = Delta(t) (+) u: the rotation on the right (exactly Delta(t)'s when u_theta = 0)
            double qe[4];
            expmap(u, qe);
            quat_to_mat(qe, W.Eu);
            right_jacobian(u, W.Gu);
            if (u[0] == 0.0 && u[1] == 0.0 && u[2] == 0.0)
                for (int c = 0; c < 4; ++c) W.dqs[c] = z[144 + c];
            else quat_mul(z + 144, qe, W.dqs);
            for (int c = 0; c < 3; ++c) { W.dps[c] = z[148 + c] + u[3 + c]; W.dvs[c] = z[151 + c] + u[6 + c]; }
            double *y = T.states + 16 * row;
            bw_imu_predict(x, z[154], W.dqs, W.dps, W.dvs, y);
            for (int c = 0; c < 6; ++c) y[10 + c] = x[10 + c] + u[9 + c];
            T.frame[row] = k;
            mat3_mul_tn(W.Eu, z + 99, W.dqdbg);
        }
        __syncwarp();
        if (!cov) return;
        double *out = T.scov + 225 * (size_t)(r.scov_off + q);
        if (!cov_ok) {
            for (int e = lane; e < 225; e += 32) out[e] = CUDART_NAN;
            return;
        }
        double (*X)[81] = V.X;
        // K9 into X[1], Sigma_c's 9 x 9 block into X[3]
        if (gap) {
            for (int e = lane; e < 81; e += 32) X[0][e] = e / 9 == e % 9 ? 1.0 : 0.0;
            __syncwarp();
            traj_at_warp(W.A, X[0], X[2], false, lane);     // A^T
            for (int e = lane; e < 81; e += 32) X[1][e] = X[2][(e % 9) * 9 + e / 9];
            __syncwarp();
            traj_mm(X[1], S.C, X[0], 9, lane);              // A C(T)
            traj_mm(X[0], X[2], X[3], 9, lane);             // .. A^T
            for (int e = lane; e < 81; e += 32) X[3][e] = Ct[e] - X[3][e];
        } else {
            traj_at_warp(W.A, V.L, X[0], false, lane);      // L(t)
            traj_mm(Ct, X[0], X[1], 9, lane);               // K9
            traj_at_warp(W.A, V.W, X[0], false, lane);      // A^T W
            traj_at_warp(W.A, X[0], X[2], true, lane);      // W(t)^T
            for (int e = lane; e < 81; e += 32) X[0][e] = X[2][(e % 9) * 9 + e / 9];
            __syncwarp();
            traj_mm(X[0], Ct, X[2], 9, lane);               // W(t) C(t)
            traj_mm(Ct, X[2], X[0], 9, lane);               // C(t) W(t) C(t)
            for (int e = lane; e < 81; e += 32) X[3][e] = Ct[e] - X[0][e];
        }
        __syncwarp();
        double *P0 = V.P[0], *P1 = V.P[1], *P2 = V.P[2], *P3 = V.P[3];
        for (int e = lane; e < 225; e += 32) {               // K into P0, Sigma_c into P1 (block diagonal)
            const int i = e / 15, c = e % 15;
            double kv = 0.0, sv = 0.0;
            if (i < 9 && c < 9) { kv = X[1][i * 9 + c]; sv = X[3][i * 9 + c]; }
            else if (i >= 9 && c >= 9 && (i - 9) / 3 == (c - 9) / 3) {
                const int b = (i - 9) / 3, ib = (i - 9) % 3, cb = (c - 9) % 3;
                const double *Cb = z + 81 + 9 * b, *CT = b == 0 ? S.cbg : S.cba, *Ci = V.Cb + 9 * b;
                if (gap) { kv = ib == cb ? 1.0 : 0.0; sv = Cb[ib * 3 + cb] - CT[ib * 3 + cb]; }
                else {
                    double ki[3];
                    for (int m = 0; m < 3; ++m)
                        ki[m] = Cb[ib * 3] * Ci[m] + Cb[ib * 3 + 1] * Ci[3 + m] + Cb[ib * 3 + 2] * Ci[6 + m];
                    kv = ki[cb];
                    sv = Cb[ib * 3 + cb] - (ki[0] * Cb[cb] + ki[1] * Cb[3 + cb] + ki[2] * Cb[6 + cb]);
                }
            }
            P0[e] = kv;
            P1[e] = sv;
        }
        __syncwarp();
        // J_k = Phi + Psi G K dr/dx_k into P3, J_k1 = Psi G K dr/dx_k1 into P2
        warp_mm15(P0, V.Dk, P2, false, lane);
        traj_rows(P2, W.Gu, W.Rk, lane);
        double dR[9];
        quat_to_mat(W.dqs, dR);
        const ImuFactorJac fj{z[154], W.dps, W.dvs, W.dqdbg, z + 108, z + 117, z + 126, z + 135};
        imu_factor_phi(P3, fj, W.Rk, dR, lane);
        for (int e = lane; e < 225; e += 32) P3[e] += P2[e];
        __syncwarp();
        for (int e = lane; e < 225; e += 32) P2[e] = P0[e];
        __syncwarp();
        traj_cols(P2, W.Jri, W.Rk, lane);
        traj_rows(P2, W.Gu, W.Rk, lane);
        // J Sigma_{k,k+1} J^T + Psi Sigma_c Psi^T
        double acc[8];
        for (int h = 0; h < 2; ++h) {
            for (int e = lane; e < 225; e += 32) {           // J_k Sigma_{k,h} + J_k1 Sigma_{k+1,h}
                const int i = e / 15, c = e % 15;
                double s = 0.0;
                for (int m = 0; m < 15; ++m)
                    s += P3[i * 15 + m] * sjoint(m, 15 * h + c) + P2[i * 15 + m] * sjoint(15 + m, 15 * h + c);
                P0[e] = s;
            }
            __syncwarp();
            const double *Jh = h == 0 ? P3 : P2;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
                const int e = lane + 32 * g;
                if (e >= 225) continue;
                const int i = e / 15, c = e % 15;
                double s = 0.0;
                for (int m = 0; m < 15; ++m) s += P0[i * 15 + m] * Jh[c * 15 + m];
                acc[g] = h == 0 ? s : acc[g] + s;
            }
            __syncwarp();
        }
        traj_rows(P1, nullptr, W.Rk, lane);
        traj_cols(P1, nullptr, W.Rk, lane);
#pragma unroll
        for (int g = 0; g < 8; ++g) {
            const int e = lane + 32 * g;
            if (e < 225) P0[e] = acc[g] + P1[e];
        }
        __syncwarp();
        for (int e = lane; e < 225; e += 32) out[e] = 0.5 * (P0[e] + P0[(e % 15) * 15 + e / 15]);
        __syncwarp();
    };

    // ---- the backward pass: the queries past t_end, then per sample from the last down
    int q = f.q2 - 1;
    for (; q >= f.q0 && tq[q] > f.t_end; --q) {
        if (lane == 0) traj_a(W.A, f.smp + (size_t)(f.m - 1) * 7, S.q, tq[q] - f.t_end, f.bg, f.ba);
        __syncwarp();
        emit(q, true);
    }
    for (int j = f.m - 1; j >= 0 && q >= f.q0; --j) {
        const double *d = f.smp + (size_t)j * 7;
        const double t_next = j + 1 < f.m ? f.smp[(size_t)(j + 1) * 7] : f.t_end;
        for (; q >= f.q0 && tq[q] >= d[0]; --q) {            // the rest of sample j from t
            if (lane == 0) traj_a(W.A, d, Z.snap + (size_t)(r.t_off + q) * kTrajSnap + 144, t_next - tq[q], f.bg, f.ba);
            __syncwarp();
            emit(q, false);
        }
        if (j == 0 || q < f.q0) break;
        if (lane == 0) {                                     // the whole sample j: lam <- A_j^T lam
            traj_a(W.A, d, kq + 4 * j, t_next - d[0], f.bg, f.ba);
            double y[9];
            traj_at_vec(W.A, W.lam, y);
            for (int i = 0; i < 9; ++i) W.lam[i] = y[i];
        }
        __syncwarp();
        if (cv) {                                            // L <- A^T L, W <- A^T W A
            traj_at_warp(W.A, V.L, V.X[0], false, lane);
            for (int e = lane; e < 81; e += 32) V.L[e] = V.X[0][e];
            traj_at_warp(W.A, V.W, V.X[0], false, lane);
            traj_at_warp(W.A, V.X[0], V.X[1], true, lane);
            for (int e = lane; e < 81; e += 32) V.W[e] = V.X[1][(e % 9) * 9 + e / 9];
            __syncwarp();
        }
    }
}

// the landmark index of every row of a slot in its packed window (rows of role < 0 with >= 2 observations, stably by
// anchor, as bw_layout_kernel orders them), -1 for the other rows
static std::vector<int32_t> landmark_of_rows(const WinSlot &s) {
    const int T = (int)s.ids.size();
    std::vector<int32_t> lm(T, -1);
    int k = 0;
    for (int a = 0; a < kMaxFrames; ++a)
        for (int r = 0; r < T; ++r)
            if (s.role[r] < 0 && __builtin_popcount(s.mask[r]) >= 2 && __builtin_ctz(s.mask[r]) == a) lm[r] = k++;
    return lm;
}

// The covariance systems a call solves: one CovRec per slot whose Sigma_xi it needs, the frames of each record's joint
// block, the Sigma_delta scratch.  stage declares their sections (the joint blocks of kind `blocks`), run launches the
// systems (with_lms: and the covariance call's landmark variances).
struct CovPlan {
    std::vector<CovRec> recs;
    std::vector<int32_t> slots, frames;
    int64_t cov_n = 0, sig_n = 0;
    Stage::Sec<CovRec> rec;
    Stage::Sec<int32_t> fr, sl, st;
    Stage::Sec<double> cov, sig, sxi;

    // a record of slot `slot` with the joint block of frames f[0 .. nf): its index, -1 when the slot's reduced system is
    // too large for cov_kernel's shared memory
    int add(const Handle *h, int slot, int nf = 0, const int32_t *f = nullptr) {
        if (cov_smem_bytes(h->hdr.h[slot]) > 220 * 1024) return -1;
        const WinSlot &s = h->slots[slot];
        const int64_t D = (s.inertial ? 15 : 6) * (int64_t)s.N;
        recs.push_back(CovRec{slot, nf, (int32_t)frames.size(), 0, cov_n, sig_n});
        slots.push_back(slot);
        frames.insert(frames.end(), f, f + nf);
        cov_n += 225 * (int64_t)nf * nf;
        sig_n += D * D;
        return (int)recs.size() - 1;
    }
    void stage(Stage &S, const Handle *h, Stage::Kind blocks) {
        const size_t n = recs.size();
        rec = S.up(recs); fr = S.up(frames); sl = S.up(slots);
        cov = S.add<double>(blocks, (size_t)cov_n); st = S.add<int32_t>(Stage::kDown, n);
        sig = S.add<double>(Stage::kScratch, (size_t)sig_n); sxi = S.add<double>(Stage::kScratch, n * h->Ncap * h->Ncap * 36);
    }
    int run(Handle *h, const Stage &S, bool with_lms = false, const CovLm *lms = nullptr, int n_lm = 0, double *var = nullptr) const {
        const int n = (int)recs.size();
        const CovLaunch L{S.dev(rec), S.dev(fr), lms, n_lm, S.dev(cov), var, S.dev(st), S.dev(sig), S.dev(sxi)};
        if (n == 0) return 0;
        return with_lms ? run_covariance(h, n, slots.data(), S.dev(sl), L) : run_cov_system(h, n, slots.data(), S.dev(sl), L);
    }
};

}  // namespace pvio

using namespace pvio;

// pvio_b200_batch_window_trajectory and (smooth) pvio_b200_batch_window_smoothed_trajectory: one validation, staging
// and download
static int trajectory_call(pvio_b200_handle hh, int n, pvio_b200_window_trajectory *records, bool smooth) {
    BwCall C(hh, smooth ? "batch_window_smoothed_trajectory" : "batch_window_trajectory");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked before anything is staged
    std::vector<BwTraj> recs(n);
    std::vector<double> times;
    CovPlan P;
    int64_t rows = 0, cov_rows = 0;
    int warps = 1;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_trajectory &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return C.bad("a visual-only slot");
        if (R.n_times < 0) return C.bad("a negative time count");
        if (R.n_times > 0 && (!R.times || !R.states || !R.frame)) return C.bad("times, states or frame missing");
        for (int q = 0; q < R.n_times; ++q) {
            if (!std::isfinite(R.times[q])) return C.bad("a time that is not finite");
            if (q > 0 && R.times[q] < R.times[q - 1]) return C.bad("times that decrease");
        }
        BwTraj &T = recs[i];
        T = BwTraj{};
        T.slot = R.slot; T.N = s.N; T.n_times = R.n_times; T.cov = -1; T.t_off = rows; T.scov_off = cov_rows;
        std::vector<int32_t> owners;                 // the frames that own a factor with samples (smooth: and the
        for (int k = 0; k + 1 < s.N; ++k) {          // frames after them)
            T.ns[k] = s.n_samples.empty() ? 0 : s.n_samples[k];
            if (T.ns[k] > 0 && (owners.empty() || owners.back() != k)) owners.push_back(k);
            if (T.ns[k] > 0 && smooth) owners.push_back(k + 1);
        }
        warps = std::max(warps, s.N - 1);
        if (R.state_cov && !owners.empty()) {        // their joint block
            T.cov_off = P.cov_n;
            T.cov = P.add(h, R.slot, (int)owners.size(), owners.data());
            if (T.cov < 0) return C.bad("reduced system too large for shared memory");
        }
        if (R.state_cov) {
            if (T.cov < 0) T.cov = -2;               // NaN rows only: no factor holds samples
            cov_rows += R.n_times;
        }
        times.insert(times.end(), R.times, R.times + R.n_times);
        rows += R.n_times;
    }
    const bool any_cov = cov_rows > 0;
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto tm = S.up(times);
    P.stage(S, h, Stage::kScratch);
    const auto sto = S.add<double>(Stage::kDown, 16 * (size_t)rows);
    const auto fro = S.add<int32_t>(Stage::kDown, (size_t)rows);
    const auto sco = S.add<double>(Stage::kDown, 225 * (size_t)cov_rows);
    const auto snap = S.add<double>(Stage::kScratch, smooth ? kTrajSnap * (size_t)rows : 0);
    const auto knot = S.add<double>(Stage::kScratch, smooth ? (size_t)n * (kMaxFrames - 1) * h->bw.Scap * 4 : 0);
    TRY(S.place(h, true));
    TRY(P.run(h, S));
    const TrajArgs T{S.dev(rec), S.dev(tm), S.dev(sto), S.dev(fro), S.dev(sco), S.dev(P.cov), S.dev(P.st), any_cov ? 1 : 0};
    if (smooth) {
        const size_t smem = traj_smooth_bytes(any_cov);
        if (smem > 48 * 1024)
            CK(h, cudaFuncSetAttribute(bw_smoothed_trajectory_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        bw_smoothed_trajectory_kernel<<<dim3(n, warps), 32, smem, h->stream>>>(launch_args<BwArgs>(h), T,
                                                                             TrajSmooth{S.dev(snap), S.dev(knot)});
        TRY(launched(h, "bw_smoothed_trajectory_kernel"));
    } else {
        const size_t smem = warps * traj_warp_bytes(any_cov);
        if (smem > 48 * 1024)
            CK(h, cudaFuncSetAttribute(bw_trajectory_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        bw_trajectory_kernel<<<n, 32 * warps, smem, h->stream>>>(launch_args<BwArgs>(h), T);
        TRY(launched(h, "bw_trajectory_kernel"));
    }
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_trajectory &R = records[i];
        const BwTraj &T = recs[i];
        const size_t nq = R.n_times;
        if (nq > 0) {
            memcpy(R.states, S.host(sto) + 16 * (size_t)T.t_off, sizeof(double) * 16 * nq);
            memcpy(R.frame, S.host(fro) + T.t_off, sizeof(int32_t) * nq);
            if (R.state_cov) memcpy(R.state_cov, S.host(sco) + 225 * (size_t)T.scov_off, sizeof(double) * 225 * nq);
        }
        R.status = T.cov >= 0 ? S.host(P.st)[T.cov] : PVIO_B200_OK;
    }
    return 0;
}


extern "C" {

int pvio_b200_batch_window_covariance(pvio_b200_handle hh, int n, pvio_b200_window_covariance *records) {
    BwCall C(hh, "batch_window_covariance");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked against its slot's host mirror before anything is staged
    CovPlan P;
    std::vector<CovLm> lms;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_covariance &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (s.N < 1) return C.bad("a window without frames");
        if (R.n_frames < 0 || R.n_frames > s.N || R.n_tracks < 0 || R.n_tracks > (int)s.ids.size())
            return C.bad("a frame or track count out of range");
        if (R.n_frames == 0 && R.n_tracks == 0) return C.bad("a record asking for nothing");
        if (R.n_frames > 0 && (!R.frames || !R.cov)) return C.bad("frames or cov missing");
        if (R.n_tracks > 0 && (!R.tracks || !R.inv_depth_var)) return C.bad("tracks or inv_depth_var missing");
        uint32_t seen = 0;
        for (int k = 0; k < R.n_frames; ++k) {
            const int f = R.frames[k];
            if (f < 0 || f >= s.N) return C.bad("a frame out of range");
            if ((seen >> f) & 1u) return C.bad("a frame named twice");
            seen |= 1u << f;
        }
        if (P.add(h, R.slot, R.n_frames, R.frames) < 0) return C.bad("reduced system too large for shared memory");
        const std::vector<int32_t> lm = R.n_tracks > 0 ? landmark_of_rows(s) : std::vector<int32_t>();
        std::vector<uint8_t> taken(s.ids.size(), 0);
        for (int k = 0; k < R.n_tracks; ++k) {
            const int r = find_row(s, R.tracks[k]);
            if (r < 0) return C.bad("a track that is not live in its slot");
            if (taken[r]) return C.bad("a track named twice");
            taken[r] = 1;
            lms.push_back(CovLm{i, R.slot, lm[r], 0});
        }
    }
    const int n_lm = (int)lms.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    P.stage(S, h, Stage::kDown);
    const auto lmv = S.up(lms);
    const auto var = S.add<double>(Stage::kDown, (size_t)n_lm);
    TRY(S.place(h, true));
    TRY(P.run(h, S, true, S.dev(lmv), n_lm, S.dev(var)));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0, t = 0; i < n; ++i) {
        pvio_b200_window_covariance &R = records[i];
        if (R.n_frames > 0) memcpy(R.cov, S.host(P.cov) + P.recs[i].cov_off, sizeof(double) * 225 * R.n_frames * R.n_frames);
        if (R.n_tracks > 0) memcpy(R.inv_depth_var, S.host(var) + t, sizeof(double) * R.n_tracks);
        t += R.n_tracks;
        R.status = S.host(P.st)[i];
    }
    return 0;
}

int pvio_b200_batch_window_landmarks(pvio_b200_handle hh, int n, pvio_b200_window_landmarks *records) {
    BwCall C(hh, "batch_window_landmarks");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked against its slot's host mirror before anything is staged; the all-tracks mode takes its rows
    // from the mirror's size, with no per-track work
    std::vector<BwLmk> recs(n);
    std::vector<int32_t> rows, cov_rec;
    CovPlan P;
    int32_t n_pts = 0, n_cov_rows = 0, max_cov_rows = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_landmarks &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        const int T = (int)s.ids.size();
        if (s.N < 1) return C.bad("a window without frames");
        if (R.n_tracks < -1 || R.n_tracks > T) return C.bad("a track count out of range");
        const bool all = R.n_tracks == -1;
        const int nr = all ? T : R.n_tracks;
        if (all && R.capacity < T) return C.bad("capacity smaller than the slot's live tracks");
        if (!all && nr > 0 && !R.tracks) return C.bad("tracks missing");
        if (nr > 0 && !R.point) return C.bad("point missing");
        if (R.inv_depth_var && !R.point_cov) return C.bad("inv_depth_var without point_cov");
        const bool cov = R.point_cov != nullptr;
        const int c = cov ? P.add(h, R.slot) : -1;
        if (cov && c < 0) return C.bad("reduced system too large for shared memory");
        BwLmk &L = recs[i];
        L = BwLmk{R.slot, nr, T, all ? -1 : (int32_t)rows.size(), n_pts, c, n_cov_rows, 0};
        if (!all) {
            std::vector<uint8_t> taken(T, 0);
            for (int k = 0; k < nr; ++k) {
                const int r = find_row(s, R.tracks[k]);
                if (r < 0) return C.bad("a track that is not live in its slot");
                if (taken[r]) return C.bad("a track named twice");
                taken[r] = 1;
                rows.push_back(r);
            }
        }
        n_pts += nr;
        if (cov) {
            cov_rec.push_back(i);
            n_cov_rows += nr;
            max_cov_rows = std::max(max_cov_rows, nr);
        }
    }
    const int n_cov = (int)cov_rec.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto rw = S.up(rows);
    const auto crc = S.up(cov_rec);
    P.stage(S, h, Stage::kScratch);
    const auto pts = S.add<double>(Stage::kDown, 3 * (size_t)n_pts);
    const auto rol = S.add<int32_t>(Stage::kDown, (size_t)n_pts);
    const auto pcov = S.add<double>(Stage::kDown, 9 * (size_t)n_cov_rows), var = S.add<double>(Stage::kDown, (size_t)n_cov_rows);
    const auto lmo = S.add<int32_t>(Stage::kScratch, (size_t)n_cov * h->Mcap);
    TRY(S.place(h, true));
    const LmkArgs L{S.dev(rec), S.dev(rw), S.dev(crc), S.dev(pts), S.dev(rol), S.dev(lmo), S.dev(P.st), S.dev(P.sxi), S.dev(pcov), S.dev(var)};
    const BwArgs a = launch_args<BwArgs>(h);
    bw_landmark_point_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L);
    TRY(launched(h, "bw_landmark_point_kernel"));
    if (n_cov > 0) {
        TRY(P.run(h, S));
        const dim3 grid(n_cov, std::max(1, (max_cov_rows + kLmkWarps - 1) / kLmkWarps));
        if (h->hs_double) bw_landmark_cov_kernel<double><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        else bw_landmark_cov_kernel<float><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        TRY(launched(h, "bw_landmark_cov_kernel"));
    }
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_landmarks &R = records[i];
        const BwLmk &L = recs[i];
        const WinSlot &s = h->slots[R.slot];
        const size_t nr = L.n_rows;
        if (nr > 0) memcpy(R.point, S.host(pts) + 3 * (size_t)L.out_off, sizeof(double) * 3 * nr);
        if (R.role && nr > 0) memcpy(R.role, S.host(rol) + L.out_off, sizeof(int32_t) * nr);
        if (R.track_id && nr > 0) {
            if (L.rows_off < 0) memcpy(R.track_id, s.ids.data(), sizeof(int32_t) * nr);
            else memcpy(R.track_id, records[i].tracks, sizeof(int32_t) * nr);
        }
        R.status = PVIO_B200_OK;
        if (L.cov >= 0) {
            if (nr > 0) memcpy(R.point_cov, S.host(pcov) + 9 * (size_t)L.cov_off, sizeof(double) * 9 * nr);
            if (R.inv_depth_var && nr > 0) memcpy(R.inv_depth_var, S.host(var) + L.cov_off, sizeof(double) * nr);
            R.status = S.host(P.st)[L.cov];
        }
        R.n_rows = (int32_t)nr;
    }
    return 0;
}

int pvio_b200_batch_window_trajectory(pvio_b200_handle hh, int n, pvio_b200_window_trajectory *records) {
    return trajectory_call(hh, n, records, false);
}

int pvio_b200_batch_window_smoothed_trajectory(pvio_b200_handle hh, int n, pvio_b200_window_trajectory *records) {
    return trajectory_call(hh, n, records, true);
}

}  // extern "C"
