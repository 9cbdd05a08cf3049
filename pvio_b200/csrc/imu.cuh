// The warp body of IMU pre-integration, PreIntegrator::integrate(t, bg, ba, true, true) / increment /
// compute_sqrt_inv_cov (pvio/src/pvio/estimation/preintegrator.cpp:39-102), shared by pvio_b200_preintegrate (imu.cu)
// and the re-integration of the resident slots' IMU factors before a solve (batch_window.cu), so both compile one piece
// of arithmetic and give bit-identical records for the same samples, t_end, biases and noise.
//
// One WARP per factor.  The sample loop is inherently serial (each increment depends on the previous
// delta); within an increment lane 0 does the O(10) small 3-vector / quaternion steps, lanes 0-26 the
// 9x9 covariance sandwich  A C A^T + B Q B^T  (3 entries each, block structure of A exploited), lanes 0-17
// the 3x3 bias-Jacobian and bias-covariance updates.  sqrt_inv_cov = LLT(cov^-1).matrixL()^T is obtained
// without inverting cov: cov = R R^T with R upper triangular (a Cholesky run from the last row up), then
// U = R^-1, which is upper triangular with positive diagonal and U^T U = cov^-1, i.e. the unique factor
// Eigen returns (preintegrator.cpp:100-102); cov is block diagonal (9 + 3 + 3) and so is U.
#pragma once
#include "ba_math.cuh"

namespace pvio {

struct ImuWarpSm {
    double C[81], T[81];      // covariance of (q, p, v) and the half product A C
    double Ri[9], Jr[9], Rd[9], M[9];      // expmap(w dt)^T, right Jacobian, delta.q, delta.q hat(a)
    double Nw[9], Na[9];      // Jr cov_w Jr^T, Rd cov_a Rd^T
    double cbg[9], cba[9];
    double dq_dbg[9], dp_dbg[9], dp_dba[9], dv_dbg[9], dv_dba[9];
    double q[4], p[3], v[3], Ra[3];
    double dt, tsum;
};

// R upper triangular with C = R R^T (n x n, row major, in place into Rm), then U = R^-1 (upper).  One thread.
static __device__ void sqrt_inv_block(const double *C, int n, int ld, double *U, int ldu) {
    double R[81];
    for (int i = 0; i < n * n; ++i) R[i] = 0.0;
    for (int j = n - 1; j >= 0; --j) {
        double d = C[j * ld + j];
        for (int k = j + 1; k < n; ++k) d -= R[j * n + k] * R[j * n + k];
        const double rjj = sqrt(d);
        R[j * n + j] = rjj;
        for (int i = 0; i < j; ++i) {
            double s = C[i * ld + j];
            for (int k = j + 1; k < n; ++k) s -= R[i * n + k] * R[j * n + k];
            R[i * n + j] = s / rjj;
        }
    }
    // U R = I, both upper triangular: U[i][j] = (delta_ij - sum_{i <= k < j} U[i][k] R[k][j]) / R[j][j]
    for (int i = 0; i < n; ++i) {
        for (int j = 0; j < n; ++j) U[i * ldu + j] = 0.0;
        for (int j = i; j < n; ++j) {
            double s = (i == j) ? 1.0 : 0.0;
            for (int k = i; k < j; ++k) s -= U[i * ldu + k] * R[k * n + j];
            U[i * ldu + j] = s / R[j * n + j];
        }
    }
}

// PreIntegrator::reset (:25-30): the warp's chain state S to the empty increment
__device__ __forceinline__ void imu_reset_warp(ImuWarpSm &S, int lane) {
    for (int i = lane; i < 81; i += 32) S.C[i] = 0.0;
    if (lane < 9) { S.cbg[lane] = 0.0; S.cba[lane] = 0.0; S.dq_dbg[lane] = 0.0; S.dp_dbg[lane] = 0.0; S.dp_dba[lane] = 0.0;
                    S.dv_dbg[lane] = 0.0; S.dv_dba[lane] = 0.0; }
    if (lane == 0) { S.q[0] = S.q[1] = S.q[2] = 0.0; S.q[3] = 1.0; S.tsum = 0.0;
                     for (int k = 0; k < 3; ++k) { S.p[k] = 0.0; S.v[k] = 0.0; } }
    __syncwarp();
}

// the warp's chain state S into D: everything imu_step_warp carries from one sample to the next
__device__ __forceinline__ void imu_copy_warp(const ImuWarpSm &S, ImuWarpSm &D, int lane) {
    for (int i = lane; i < 81; i += 32) D.C[i] = S.C[i];
    if (lane < 9) { D.cbg[lane] = S.cbg[lane]; D.cba[lane] = S.cba[lane]; D.dq_dbg[lane] = S.dq_dbg[lane];
                    D.dp_dbg[lane] = S.dp_dbg[lane]; D.dp_dba[lane] = S.dp_dba[lane]; D.dv_dbg[lane] = S.dv_dbg[lane];
                    D.dv_dba[lane] = S.dv_dba[lane]; }
    if (lane == 0) { for (int k = 0; k < 4; ++k) D.q[k] = S.q[k];
                     for (int k = 0; k < 3; ++k) { D.p[k] = S.p[k]; D.v[k] = S.v[k]; }
                     D.tsum = S.tsum; }
    __syncwarp();
}

// PreIntegrator::increment (:39-81) of one sample d ([7] t, w xyz, a xyz) over dt, on the warp's chain state S; noise
// [4][9] cov_w, cov_a, cov_bg, cov_ba.  imu_integrate_warp runs it per sample; the trajectory kernel (bw_query.cu)
// runs it on a copy of the chain to stop the integration at a query time, so both give the same bits.
__device__ __forceinline__ void imu_step_warp(ImuWarpSm &S, int lane, const double *d, double dt, const double bg[3],
                                              const double ba[3], const double *noise) {
    const double w[3] = {d[1] - bg[0], d[2] - bg[1], d[3] - bg[2]};                       // :42-43
    const double acc[3] = {d[4] - ba[0], d[5] - ba[1], d[6] - ba[2]};
    if (lane == 0) {
        const double th[3] = {w[0] * dt, w[1] * dt, w[2] * dt};
        double qi[4], qc[4], Ha[9];
        expmap(th, qi);
        quat_conj(qi, qc);
        quat_to_mat(qc, S.Ri);
        right_jacobian(th, S.Jr);
        quat_to_mat(S.q, S.Rd);
        hat(acc, Ha);
        mat3_mul(S.Rd, Ha, S.M);
        mat3_vec(S.Rd, acc, S.Ra);
        S.dt = dt;
    }
    __syncwarp();
    // noise blocks: Nw = Jr cov_w Jr^T, Na = Rd cov_a Rd^T (lanes 0-8, 9-17)
    if (lane < 18) {
        const double *X = lane < 9 ? S.Jr : S.Rd, *Q = noise + (lane < 9 ? 0 : 9);
        const int e = lane % 9, i = e / 3, j = e % 3;
        double sacc = 0.0;
        for (int k = 0; k < 3; ++k)
            for (int m = 0; m < 3; ++m) sacc += X[i * 3 + k] * Q[k * 3 + m] * X[j * 3 + m];
        (lane < 9 ? S.Nw : S.Na)[e] = sacc;
    }
    // T = A C with A = [[Ri, 0, 0], [Pq, I, dt I], [Vq, 0, I]], Vq = -dt M, Pq = -dt^2/2 M   (:46-51)
    for (int e = lane; e < 81; e += 32) {
        const int r = e / 9, c = e % 9;
        double t = 0.0;
        if (r < 3) { for (int k = 0; k < 3; ++k) t += S.Ri[r * 3 + k] * S.C[k * 9 + c]; }
        else if (r < 6) {
            for (int k = 0; k < 3; ++k) t += S.M[(r - 3) * 3 + k] * S.C[k * 9 + c];
            t = -0.5 * dt * dt * t + S.C[r * 9 + c] + dt * S.C[(r + 3) * 9 + c];
        } else {
            for (int k = 0; k < 3; ++k) t += S.M[(r - 6) * 3 + k] * S.C[k * 9 + c];
            t = -dt * t + S.C[r * 9 + c];
        }
        S.T[e] = t;
    }
    __syncwarp();
    // C = T A^T + B Q B^T   (:53-65)
    const double inv_dt = 1.0 / fmax(dt, 1.0e-7);
    for (int e = lane; e < 81; e += 32) {
        const int r = e / 9, c = e % 9;
        double t = 0.0;
        if (c < 3) { for (int k = 0; k < 3; ++k) t += S.T[r * 9 + k] * S.Ri[c * 3 + k]; }
        else if (c < 6) {
            for (int k = 0; k < 3; ++k) t += S.T[r * 9 + k] * S.M[(c - 3) * 3 + k];
            t = -0.5 * dt * dt * t + S.T[r * 9 + c] + dt * S.T[r * 9 + c + 3];
        } else {
            for (int k = 0; k < 3; ++k) t += S.T[r * 9 + k] * S.M[(c - 6) * 3 + k];
            t = -dt * t + S.T[r * 9 + c];
        }
        const int rb = r / 3, cb = c / 3, ri = r % 3, ci = c % 3;
        double nz = 0.0;
        if (rb == 0 && cb == 0) nz = dt * dt * inv_dt * S.Nw[ri * 3 + ci];
        else if (rb == 1 && cb == 1) nz = 0.25 * dt * dt * dt * dt * inv_dt * S.Na[ri * 3 + ci];
        else if (rb == 2 && cb == 2) nz = dt * dt * inv_dt * S.Na[ri * 3 + ci];
        else if (rb + cb == 3 && rb != 0 && cb != 0) nz = 0.5 * dt * dt * dt * inv_dt * S.Na[ri * 3 + ci];
        S.C[e] = t + nz;
    }
    // bias Jacobians (:71-75: dp first, then dv, then dq, each from the OLD values) and bias covariances (:66-67)
    double n_dp_dbg = 0.0, n_dp_dba = 0.0, n_dv_dbg = 0.0, n_dv_dba = 0.0, n_dq_dbg = 0.0;
    if (lane < 9) {
        const int i = lane / 3, j = lane % 3;
        double mq = 0.0, rq = 0.0;
        for (int k = 0; k < 3; ++k) { mq += S.M[i * 3 + k] * S.dq_dbg[k * 3 + j]; rq += S.Ri[i * 3 + k] * S.dq_dbg[k * 3 + j]; }
        n_dp_dbg = S.dp_dbg[lane] + dt * S.dv_dbg[lane] - 0.5 * dt * dt * mq;
        n_dp_dba = S.dp_dba[lane] + dt * S.dv_dba[lane] - 0.5 * dt * dt * S.Rd[lane];
        n_dv_dbg = S.dv_dbg[lane] - dt * mq;
        n_dv_dba = S.dv_dba[lane] - dt * S.Rd[lane];
        n_dq_dbg = rq - dt * S.Jr[lane];
        S.cbg[lane] += noise[18 + lane] * dt;
        S.cba[lane] += noise[27 + lane] * dt;
    }
    __syncwarp();
    if (lane < 9) { S.dp_dbg[lane] = n_dp_dbg; S.dp_dba[lane] = n_dp_dba; S.dv_dbg[lane] = n_dv_dbg; S.dv_dba[lane] = n_dv_dba;
                    S.dq_dbg[lane] = n_dq_dbg; }
    if (lane == 0) {                                                                      // :78-81
        S.tsum += dt;
        for (int k = 0; k < 3; ++k) {
            S.p[k] += dt * S.v[k] + 0.5 * dt * dt * S.Ra[k];
            S.v[k] += dt * S.Ra[k];
        }
        const double th[3] = {w[0] * dt, w[1] * dt, w[2] * dt};
        double qi[4], qn[4];
        expmap(th, qi);
        quat_mul(S.q, qi, qn);
        const double nrm = sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
        for (int k = 0; k < 4; ++k) S.q[k] = qn[k] / nrm;
    }
    __syncwarp();
}

// One factor on one warp (S: the warp's shared scratch); bg / ba the biases of the factor's first frame.  F describes
// the factor where the kernel keeps it: F.samples ([*][7] t, w xyz, a xyz) rows F.begin() .. F.end() - 1 (at least
// one), the last integrated up to F.t_end(); F.noise [4][9] cov_w, cov_a, cov_bg, cov_ba; F.rec() the record
// [kImuStride] (PVIO_B200_IMU_* layout).  Each is read where the arithmetic needs it.
template <typename Factor>
__device__ __forceinline__ void imu_integrate_warp(ImuWarpSm &S, int lane, const Factor &F, const double bg[3],
                                                   const double ba[3]) {
    imu_reset_warp(S, lane);
    const int b0 = F.begin(), b1 = F.end();
    for (int s = b0; s < b1; ++s) {
        const double *d = F.samples + (size_t)s * 7;
        const double t_next = (s + 1 < b1) ? F.samples[(size_t)(s + 1) * 7] : F.t_end();      // :89-92
        imu_step_warp(S, lane, d, t_next - d[0], bg, ba, F.noise);
    }
    // ---- record
    double *rec = F.rec();
    for (int i = lane; i < kImuStride; i += 32) rec[i] = 0.0;
    __syncwarp();
    if (lane == 0) {
        rec[0] = S.tsum;
        for (int k = 0; k < 4; ++k) rec[1 + k] = S.q[k];
        for (int k = 0; k < 3; ++k) { rec[5 + k] = S.p[k]; rec[8 + k] = S.v[k]; rec[281 + k] = bg[k]; rec[284 + k] = ba[k]; }
        sqrt_inv_block(S.C, 9, 9, rec + 11, 15);
    } else if (lane == 1) {
        sqrt_inv_block(S.cbg, 3, 3, rec + 11 + 9 * 15 + 9, 15);
    } else if (lane == 2) {
        sqrt_inv_block(S.cba, 3, 3, rec + 11 + 12 * 15 + 12, 15);
    }
    if (lane >= 3 && lane < 12) {
        const int e = lane - 3;
        rec[236 + e] = S.dq_dbg[e]; rec[245 + e] = S.dp_dbg[e]; rec[254 + e] = S.dp_dba[e];
        rec[263 + e] = S.dv_dbg[e]; rec[272 + e] = S.dv_dba[e];
    }
}

}  // namespace pvio
