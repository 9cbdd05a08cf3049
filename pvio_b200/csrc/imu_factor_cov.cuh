// First-order propagation of a state covariance through one IMU factor, in the coordinates of
// pvio_b200_batch_window_covariance ([dtheta dp dv dbg dba], q perturbed on the right):
//
//   Sigma = Phi Sigma_src Phi^T + Psi Sigma_d Psi^T
//
// with Phi the Jacobian of PreIntegrator::predict (preintegrator.cpp:102-109) in the source state, through the factor's
// bias Jacobians, and Psi its Jacobian in the factor's delta.  Shared by the FACTOR seed of the IMU stream slots
// (imu_stream_seed_kernel, imu_stream.cu), which forms Sigma_d from the factor's sqrt_inv_cov, and the trajectory of
// the resident slots (bw_trajectory_kernel, bw_query.cu), which takes a partial integration's delta.cov directly.
// One warp, 15 x 15 row-major matrices in shared memory.
#pragma once
#include "ba_math.cuh"

namespace pvio {

// C = A B (bt: A B^T), 15 x 15, by the warp's lanes
static __device__ void warp_mm15(const double *A, const double *B, double *C, bool bt, int lane) {
    for (int e = lane; e < 225; e += 32) {
        const int i = e / 15, j = e % 15;
        double s = 0.0;
        for (int m = 0; m < 15; ++m) s += A[i * 15 + m] * (bt ? B[j * 15 + m] : B[m * 15 + j]);
        C[e] = s;
    }
    __syncwarp();
}

// 3 x 3 block (bi, bj) of the 15 x 15 M set to s X (X row-major 3 x 3, or the identity when null)
static __device__ void put_block(double *M, int bi, int bj, const double *X, double s = 1.0) {
    for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c) M[(3 * bi + r) * 15 + 3 * bj + c] = X ? s * X[3 * r + c] : (r == c ? s : 0.0);
}

// The parts of a factor the propagation reads: its length T, delta p and delta v, and its bias Jacobians, each 3 x 3
// row-major (the PVIO_B200_IMU_* blocks of a record)
struct ImuFactorJac {
    double T;
    const double *dp, *dv, *dq_dbg, *dp_dbg, *dp_dba, *dv_dbg, *dv_dba;
};

// Phi into B (15 x 15, zeroed here): the Jacobian of PreIntegrator::predict in the source state, through the factor's
// bias Jacobians; Rs = R(q_src), dR = R(delta q)
static __device__ __forceinline__ void imu_factor_phi(double *B, const ImuFactorJac &f, const double Rs[9],
                                                      const double dR[9], int lane) {
    for (int e = lane; e < 225; e += 32) B[e] = 0.0;
    __syncwarp();
    if (lane == 0) {
        double H[9], X[9], Xt[9];
        for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 3; ++c) Xt[3 * r + c] = dR[3 * c + r];
        put_block(B, 0, 0, Xt);
        put_block(B, 0, 3, f.dq_dbg);
        hat(f.dp, H);
        mat3_mul(Rs, H, X);
        put_block(B, 1, 0, X, -1.0);
        put_block(B, 1, 1, nullptr);
        put_block(B, 1, 2, nullptr, f.T);
        mat3_mul(Rs, f.dp_dbg, X);
        put_block(B, 1, 3, X);
        mat3_mul(Rs, f.dp_dba, X);
        put_block(B, 1, 4, X);
        hat(f.dv, H);
        mat3_mul(Rs, H, X);
        put_block(B, 2, 0, X, -1.0);
        put_block(B, 2, 2, nullptr);
        mat3_mul(Rs, f.dv_dbg, X);
        put_block(B, 2, 3, X);
        mat3_mul(Rs, f.dv_dba, X);
        put_block(B, 2, 4, X);
        put_block(B, 3, 3, nullptr);
        put_block(B, 4, 4, nullptr);
    }
    __syncwarp();
}

// In: A = Sigma_src, D = Sigma_d; Rs = R(q_src), dR = R(delta q).  Out: A = Phi Sigma_src Phi^T, D = Psi Sigma_d Psi^T
// (the caller adds and symmetrises them); B and C are scratch.
static __device__ __forceinline__ void imu_factor_propagate(double *A, double *B, double *C, double *D,
                                                            const ImuFactorJac &f, const double Rs[9],
                                                            const double dR[9], int lane) {
    imu_factor_phi(B, f, Rs, dR, lane);              // Phi into B
    warp_mm15(B, A, C, false, lane);                 // Phi Sigma_src
    warp_mm15(C, B, A, true, lane);                  // .. Phi^T, into A
    if (lane == 0) {                                 // Psi into B
        for (int e = 0; e < 225; ++e) B[e] = 0.0;
        put_block(B, 0, 0, nullptr);
        put_block(B, 1, 1, Rs);
        put_block(B, 2, 2, Rs);
        put_block(B, 3, 3, nullptr);
        put_block(B, 4, 4, nullptr);
    }
    __syncwarp();
    warp_mm15(B, D, C, false, lane);                 // Psi Sigma_d
    warp_mm15(C, B, D, true, lane);                  // .. Psi^T, into D
}

}  // namespace pvio
