// Dense fp64 Cholesky solve of a window's reduced system in shared memory: the tile layout and the factorisations
// solve_kernel and solve_kernel_visual run (ba_solve.cuh), and that pvio_b200_selftest_chol runs on caller-given systems
// (selftest.cu).
#pragma once

namespace pvio {

// The dense system is stored as packed lower-triangular 4x4 TILES (tile (I,J), J <= I, at
// I(I+1)/2 + J, 16 doubles row-major) so that the factorisation works on register-sized blocks.
// A tile occupies kTP = 18 doubles: the same element of consecutive tiles then lies 4 banks apart, so a warp whose
// lanes work on consecutive tiles reads 16 bytes per lane without bank conflicts (at a pitch of 16 every lane hit the
// same four banks: the factorisation was shared-memory-bandwidth bound, 5.7 K cycles per block column at D = 135).
constexpr int kTP = 18;
__device__ __forceinline__ int tile_off(int I, int J) { return (I * (I + 1) / 2 + J) * kTP; }
__device__ __forceinline__ int tri(int i, int j) {   // element (i,j), j <= i
    return tile_off(i >> 2, j >> 2) + ((i & 3) << 2) + (j & 3);
}

#ifdef PVIO_SOLVE_STAMPS          // tuning builds of tools/ only: clock64() at the phase boundaries of solve_kernel
__device__ long long g_solve_stamps[16];
#define SOLVE_STAMP(k) do { __syncthreads(); if (threadIdx.x == 0 && blockIdx.x == 0) g_solve_stamps[k] = clock64(); } while (0)
#define CHOL_T0() long long ct__ = clock64()
#define CHOL_ACC(k) do { if (threadIdx.x == 0 && blockIdx.x == 0) { const long long n__ = clock64(); g_solve_stamps[k] += n__ - ct__; ct__ = n__; } } while (0)
#else
#define SOLVE_STAMP(k) do { } while (0)
#define CHOL_T0() do { } while (0)
#define CHOL_ACC(k) do { } while (0)
#endif


// Tiled dense Cholesky A = L L^T + solve, all threads of the CTA, fp64, in shared memory.
// nb block rows of 4 (padding rows carry an identity diagonal).  The right-hand side is block row
// nb of the packed tile array (row 0 of its tiles), so the panel / trailing phases carry out the
// forward substitution for free.  Per block column kb:
//   (b) one thread per panel tile row (incl. the rhs row): A_Ik <- A_Ik L_kk^-T;
//   (c) trailing tiles A_IJ -= A_Ik A_Jk^T: one thread per tile (kPerTile: wide CTAs, 64 FMAs from 48 loads) or per
//       tile row (narrow CTAs of the batched visual kernel);
//   (a) LOOK-AHEAD: the owner(s) of the next diagonal tile update it first and thread 0 factors it (4x4 Cholesky +
//       inverse of the factor, a serial chain of ~500 cycles) WHILE the other threads finish the trailing update.
// 2 barriers per block column.  The back substitution L^T x = y runs on warp 0 with warp-level barriers only.
// A must hold (nb+1)(nb+2)/2 tiles of kTP doubles.  Returns false (uniformly) if a pivot is
// not positive / finite (the system must be positive definite, as for ceres' Cholesky-based SPARSE_SCHUR).
// L_kk itself is not needed once its inverse is known (panel and back substitution multiply by inv(L_kk)): the inverse
// overwrites the diagonal tile, no separate array
__device__ __forceinline__ void chol_factor4(double *Akk, int *flag_sm) {
    double L[16], Li[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) { L[e] = Akk[e]; Li[e] = 0.0; }
    bool good = true;
    double idg[4];                       // reciprocals of the diagonal of L (no divisions below)
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        double d = L[c * 4 + c];
#pragma unroll
        for (int m = 0; m < c; ++m) d -= L[c * 4 + m] * L[c * 4 + m];
        if (!(d > 0.0) || !isfinite(d)) { good = false; d = 1.0; }
        const double id = rsqrt(d);
        idg[c] = id;
        L[c * 4 + c] = d * id;
#pragma unroll
        for (int r = c + 1; r < 4; ++r) {
            double v = L[r * 4 + c];
#pragma unroll
            for (int m = 0; m < c; ++m) v -= L[r * 4 + m] * L[c * 4 + m];
            L[r * 4 + c] = v * id;
        }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
        Li[c * 4 + c] = idg[c];
#pragma unroll
        for (int r = c + 1; r < 4; ++r) {
            double v = 0.0;
#pragma unroll
            for (int m = c; m < r; ++m) v -= L[r * 4 + m] * Li[m * 4 + c];
            Li[r * 4 + c] = v * idg[r];
        }
    }
#pragma unroll
    for (int e = 0; e < 16; ++e) Akk[e] = Li[e];
    if (!good) *flag_sm = 0;
}

// lower-triangle tile index e -> (ii, jj), jj <= ii
__device__ __forceinline__ void tri_unrank(int e, int &ii, int &jj) {
    ii = (int)((sqrtf(8.0f * e + 1.0f) - 1.0f) * 0.5f);
    while ((ii + 1) * (ii + 2) / 2 <= e) ++ii;
    while (ii * (ii + 1) / 2 > e) --ii;
    jj = e - ii * (ii + 1) / 2;
}

// back substitution x = L^-T y on warp 0 (y: row 0 of the rhs tiles; the diagonal tiles hold the inverse factors)
__device__ __forceinline__ void chol_back_substitute(double *A, double *x, int nb) {
    const int tid = threadIdx.x;
    const double *R = A + tile_off(nb, 0);
    if (tid < 32) {
        for (int i = tid; i < nb * 4; i += 32) x[i] = R[(i >> 2) * kTP + (i & 3)];
        __syncwarp();
        for (int kb = nb - 1; kb >= 0; --kb) {
            const double *Li = A + tile_off(kb, kb);
            double o = 0.0;
            if (tid < 4) {
#pragma unroll
                for (int m = 0; m < 4; ++m) o += (m >= tid) ? Li[m * 4 + tid] * x[kb * 4 + m] : 0.0;   // Linv^T
            }
            __syncwarp();
            if (tid < 4) x[kb * 4 + tid] = o;
            __syncwarp();
            for (int e = tid; e < kb * 4; e += 32) {
                const int J = e >> 2, c = e & 3;
                const double *X = A + tile_off(kb, J);      // tile (kb, J)
                x[e] -= X[c] * x[kb * 4] + X[4 + c] * x[kb * 4 + 1] + X[8 + c] * x[kb * 4 + 2] + X[12 + c] * x[kb * 4 + 3];
            }
            __syncwarp();
        }
    }
}

template <bool kPerTile>
__device__ inline bool chol_solve_tiled(double *A, double *x, int nb, int *flag_sm) {
    const int tid = threadIdx.x, nt = blockDim.x;
    double *R = A + tile_off(nb, 0);                       // rhs block row: tiles (nb, J), row 0 used
    for (int i = tid; i < nb * kTP; i += nt) { const int J = i / kTP, o = i - J * kTP; R[i] = (o < 4) ? x[J * 4 + o] : 0.0; }
    if (tid == 0) *flag_sm = 1;
    __syncthreads();
    if (tid == 0) chol_factor4(A + tile_off(0, 0), flag_sm);
    __syncthreads();
#ifdef PVIO_SOLVE_STAMPS
    if (tid == 0 && blockIdx.x == 0) for (int k = 10; k < 16; ++k) g_solve_stamps[k] = 0;
#endif
    CHOL_T0();
    for (int kb = 0; kb < nb; ++kb) {
        if (*flag_sm == 0) break;                      // uniform
        // (b) panel tiles incl. the rhs block row (I = nb): X <- X * Linv^T, one thread per tile ROW
        for (int e = tid; e < (nb - kb) * 4; e += nt) {
            const int I = kb + 1 + (e >> 2), r = e & 3;
            if (I == nb && r != 0) continue;           // only row 0 of the rhs tiles carries data
            double *X = A + tile_off(I, kb) + r * 4;
            const double *Li = A + tile_off(kb, kb);
            const double x0 = X[0], x1 = X[1], x2 = X[2], x3 = X[3];
            X[0] = x0 * Li[0];
            X[1] = x0 * Li[4] + x1 * Li[5];
            X[2] = x0 * Li[8] + x1 * Li[9] + x2 * Li[10];
            X[3] = x0 * Li[12] + x1 * Li[13] + x2 * Li[14] + x3 * Li[15];
        }
        CHOL_ACC(10);
        __syncthreads();
        CHOL_ACC(11);
        // (c) trailing tiles (I,J), kb < J <= I < nb, plus the rhs row (I = nb, kb < J < nb); tile 0 is the next diagonal tile
        const int n = nb - kb - 1, ntile = n * (n + 1) / 2;
        if (kPerTile) {
            for (int e = tid; e < ntile + n; e += nt) {
                int I, J;
                if (e < ntile) { int ii, jj; tri_unrank(e, ii, jj); I = kb + 1 + ii; J = kb + 1 + jj; }
                else { I = nb; J = kb + 1 + (e - ntile); }
                const double *P = A + tile_off(I, kb), *Q = A + tile_off(J, kb);
                double *C = A + tile_off(I, J);
                double q[16];
#pragma unroll
                for (int k = 0; k < 16; ++k) q[k] = Q[k];
                const int rows = (I == nb) ? 1 : 4;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (r >= rows) break;
                    const double p0 = P[r * 4], p1 = P[r * 4 + 1], p2 = P[r * 4 + 2], p3 = P[r * 4 + 3];
#pragma unroll
                    for (int c = 0; c < 4; ++c) C[r * 4 + c] -= p0 * q[c * 4] + p1 * q[c * 4 + 1] + p2 * q[c * 4 + 2] + p3 * q[c * 4 + 3];
                }
                if (e == 0) { CHOL_ACC(12); chol_factor4(C, flag_sm); CHOL_ACC(13); }     // look-ahead: tile (kb+1, kb+1) is complete
            }
        } else {
            for (int e4 = tid; e4 < (ntile + n) * 4; e4 += nt) {
                const int e = e4 >> 2, r = e4 & 3;
                int I, J;
                if (e < ntile) { int ii, jj; tri_unrank(e, ii, jj); I = kb + 1 + ii; J = kb + 1 + jj; }
                else { I = nb; J = kb + 1 + (e - ntile); }
                if (!(I == nb && r != 0)) {
                    const double *P = A + tile_off(I, kb) + r * 4, *Q = A + tile_off(J, kb);
                    double *C = A + tile_off(I, J) + r * 4;
                    const double p0 = P[0], p1 = P[1], p2 = P[2], p3 = P[3];
#pragma unroll
                    for (int c = 0; c < 4; ++c) C[c] -= p0 * Q[c * 4] + p1 * Q[c * 4 + 1] + p2 * Q[c * 4 + 2] + p3 * Q[c * 4 + 3];
                }
                if (e4 < 4 && n > 0) {                 // threads 0..3 hold the four rows of tile (kb+1, kb+1): look-ahead
                    __syncwarp(0xFu);
                    if (e4 == 0) chol_factor4(A + tile_off(kb + 1, kb + 1), flag_sm);
                }
            }
        }
        CHOL_ACC(14);
        __syncthreads();
        CHOL_ACC(15);
    }
    if (*flag_sm == 0) return false;
    // y = L^-1 b now sits in row 0 of the rhs tiles; back substitution x = L^-T y on warp 0
    chol_back_substitute(A, x, nb);
    __syncthreads();
    return true;
}

// diagonal tile C -= L L^T with L = the panel tile (J, k) of its own block row: one tile load, the lower triangle only
// (the strict upper triangle of a diagonal tile is never read: chol_factor4 uses L[r][c], c <= r)
__device__ __forceinline__ void chol_diag_update(double (&c)[16], const double *Lt) {
    const double2 *P2 = reinterpret_cast<const double2 *>(Lt);
    double q[16];
#pragma unroll
    for (int k = 0; k < 8; ++k) { const double2 v = P2[k]; q[2 * k] = v.x; q[2 * k + 1] = v.y; }
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int cc = 0; cc <= r; ++cc)
            c[r * 4 + cc] -= q[r * 4] * q[cc * 4] + q[r * 4 + 1] * q[cc * 4 + 1] + q[r * 4 + 2] * q[cc * 4 + 2] + q[r * 4 + 3] * q[cc * 4 + 3];
}

// The same factorisation with the TRAILING MATRIX IN REGISTERS and the critical path on a warp of its own (wide CTA of
// 8 warps, the inertial single window: D = 135 ... 165).  What bounded chol_solve_tiled: each block
// column is a serial chain -- update of the next diagonal tile, its 4 x 4 factorisation + inverse by ONE thread (~750
// cycles of dependent fp64 rsqrt / multiply-adds) -- and the warp that held that thread also had its share of trailing
// tiles to do before or after, so the other warps waited ~3.4 K cycles per block column at the barrier.  Here
//   warp 0        owns the DIAGONAL tiles (lane l: tiles l and l + 32), nothing else: per block column it updates the
//                 next diagonal tile, one lane factors it, then the lanes update their remaining diagonal tiles;
//   warps 1..7    own the off-diagonal tiles and the rhs row (tile e = t + s * 224 by descending column, up to kSlots
//                 per thread) IN REGISTERS for the whole factorisation: a block column costs a tile two 128-byte panel
//                 tiles read from shared memory and no write (chol_solve_tiled: 512 B per tile and step).
// Shared memory holds what others need: the inverse factor of each diagonal tile and the finished panel tiles L_Ik
// (also what the back substitution reads).  ONE barrier per block column: trailing update C -= L_Ik L_Jk^T, then the
// owners of the next column's tiles wait for warp 0 to publish the inverse factor (a shared flag, no barrier) and store
// their panel tiles X <- X L^-T.
template <int kSlots>
__device__ inline bool chol_solve_regs(double *A, double *x, int nb, int *flag_sm) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, warp = tid >> 5;
    const int ntask = nb * (nb + 1) / 2, nown = nt - 32;      // off-diagonal tiles + the rhs row
    double *R = A + tile_off(nb, 0);                       // rhs block row: tiles (nb, J), row 0 used
    for (int i = tid; i < nb * kTP; i += nt) { const int J = i / kTP, o = i - J * kTP; R[i] = (o < 4) ? x[J * 4 + o] : 0.0; }
    if (tid == 0) *flag_sm = 1;
    __syncthreads();
    int tI[kSlots], tJ[kSlots];
    double c[kSlots][16];
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
        tI[s] = -1; tJ[s] = -1;
        if (warp == 0) {
            if (s < 2 && lane + 32 * s < nb) tI[s] = tJ[s] = lane + 32 * s;
        } else {
            // columns in DESCENDING order (column J: its nb - 1 - J off-diagonal tiles, then its rhs tile): the tiles still
            // active at block column kb (J > kb) are the first ones of this order, i.e. they sit in the lowest slots of
            // all threads -- a warp executes as many tile bodies per block column as slots are still alive, not kSlots --
            // and the panel tiles of one column are neighbours (one or two warps, one slot)
            const int e = tid - 32 + s * nown;
            if (e < ntask) { int ii, jj; tri_unrank(e, ii, jj); tJ[s] = nb - 1 - ii; tI[s] = tJ[s] + 1 + jj; }
        }
        if (tI[s] >= 0) {
            const double2 *src = reinterpret_cast<const double2 *>(A + tile_off(tI[s], tJ[s]));
#pragma unroll
            for (int k = 0; k < 8; ++k) { const double2 v = src[k]; c[s][2 * k] = v.x; c[s][2 * k + 1] = v.y; }
        } else {
#pragma unroll
            for (int k = 0; k < 16; ++k) c[s][k] = 0.0;
        }
    }
    if (tid == 0) chol_factor4(A + tile_off(0, 0), flag_sm);      // tile (0, 0) is still intact in shared memory
    __syncthreads();
    // panel tile X <- X L_kk^-T of column `col` for every owned tile of that column (incl. the rhs row), into shared memory
    auto panel = [&](int col) {
        const double *Li = A + tile_off(col, col);
#pragma unroll
        for (int s = 0; s < kSlots; ++s) {
            if (tJ[s] != col) continue;                // (tI > col for every off-diagonal tile of the column)
            const int rows = (tI[s] == nb) ? 1 : 4;
            double *X = A + tile_off(tI[s], col);
            const double l0 = Li[0], l4 = Li[4], l5 = Li[5], l8 = Li[8], l9 = Li[9], l10 = Li[10], l12 = Li[12], l13 = Li[13],
                         l14 = Li[14], l15 = Li[15];
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                if (r >= rows) break;
                const double x0 = c[s][r * 4], x1 = c[s][r * 4 + 1], x2 = c[s][r * 4 + 2], x3 = c[s][r * 4 + 3];
                double2 o0, o1;
                o0.x = x0 * l0;
                o0.y = x0 * l4 + x1 * l5;
                o1.x = x0 * l8 + x1 * l9 + x2 * l10;
                o1.y = x0 * l12 + x1 * l13 + x2 * l14 + x3 * l15;
                reinterpret_cast<double2 *>(X + r * 4)[0] = o0;
                reinterpret_cast<double2 *>(X + r * 4)[1] = o1;
            }
        }
    };
    __shared__ int diag_ready_sm;                      // the last block column whose diagonal tile is factored (inverse in shared memory)
    volatile int *diag_ready = &diag_ready_sm;
    if (tid == 0) *diag_ready = 0;
    if (warp != 0) panel(0);
    __syncthreads();
    // One barrier per block column.  After it the panel tiles of column kb are in shared memory.  Warp 0 updates the next
    // diagonal tile, factors it and PUBLISHES it (diag_ready, no barrier); the other warps update their tiles with column
    // kb -- and the owners of the tiles of column kb + 1 then pick the inverse factor up as soon as it is published and
    // store their finished panel tiles, so that the next block column starts right after the barrier.
    for (int kb = 0; kb < nb; ++kb) {
        if (*flag_sm == 0) break;                      // uniform
        if (warp == 0) {
            const int sd = (kb + 1) >> 5;              // uniform: the slot of the next diagonal tile goes first
#pragma unroll
            for (int pass = 0; pass < 2; ++pass)
#pragma unroll
                for (int s = 0; s < 2; ++s) {
                    if ((pass == 0) != (s == sd)) continue;
                    if (tJ[s] > kb) chol_diag_update(c[s], A + tile_off(tJ[s], kb));
                    if (pass == 0 && tJ[s] == kb + 1) {
                        double2 *dst = reinterpret_cast<double2 *>(A + tile_off(kb + 1, kb + 1));
#pragma unroll
                        for (int k = 0; k < 8; ++k) { double2 v; v.x = c[s][2 * k]; v.y = c[s][2 * k + 1]; dst[k] = v; }
                        chol_factor4(A + tile_off(kb + 1, kb + 1), flag_sm);
                        __threadfence_block();
                        *diag_ready = kb + 1;
                    }
                }
        } else {
            // trailing update of the owned off-diagonal / rhs tiles (I, J), kb < J < I; the highest live slot first: it
            // holds the tiles of column kb + 1
            bool next_panel = false;
#pragma unroll
            for (int s = kSlots - 1; s >= 0; --s) {
                if (tJ[s] <= kb) continue;
                next_panel |= tJ[s] == kb + 1;
                const double2 *P2 = reinterpret_cast<const double2 *>(A + tile_off(tI[s], kb));
                const double2 *Q2 = reinterpret_cast<const double2 *>(A + tile_off(tJ[s], kb));
                double q[16];
#pragma unroll
                for (int k = 0; k < 8; ++k) { const double2 v = Q2[k]; q[2 * k] = v.x; q[2 * k + 1] = v.y; }
                const int rows = (tI[s] == nb) ? 1 : 4;
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    if (r >= rows) break;
                    const double2 pa = P2[2 * r], pb = P2[2 * r + 1];
#pragma unroll
                    for (int cc = 0; cc < 4; ++cc)
                        c[s][r * 4 + cc] -= pa.x * q[cc * 4] + pa.y * q[cc * 4 + 1] + pb.x * q[cc * 4 + 2] + pb.y * q[cc * 4 + 3];
                }
            }
            if (next_panel) {
                while (*diag_ready < kb + 1) { }
                __threadfence_block();
                panel(kb + 1);
            }
        }
        __syncthreads();
    }
    if (*flag_sm == 0) return false;
    // y = L^-1 b now sits in row 0 of the rhs tiles; back substitution x = L^-T y on warp 0
    chol_back_substitute(A, x, nb);
    __syncthreads();
    return true;
}

// The factorisation solve_body<kFull> runs, also called by pvio_b200_selftest_chol so that the tests judge the same
// choice.  Wide CTA (8 warps) and a system whose off-diagonal tiles fit into 4 (5) register slots per thread of warps
// 1..7, its diagonal into the 64 slots of warp 0: the register-resident factorisation; otherwise the tiled one.
template <bool kFull>
__device__ __forceinline__ bool chol_solve(double *A, double *x, int nb, int *flag_sm) {
    const int nt = blockDim.x;
    const int n_off = nb * (nb - 1) / 2 + nb;
    return (kFull && nt == 256 && nb <= 64 && n_off <= 4 * 224) ? chol_solve_regs<4>(A, x, nb, flag_sm)
         : (kFull && nt == 256 && nb <= 64 && n_off <= 5 * 224) ? chol_solve_regs<5>(A, x, nb, flag_sm)
                                                                : chol_solve_tiled<kFull>(A, x, nb, flag_sm);
}

}  // namespace pvio
