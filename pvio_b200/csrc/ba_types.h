// Device-side (packed) layout of a batch of sliding windows.  See DESIGN.md "Data layout".
// Observation / landmark records are the 16-byte fp32 records SURVEY.md 8(d) counts as
// algorithmic bytes; all STATE (poses, motion, inverse depths) stays fp64 because the
// residual must be evaluated in fp64 to meet the 1e-5 relative tolerance on dx.
#pragma once
#include <stdint.h>
#include <vector_types.h>

namespace pvio {

constexpr int kMaxFrames = 16;      // PVIO_B200_MAX_FRAMES
constexpr int kFrameStride = 16;    // doubles per frame state
constexpr int kImuStride = 288;     // doubles per IMU factor record
constexpr int kMaxChunks = 96;      // anchor-homogeneous chunks of <= 32 landmarks per window
constexpr int kAcc = 16;            // doubles per window accumulated by the update / J.v sweeps
constexpr int kMaxSeg = kMaxFrames * (kMaxFrames - 1) / 2;   // (target, anchor) segments of the frame-major table
constexpr int kSegTab = 2 * (kMaxSeg + 1);                   // ints per window: seg_begin[kMaxSeg + 1], seg_row[kMaxSeg + 1]

struct __align__(8) ObsRec {        // one reprojection residual block (non-anchor observation), 8 B
    float zx, zy;                   // normalised keypoint in the target frame
};                                  // SURVEY's 16-B record also carried the landmark and frame indices: the
                                    // landmark is implied by the CSR offset in LmRec, the frame by the
                                    // landmark's frame mask (observations are stored in increasing frame
                                    // order, so record j belongs to the j-th set bit): half the bytes to move

struct __align__(16) LmRec {        // one inverse-depth landmark
    float zrx, zry;                 // normalised keypoint in the anchor frame
    int32_t meta;                   // anchor | in_victim << 4 | n_obs << 8 | target-frame mask << 16
    int32_t obs_begin;              // first ObsRec of this landmark
};
#if defined(__CUDACC__)
#define PVIO_HD __host__ __device__ __forceinline__
#else
#define PVIO_HD inline
#endif
PVIO_HD int lm_anchor(int32_t meta) { return meta & 0xf; }
PVIO_HD int lm_victim(int32_t meta) { return (meta >> 4) & 1; }
PVIO_HD int lm_nobs(int32_t meta) { return (meta >> 8) & 0x1f; }
PVIO_HD unsigned lm_mask(int32_t meta) { return (unsigned)meta >> 16; }
PVIO_HD int32_t lm_meta(int anchor, int victim, int n_obs, unsigned mask) {
    return (int32_t)((unsigned)anchor | ((unsigned)victim << 4) | ((unsigned)n_obs << 8) | (mask << 16));
}

// Frame-major observation table (built on the device from the landmark-major one, ba_fobs.cuh): the residual
// blocks sorted by (target frame t, anchor frame a, landmark), segment sp = t (t - 1) / 2 + a.  A warp of the
// linearise / update sweeps works on 32 consecutive entries of ONE segment ("row"), so the target frame is
// warp-uniform (held in registers) and the per-(t, a) direct blocks are plain register sums.  Stored as two arrays of
// the same index: fz (keypoint in the target frame, 8 B) and flm (packed landmark index, 2 B: Mcap <= 65536), 10 B
// per residual block.
typedef uint16_t FLm;

// per-landmark sums of the linearise sweep (H_ll, g_l), formed by the Schur kernel
struct LmSum { double hll, gl; };

struct WinHdr {                     // per-window integers
    int32_t N, M, K, use_inertial;
    int32_t n_imu, n_prior, n_planes, n_ptracks;
    int32_t fixed_mask;             // bit f: FF_FIX_POSE
    int32_t n_chunks;
    int32_t pad0, pad1;
    int32_t chunk_begin[kMaxChunks];   // first landmark of chunk c
    int32_t chunk_meta[kMaxChunks];    // count | anchor << 8
};

struct WinConst {                   // per-window doubles
    double cam_q[4], cam_p[3];
    double imu_q[4], imu_p[3];
    double sic[4];                  // sqrt_inv_cov 2x2
    double fx, fy, cauchy_a, plane_sic;
    double origin[3];               // window origin subtracted from all positions (mean frame position)
    double pad;
};

struct __align__(16) WinCtrl {      // per-window solver state (device resident)
    double mu, radius;
    double cost, cand_cost;         // 0.5 * sum rho(s): current / candidate
    double cost_vis, cand_cost_vis; // reprojection part accumulated by the sweeps
    double g_dot_dx, dx_reg_dx, gn_norm2, gmax, xnorm2, dxnorm2;
    double model_change;
    double grad2, v_reg_dx;         // |D^-1 S g|^2 and v^T (mu D) dx over the pose block (dogleg)
    // device-side trust-region loop (ba_tr.cuh)
    double step_a, step_b;          // step = step_b * dx_gn - step_a * v of the current iteration
    double step_norm;               // its norm in the scaled space
    double initial_cost;
    double max_time_ns, t_start_ns; // solver_options.h:30; %globaltimer at the start of the solve
    int32_t iteration, accepted, done, termination;
    int32_t solve_failed, have_scale, usable, reuse;   // reuse: the next iteration keeps linearisation and GN solve
    int32_t need_jv, skip, max_iter, fresh;            // skip: the rest of this iteration's kernels do nothing
    int32_t buf, have_lin, pad0, pad1;                 // buf: buffer set (LinBufs) holding the linearisation of the STATE;
                                                       // have_lin: it is valid for the current state and mu
};

// The linearisation of a window (records, pivots, direct blocks, reduced system, reprojection cost) lives in one of two
// buffer sets.  An iteration of the trust-region loop linearises its CANDIDATE into the other set: the cost of that
// sweep decides the step, and when the step is accepted the Jacobians of the new state are already there (WinCtrl::buf
// flips) -- the residual-only evaluation ceres does for the decision and the relinearisation that follows it are ONE
// sweep here.  Offsets of set 1 from set 0: bytes for the type-erased arrays, elements for the others.
struct LinBufs {
    size_t hs, jr, lm_w;            // bytes
    size_t lm_msk, lm_aux, Hred, Hdd, g, cost;   // elements
};

// per-landmark Schur scalars written by the linearise kernel, read by the update kernel
struct __align__(16) LmAux {
    double hll_reg;                 // H_ll + mu * clamp(.)  (the pivot the Schur complement divides by)
    double gl;                      // g_l
    double hll;                     // H_ll
    double pad;
};

// Every per-batch device array the bundle-adjustment kernels read or write, with the capacities that index them.  The
// handle keeps one copy, rebuilt whenever an array is reallocated; each kernel's argument struct derives from it and adds
// only its per-launch fields.  Arrays of [W] windows; "2x": two buffer sets, set 1 at the LinBufs offset.
struct BatchArrays {
    WinHdr *hdr;                    // [W]
    WinConst *cst;                  // [W]
    ObsRec *obs;                    // [W][Kcap] landmark-major table as the shim gathers it
    LmRec *lms;                     // [W][Mcap]
    double *rho;                    // [W][Mcap] state (overwritten by the candidate on acceptance)
    double *frames;                 // [W][Ncap][16] state
    WinCtrl *ctrl;                  // [W]
    double *lm_scale;               // [W][Mcap] Jacobi scale of each inverse depth (fixed at iteration 0)
    LmAux *lm_aux;                  // 2x [W][Mcap] H_ll + reg, g_l, H_ll of every landmark (lm_finish -> update sweep)
    void *hs;                       // 2x [W][Ncap][Mcap][6] real: UNSCALED h_lt = Y^T j of every (landmark, target)
    float2 *fz;                     // [W][Kcap] frame-major table (ba_fobs.cuh): keypoint of each residual block
    FLm *flm;                       // [W][Kcap]   and its landmark
    int32_t *seg;                   // [W][kSegTab]: seg_begin[sp], then seg_row[sp] (rows of 32 before segment sp)
    double *dx_pose;                // [W][Ncap][15] pose/motion step in delta coordinates
    double *rho_cand;               // [W][Mcap] candidate
    double *frames_cand;            // [W][Ncap][16] candidate
    double *dx_lm;                  // [W][Mcap]
    double *lm_v;                   // [W][Mcap] the same for each inverse depth (update kMode 1 -> kMode 2)
    double *acc;                    // [W][kAcc] scalars of the sweeps: 0 cand_cost_vis, 1 g.dx(lm), 2 dx.reg.dx(lm),
                                    //   3 gn_norm2(lm), 4 |step|^2(lm), 5 |x|^2(lm), 6 ambient |x - x_cand|^2 (frames),
                                    //   7 |D^-1 S g|^2 (lm), 8 v.reg.dx (lm), 9-10 |J v|^2
    int Ncap, Mcap, Kcap;           // frames / landmarks / observations per window
    int Pcap, Tcap, Ocap;           // planes / plane tracks / plane observations per window
    double *v_pose;                 // [W][Ncap][15] scaled steepest-descent direction S^2 g / clamp(S^2 diag H)
    LinBufs bufs;
    void *lm_w;                     // 2x [W][Mcap][2] real: w_l = 1 / (H_ll + reg), w_l g_l (lm_finish -> Schur kernel)
    int32_t *lm_msk;                // 2x [W][Mcap] frames of the landmark (targets | anchor), 0: not eliminated
    void *jr;                       // 2x [W][Ncap][Mcap][2] real: (j.j, j.r) of every (landmark, target) residual block;
                                    //    lm_finish sums them per landmark in frame order (deterministic, no atomics).  Only
                                    //    written when several CTAs share a window or the shared-memory sums do not fit
                                    //    (PipeArgs::lm_part)
    double *Hred;                   // 2x [W][npairs_cap][36] block-lower-triangular reduced system (xi coords)
    double *Hdd;                    // 2x [W][Ncap][36] direct (pre-Schur) diagonal blocks
    double *gdir;                   // 2x [W][Ncap][6] direct gradient
    double *gred;                   // 2x [W][Ncap][6] reduced gradient
    double *cost_vis;               // 2x [W] reprojection cost of the sweeps
    double *pose_scale;             // [W][15 Ncap]
    double *aux_cost;               // [W] non-vision (IMU + prior + plane) cost of the candidate
    // IMU and prior: allocated with the first window that has motion states
    int32_t *imu_idx;               // [W][Ncap][2] (frame_i, frame_j)
    double *imu_data;               // [W][Ncap][kImuStride]
    int32_t *prior_frames;          // [W][Ncap]
    const double *prior_S;          // [W][dcap * dcap], dcap = 15 Ncap
    const double *prior_L;          // [W][dcap * dcap] Lambda = S^T S
    const double *prior_e;          // [W][dcap]
    const double *prior_x0;         // [W][Ncap][16]
    // planes: allocated with the first window that has plane tracks
    double *plane_param;            // [W][Pcap][4]
    int32_t *pt_plane;              // [W][Tcap]
    int32_t *pt_begin;              // [W][Tcap + 1]
    int32_t *pt_frame;              // [W][Ocap]
    float *pt_z;                    // [W][Ocap][2] (observations are stored fp32 like the reprojection table)
    double *pt_J;                   // [W][Tcap][6 Ncap + 2] scratch: corrected Jacobian rows of the plane tracks
};

// One record of a covariance call (pvio_b200_batch_window_covariance, ba_cov.cuh) and one of its named tracks
struct CovRec {
    int32_t slot, n_frames, frames_off, pad;   // frames_off: ints into the call's frame list
    int64_t cov_off;                           // doubles into the call's frame blocks: (15 n_frames)^2
    int64_t sig_off;                           // doubles into the call's Sigma_delta scratch: (stride N)^2
};
struct CovLm { int32_t rec, slot, lm, pad; };  // lm: the track's landmark in the packed window, -1: none (variance NaN)

}  // namespace pvio
