/* pvio_b200 -- C ABI of the H100-native (sm_90a) sliding-window bundle-adjustment + KLT backend.
 *
 * Drop-in boundary for ONE hot path of zju3dv/PVIO (reference paths relative to
 * /root/reference):
 *   - pvio_b200_ba_solve        replaces the ceres::Solve call in
 *                               pvio/src/pvio/estimation/bundle_adjustor.cpp:244-249
 *                               (BundleAdjustorSolver::solve :63-299; post-pass :277-296)
 *   - pvio_b200_ba_gn_step      one linearise -> Schur -> solve -> Plus -> cost iteration
 *                               (test / benchmark unit; what Ceres does once per iteration)
 *   - pvio_b200_ba_marginalize  replaces BundleAdjustor::marginalize_frame,
 *                               bundle_adjustor.cpp:348-599
 *   - pvio_b200_klt_track       replaces cv::calcOpticalFlowPyrLK in
 *                               pvio-extra/src/pvio/extra/opencv_image.cpp:103
 *                               (OpenCvImage::track_keypoints :88-136)
 *   - pvio_b200_reprojection_error  BundleAdjustor::compute_reprojection_error :321-336
 *
 * Conventions (SURVEY.md 8b): plain pointers and sizes, caller-owned arrays, the callee
 * never frees them; doubles at the boundary (the reference's state is fp64); no
 * exceptions; integer return codes (0 = ok, < 0 = error, see PVIO_B200_E*); one
 * in-flight call per handle (the reference calls solve from one thread,
 * core/frontend_worker.cpp:58-77); handles are independent across GPUs.
 * There is no CPU fallback: every entry point fails with PVIO_B200_ENODEV without a GPU.
 */
#ifndef PVIO_B200_H
#define PVIO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PVIO_B200_OK 0
#define PVIO_B200_ENODEV (-1)   /* no CUDA device / driver error            */
#define PVIO_B200_EINVAL (-2)   /* bad argument or window exceeds capacity   */
#define PVIO_B200_ENOMEM (-3)
#define PVIO_B200_ECUDA (-4)    /* kernel / runtime failure (see last_error) */
#define PVIO_B200_ENUMERIC (-5) /* reduced system not positive definite      */

#define PVIO_B200_MAX_FRAMES 16      /* N: window frames (reference: 9..11)  */
#define PVIO_B200_FRAME_STRIDE 16    /* doubles per frame: q(x,y,z,w) p v bg ba, estimation/state.h:43-69 */
#define PVIO_B200_IMU_STRIDE 288     /* doubles per IMU factor, layout below */

/* IMU factor record = the PreIntegrator outputs the cost functor reads
 * (estimation/preintegrator.h:29-44, ceres/preintegration_error_cost.h:53-76):
 *   [0] dt | [1..4] dq (x,y,z,w) | [5..7] dp | [8..10] dv |
 *   [11..235] sqrt_inv_cov 15x15 row-major |
 *   [236..244] dq_dbg | [245..253] dp_dbg | [254..262] dp_dba | [263..271] dv_dbg |
 *   [272..280] dv_dba (3x3 row-major) | [281..283] bg0 | [284..286] ba0 | [287] pad
 * bg0/ba0: the bias linearisation point (frame_i->motion at integrate() time; SURVEY quirk Q1). */
#define PVIO_B200_IMU_DT 0
#define PVIO_B200_IMU_DQ 1
#define PVIO_B200_IMU_DP 5
#define PVIO_B200_IMU_DV 8
#define PVIO_B200_IMU_SQRT_INV_COV 11
#define PVIO_B200_IMU_DQ_DBG 236
#define PVIO_B200_IMU_DP_DBG 245
#define PVIO_B200_IMU_DP_DBA 254
#define PVIO_B200_IMU_DV_DBG 263
#define PVIO_B200_IMU_DV_DBA 272
#define PVIO_B200_IMU_BG0 281
#define PVIO_B200_IMU_BA0 284

/* One sliding window, gathered by the shim from Map/Frame/Track exactly in the order
 * bundle_adjustor.cpp:75-242 walks them.  Keypoints are normalised image coordinates. */
typedef struct pvio_b200_window {
    int32_t n_frames;            /* map->frame_num()                              :75  */
    int32_t n_landmarks;         /* VALID non-PLANE tracks with a parameter block :91-103 */
    int32_t n_obs;               /* reprojection residual blocks (anchor excluded) :149 */
    int32_t use_inertial;        /* solve(map, config, use_inertial)              :63  */
    const uint8_t *frame_fixed;  /* [N] Frame::flag(FF_FIX_POSE)                  :79  */
    double cam_q_cs[4], cam_p_cs[3]; /* Frame::camera (estimation/state.h:38-41)       */
    double imu_q_cs[4], imu_p_cs[3]; /* Frame::imu                                     */
    double sqrt_inv_cov[4];      /* Frame::sqrt_inv_cov 2x2 row-major (core/core.cpp:112-116) */
    double fx, fy;               /* Frame::K(0,0), K(1,1): post-pass pixel error  :291 */
    double cauchy_a;             /* ceres::CauchyLoss(1.0)                        :58  */
    const int32_t *lm_anchor;    /* [M] index of Track::first_frame()                  */
    const double *lm_z_ref;      /* [M][2] first_keypoint()                            */
    const int32_t *lm_obs_begin; /* [M+1] CSR offsets into obs_*                       */
    const uint8_t *lm_in_victim; /* [M] track observed by the frame to marginalise :454 (may be NULL) */
    const int32_t *obs_frame;    /* [K] sorted by landmark, then frame index           */
    const double *obs_z;         /* [K][2]                                             */
    int32_t n_imu;               /* pre-integration factors                      :220-242 */
    const int32_t *imu_frame_i;  /* [n_imu]                                            */
    const int32_t *imu_frame_j;  /* [n_imu]                                            */
    const double *imu_data;      /* [n_imu][PVIO_B200_IMU_STRIDE]                      */
    int32_t n_prior;             /* frames related to the marginalisation prior  :126-139 */
    const int32_t *prior_frames; /* [n_prior] window index of each related frame       */
    const double *prior_S;       /* [(15 n)^2] row-major sqrt_inv_cov (marginalization_error_cost.h:103) */
    const double *prior_e;       /* [15 n] infovec                                     */
    const double *prior_state0;  /* [n_prior][16] pose_0 / motion_0 snapshots :44-45   */
    int32_t n_planes;            /* planes with >= 20 tracks                     :165  */
    const double *plane_param;   /* [n_planes][4] normal(3), distance                  */
    double plane_sqrt_inv_cov;   /* sqrt(1 / config->plane_distance_cov())       :181  */
    int32_t n_plane_tracks;
    const int32_t *pt_plane;     /* [T] plane index of each plane-track          :183  */
    const int32_t *pt_obs_begin; /* [T+1] CSR offsets                                  */
    const int32_t *pt_obs_frame; /* [...] every observation of the track         :186  */
    const double *pt_obs_z;      /* [...][2]                                           */
} pvio_b200_window;

/* In/out state: Frame::pose, Frame::motion, Track::landmark.inv_depth -- overwritten in
 * place as ceres does (bundle_adjustor.cpp:77-101). */
typedef struct pvio_b200_state {
    double *frames;    /* [N][PVIO_B200_FRAME_STRIDE] */
    double *inv_depth; /* [M] */
} pvio_b200_state;

typedef struct pvio_b200_options {
    int32_t max_iterations; /* config->solver_iteration_limit() (10)   solver_options.h:29 */
    double max_time;        /* config->solver_time_limit() seconds     solver_options.h:30 */
    int32_t alias_bias;     /* 1: bias linearisation point follows the accepted state (quirk Q1,
                               the reference's behaviour); 0: frozen at solve entry          */
    int32_t run_postpass;   /* 1: run the landmark depth / pixel-error pass :277-296         */
    double initial_trust_region_radius; /* 0: ceres default 1e4 (PVIO does not override it);
                               other values exist to exercise the dogleg legs in tests         */
} pvio_b200_options;

#define PVIO_B200_TERM_CONVERGENCE 0
#define PVIO_B200_TERM_NO_CONVERGENCE 1
#define PVIO_B200_TERM_FAILURE 2

typedef struct pvio_b200_summary {
    int32_t iterations;      /* trust-region iterations executed                          */
    int32_t accepted_steps;
    int32_t termination;     /* PVIO_B200_TERM_*                                          */
    int32_t usable;          /* ceres Summary::IsSolutionUsable()                   :298  */
    double initial_cost, final_cost;
    double final_radius, final_mu;
    double solve_seconds;    /* device time of the solve (CUDA events)                    */
} pvio_b200_summary;

typedef struct pvio_b200_handle_s *pvio_b200_handle;

/* ---- lifetime ---------------------------------------------------------------------- */
/* Owns device buffers, one stream, CUDA graphs.  max_windows > 1 enables the batched
 * entry points (BASELINE config 5 and the roofline launch). */
int pvio_b200_create(int device, int max_windows, int max_frames, int max_landmarks,
                     int max_obs, pvio_b200_handle *out);
void pvio_b200_destroy(pvio_b200_handle h);
const char *pvio_b200_last_error(pvio_b200_handle h);
/* number of kernels this library launched since creation (bench.py "gpu_launches") */
int64_t pvio_b200_kernel_launches(pvio_b200_handle h);
const char *pvio_b200_version(void);

/* ---- single window: the reference-facing calls ------------------------------------- */
/* Full solve; state updated in place.  valid/quality ([M], may be NULL) receive the
 * post-pass result (TF_VALID after the depth test, landmark.quality). */
int pvio_b200_ba_solve(pvio_b200_handle h, const pvio_b200_window *w, pvio_b200_state *s,
                       const pvio_b200_options *opt, pvio_b200_summary *summary,
                       uint8_t *valid, double *quality);

/* One regularised Gauss-Newton iteration at `s` (not modified): dx = -(H + mu D)^-1 g in
 * the local coordinates [N][15] then [M] (theta, p, v, bg, ba per frame; d inv_depth per
 * landmark; masked coordinates are 0), the cost at s, and the cost after Plus(s, dx).
 * Hred/gred (may be NULL) receive the reduced system in the same [N][15] layout
 * (row-major D x D, D = 15 N). */
int pvio_b200_ba_gn_step(pvio_b200_handle h, const pvio_b200_window *w, const pvio_b200_state *s,
                         double mu, double *dx, double *cost, double *new_cost,
                         double *Hred, double *gred);

/* New prior over the remaining frames after marginalising frame `index`:
 * S_out [(15(N-1))^2] row-major, e_out [15(N-1)]; H_out/b_out (may be NULL) the
 * information matrix / vector before the eigen factorisation. */
int pvio_b200_ba_marginalize(pvio_b200_handle h, const pvio_b200_window *w, const pvio_b200_state *s,
                             int index, double *S_out, double *e_out, double *H_out, double *b_out);

/* ---- resident sliding window (SURVEY 8(f) rank 1) ----------------------------------- */
/* The window persists in the handle between keyframes instead of being rebuilt from Map / Frame / Track at every
 * solve (bundle_adjustor.cpp:75-242): the shim reports what CHANGED.  The whole window stays ON THE DEVICE, the
 * marginalisation prior included: pvio_b200_window_drop_victim leaves S, e and the linearisation point where the solve
 * kernels read them.  One resident window per handle.  Frame arguments are window indices (0 = oldest).
 * These calls are the resident batched windows below, on slot 0 (each edit call is one pvio_b200_batch_window_edit),
 * so their rules apply:
 *  - pvio_b200_window_* and pvio_b200_batch_window_* on slot 0 are the same window.  A call that packs slot 0 ends it
 *    (ba_solve, ba_gn_step, ba_marginalize, reprojection_error, batch_set_window(0)); then these calls return
 *    PVIO_B200_EINVAL until pvio_b200_window_reset.
 *  - The slot limits apply: live one-observation tracks count toward max_landmarks, a landmark has fewer than 16
 *    observations, a window at most 96 landmark chunks.
 *  - A rejected call changes nothing.
 *  - A prior on a window without motion states (use_inertial == 0) is rejected.
 * Every other call before pvio_b200_window_reset returns PVIO_B200_EINVAL.  Track ids count from 0 per reset and are never
 * reused. */
/* Start an empty window.  Of `constants` the scalar members are kept (extrinsics, sqrt_inv_cov, fx, fy, cauchy_a,
 * use_inertial); its arrays and plane counts are ignored. */
int pvio_b200_window_reset(pvio_b200_handle h, const pvio_b200_window *constants);
/* sliding_window_tracker.cpp:113-118.  state [PVIO_B200_FRAME_STRIDE]; imu_record [PVIO_B200_IMU_STRIDE]: the
 * pre-integration factor (previous frame, this frame), NULL for the first frame / a visual-only window. */
int pvio_b200_window_append_frame(pvio_b200_handle h, const double *state, int fixed, const double *imu_record);
/* New tracks, each with its first observation z [n][2] in frame[i] and an initial inverse depth (the shim's
 * triangulation, track.cpp:83-106).  ids_out [n] (may be NULL): handles for the calls below. */
int pvio_b200_window_add_tracks(pvio_b200_handle h, int n, const int32_t *frame, const double *z,
                                const double *inv_depth, int32_t *ids_out);
/* Track::add_keypoint (track.cpp:32-37): observations arrive in increasing frame order per track. */
int pvio_b200_window_add_observations(pvio_b200_handle h, int n, const int32_t *track, const int32_t *frame, const double *z);
/* Map::prune_tracks.  Removing a track that is already gone returns 0; an id never handed out, PVIO_B200_EINVAL. */
int pvio_b200_window_remove_track(pvio_b200_handle h, int32_t track);
/* A prior given by the caller over frames 0 .. n_prior-1 (the 1e15 gauge prior of the first window,
 * sliding_window_tracker.cpp:100-112); later priors come from pvio_b200_window_drop_victim. */
int pvio_b200_window_set_prior(pvio_b200_handle h, int n_prior, const double *S, const double *e, const double *state0);
/* BundleAdjustor::solve on the resident window (tracks with >= 2 observations take part); states and inverse
 * depths are updated in the handle.  No landmark post-pass runs. */
int pvio_b200_window_solve(pvio_b200_handle h, const pvio_b200_options *opt, pvio_b200_summary *summary);
/* Map::marginalize_frame(0) (map.cpp:76-88): marginaliser -> new prior (device resident), the victim's observations
 * leave their tracks, tracks anchored in it are re-anchored from the current estimate (track.cpp:42-49). */
int pvio_b200_window_drop_victim(pvio_b200_handle h);
/* Read back: frames [n_frames][PVIO_B200_FRAME_STRIDE]; per queried track its inverse depth, anchor frame and
 * observation count.  A gone track reports anchor -1 and 0 observations, and its inverse depth is not written; an id
 * never handed out is PVIO_B200_EINVAL.  Any output pointer may be NULL.  With frames == NULL and n_tracks == 0 the
 * call answers n_frames without touching the device. */
int pvio_b200_window_get(pvio_b200_handle h, int32_t *n_frames, double *frames, int n_tracks, const int32_t *tracks,
                         double *inv_depth, int32_t *anchor_frame, int32_t *n_observations);

/* Mean pixel reprojection error over all observations of the window's landmarks. */
int pvio_b200_reprojection_error(pvio_b200_handle h, const pvio_b200_window *w,
                                 const pvio_b200_state *s, double *error);

/* ---- batched windows (independent problems, one CTA-group each) --------------------- */
/* Pack window `slot` (0 <= slot < max_windows) into the pinned staging area in device
 * layout (fp32 observation table, fp64 state).  Nothing is copied to the GPU yet. */
int pvio_b200_batch_set_window(pvio_b200_handle h, int slot, const pvio_b200_window *w,
                               const pvio_b200_state *s);
/* Replicate slot 0 into slots 1..n-1 (synthetic batches of identical shape). */
int pvio_b200_batch_replicate(pvio_b200_handle h, int n);
/* Host -> device copy of the first n packed windows (async on the handle's stream). */
int pvio_b200_batch_upload(pvio_b200_handle h, int n);
/* One GN iteration for the first n windows, device-resident; apply != 0 keeps the
 * updated state on the device (as an accepted step). */
int pvio_b200_batch_gn_step(pvio_b200_handle h, int n, double mu, int apply);
/* Device -> host: dx [n][15 N + M] (stride dx_stride doubles), costs [n][2]. */
int pvio_b200_batch_download(pvio_b200_handle h, int n, double *dx, int64_t dx_stride, double *costs);
/* upload + gn_step + download in one call: the end-to-end path bench.py times. */
int pvio_b200_batch_gn_step_host(pvio_b200_handle h, int n, double mu, double *dx,
                                 int64_t dx_stride, double *costs);
/* Full trust-region solve (ceres::Solve semantics per window: dogleg, per-window termination, at most
 * opt->max_iterations iterations) of the first n uploaded windows, entirely on the device: no host round trip per
 * iteration.  The device-resident states are overwritten with the solutions (BASELINE config 5: independent windows). */
int pvio_b200_batch_solve(pvio_b200_handle h, int n, const pvio_b200_options *opt);
/* Device -> host: solved states frames [n][frames_stride] (16 doubles per frame), inv_depth [n][inv_depth_stride] in
 * the caller's landmark order, one summary per window (solve_seconds is not filled).  Any pointer may be NULL. */
int pvio_b200_batch_download_state(pvio_b200_handle h, int n, double *frames, int64_t frames_stride, double *inv_depth,
                                   int64_t inv_depth_stride, pvio_b200_summary *summaries);
/* upload + batch_solve + download_state in one call with HOST buffers, pipelined over sub-batches: one host -> device
 * copy buys up to max_iterations iterations per window. */
int pvio_b200_batch_solve_host(pvio_b200_handle h, int n, const pvio_b200_options *opt, double *frames, int64_t frames_stride,
                               double *inv_depth, int64_t inv_depth_stride, pvio_b200_summary *summaries);
/* BundleAdjustor::marginalize_frame(map, 0) (bundle_adjustor.cpp:348-599) for each of the first n uploaded windows, at
 * their device-resident states (e.g. right after pvio_b200_batch_solve).  Every window must carry motion states, have
 * N >= 2 and 15 (N - 1) <= 165.  The victim's landmarks are the ones flagged lm_in_victim when the slot was packed.
 * The new prior of window i (S_i, e_i over its frames 1 .. N_i - 1, linearised at those frames' current states) is
 * written into slot i's prior arrays on the device.  A later pvio_b200_batch_set_window(i, w', ...) of the shifted
 * window with w'.prior_S == NULL and w'.n_prior == N_i - 1 names that prior, and it is not uploaded again; until the
 * slot is packed and uploaded again, its old window is not to be solved.  The device states are not modified.
 * S_out [n][S_stride] (row-major dk_i x dk_i at the start of each row, dk_i = 15 (N_i - 1)) and e_out [n][e_stride]
 * may be NULL.  Every window is checked before anything runs: on PVIO_B200_EINVAL no slot has changed. */
int pvio_b200_batch_marginalize(pvio_b200_handle h, int n, double *S_out, int64_t S_stride,
                                double *e_out, int64_t e_stride);

/* ---- resident batched windows: many sequences' sliding windows kept on the device --------------------------------- */
/* A slot made resident by pvio_b200_batch_window_reset holds its sequence's whole window on the device between camera
 * frames: frame states, IMU records, the prior and every live track (frame mask, fp64 keypoint per frame, inverse depth).
 * The caller sends only what changed; the packed tables the solve kernels read are rebuilt on the device exactly as
 * pvio_b200_batch_set_window would pack the window of the tracks with >= 2 observations, in id order, stably sorted by
 * anchor.  Frame arguments are window indices (0 = oldest).  Slot 0 is also the window of pvio_b200_window_*.
 * Rules:
 *  - Every call checks all its inputs before it stages or launches anything: on PVIO_B200_EINVAL no slot has changed.
 *    Rejected: a slot out of range or not resident, a slot named twice, an unknown or dead track, observations out of
 *    frame order, more than max_frames frames, more live tracks than max_landmarks (rounded up to a multiple of 4; one-
 *    observation tracks count), more than max_obs observations, a landmark with 16 or more observations, more than 96
 *    landmark chunks, a drop on a window without motion states or with 15 (N - 1) > 165.
 *  - Track ids are per slot, increasing, never reused until the slot is reset; the storage of dead tracks is reused, so a
 *    sequence is limited by its live tracks only.
 *  - A resident slot changes through these calls (and, for slot 0, pvio_b200_window_*) only.
 *    pvio_b200_batch_set_window on it, and any single-window call that packs into slot 0 (ba_solve, ba_gn_step,
 *    ba_marginalize, reprojection_error), end its residency; then these calls return PVIO_B200_EINVAL for it until it
 *    is reset.  batch_upload, batch_replicate, batch_gn_step,
 *    batch_solve, batch_marginalize and the *_host calls over a range holding a resident slot return PVIO_B200_EINVAL.
 *  - The kernel-launch count of a call does not depend on n.  An edit call makes one host -> device and one
 *    device -> host copy. */
/* Start an empty resident window in `slot`.  Of `constants` the scalar members are kept (as pvio_b200_window_reset),
 * plane_sqrt_inv_cov among them; n_planes > 0 is rejected (planes arrive through pvio_b200_batch_window_set_planes). */
int pvio_b200_batch_window_reset(pvio_b200_handle h, int slot, const pvio_b200_window *constants);
/* A prior given by the caller over frames 0 .. n_prior-1 (the 1e15 gauge prior of the first window,
 * sliding_window_tracker.cpp:100-112).  S [(15 n_prior)^2] row-major, e [15 n_prior], state0 [n_prior][16]. */
int pvio_b200_batch_window_set_prior(pvio_b200_handle h, int slot, int n_prior, const double *S, const double *e,
                                     const double *state0);
/* One camera frame of one sequence, applied in this order:
 *  1. replace_last: drop the newest frame, its IMU factor and its observations (map->erase_frame(frame_num - 1));
 *     a track left without observations dies;
 *  2. state != NULL: a new frame (state [16], fixed), imu_record [PVIO_B200_IMU_STRIDE] the factor (previous frame,
 *     new frame), NULL for the first frame or a visual-only window;
 *  3. new tracks: first frame, keypoint z [n][2] and initial inverse depth; their ids go to new_ids (may be NULL);
 *  4. observations (track id, frame, z [n][2]) in increasing frame order per track;
 *  5. track removals (Map::prune_tracks). */
typedef struct pvio_b200_window_edit {
    int32_t slot;
    int32_t replace_last;
    const double *state;
    int32_t fixed;
    const double *imu_record;
    int32_t n_new_tracks;
    const int32_t *new_frame;
    const double *new_z;
    const double *new_inv_depth;
    int32_t *new_ids;
    int32_t n_obs;
    const int32_t *obs_track;
    const int32_t *obs_frame;
    const double *obs_z;
    int32_t n_remove;
    const int32_t *remove;
} pvio_b200_window_edit;           /* 120 bytes on LP64 */
/* n edits, each naming a different resident slot. */
int pvio_b200_batch_window_edit(pvio_b200_handle h, int n, const pvio_b200_window_edit *edits);
/* Plane factors of a resident slot (bundle_adjustor.cpp:162-196).  Every live track has a role, -1 for a new track:
 *  -1      a landmark (TF_VALID, not TF_PLANE): inverse-depth landmark with >= 2 observations, in the marginaliser's
 *          victim set when anchored in frame 0;
 *  -2      a landmark that is TF_PLANE on a plane with fewer than 20 tracks: solved like -1, never in the victim set;
 *  p >= 0  a plane track of plane p (landmark.plane_id of a plane with >= 20 tracks): one plane-distance factor over all
 *          its window observations, anchor included; no inverse depth is solved, never in the victim set.
 * A record replaces the slot's planes (n_planes 0 .. 4, plane_param [n_planes][4]: normal, distance) unless n_planes is
 * -1, then sets the role of n_set live tracks, and their inverse depth in their anchor frame where inv_depth (may be
 * NULL) is not NaN.  Rejected: a plane count outside -1 .. 4, non-finite plane parameters, an unknown or dead track, a
 * track named twice, a role other than -1, -2 or a plane index below the slot's plane count after the record, an
 * infinite inverse depth, and a track left with a role of a plane the record removes.  Edits, drops and resets keep the
 * role of every track that stays; a reset clears the planes and the roles.  One host -> device copy; the named slots
 * are re-laid out. */
typedef struct pvio_b200_window_planes {
    int32_t slot;
    int32_t n_planes;                 /* -1: keep the slot's planes; 0 .. 4: replace them */
    const double *plane_param;        /* [n_planes][4] normal, distance */
    int32_t n_set;
    const int32_t *track;             /* [n_set] live track ids of the slot */
    const int32_t *role;              /* [n_set] -1, -2 or a plane index below the slot's plane count after this record */
    const double *inv_depth;          /* [n_set] or NULL: new inverse depth in the track's anchor frame, NaN = keep */
} pvio_b200_window_planes;            /* 48 bytes on LP64 */
/* n records, each naming a different resident slot. */
int pvio_b200_batch_window_set_planes(pvio_b200_handle h, int n, const pvio_b200_window_planes *records);
/* BundleAdjustor::solve on the named slots: the trust-region chain of pvio_b200_batch_solve (per-window termination),
 * then the landmark post-pass (unless opt->run_postpass == 0); solved states and inverse depths stay in the slots and the
 * post-pass flags in the tracks.  Slots not named keep their windows bit for bit and run no iteration (their solver
 * records are marked finished).  summaries [n] (may be NULL), in the order of `slots`. */
int pvio_b200_batch_window_solve(pvio_b200_handle h, int n, const int32_t *slots, const pvio_b200_options *opt,
                                 pvio_b200_summary *summaries);
/* Map::marginalize_frame(0) on the named slots: the marginaliser of pvio_b200_batch_marginalize with the new prior
 * left in the slot, then the victim leaves: a track anchored in it is re-anchored in its next frame from the current
 * states (track.cpp:42-49), its observations leave their tracks, frames, IMU factors and fixed flags shift by one.
 * S_out [n][S_stride], e_out [n][e_stride] (may be NULL): the new priors, as pvio_b200_batch_marginalize returns them. */
int pvio_b200_batch_window_drop_victim(pvio_b200_handle h, int n, const int32_t *slots, double *S_out, int64_t S_stride,
                                       double *e_out, int64_t e_stride);
/* The covariance of each named slot's window at its current state (after a solve: the solved state) with its IMU records
 * as they stand: the inverse of H = J^T J of every residual block the solve adds (prior; reprojection and plane blocks
 * with the Cauchy corrector; IMU), in the solve's local coordinates, without the trust-region regulariser, over the free
 * coordinates of the solve.  The landmarks are eliminated exactly; the gauge is the window's own (its prior).
 *  - cov: the joint covariance of the named frames, 15 coordinates per frame [dtheta dp dv dbg dba], in the order named;
 *    0 in the rows and columns a frame does not have (the pose of a FF_FIX_POSE frame, v / bg / ba of a visual-only
 *    window).
 *  - inv_depth_var: Var(rho) of each named track; NaN for a plane track or a track with one observation.
 *  - status: PVIO_B200_OK, or PVIO_B200_ENUMERIC when the scaled H over the free frame coordinates is not positive
 *    definite; then every output of the record is NaN, and the call still succeeds.
 * Rejected (PVIO_B200_EINVAL, no output changed): a slot out of range, not resident, named twice or without frames; a
 * frame out of range or named twice; an unknown or repeated track; a missing array; a record asking for nothing.  The
 * call changes no slot; it makes one host -> device copy, four kernel launches whatever n is, one device -> host copy and
 * one synchronisation. */
typedef struct pvio_b200_window_covariance {
    int32_t slot;
    int32_t n_frames;         /* 0 .. N frames, window indices, distinct                      */
    const int32_t *frames;
    double *cov;              /* [(15 n_frames)^2] row-major, frames in the order named       */
    int32_t n_tracks;         /* 0 .. live tracks                                             */
    const int32_t *tracks;    /* live track ids of the slot, distinct                         */
    double *inv_depth_var;    /* [n_tracks]                                                   */
    int32_t status;           /* out: PVIO_B200_OK or PVIO_B200_ENUMERIC                      */
} pvio_b200_window_covariance; /* 56 bytes on LP64 */
int pvio_b200_batch_window_covariance(pvio_b200_handle h, int n, pvio_b200_window_covariance *records);
/* The map of each named slot at its current state: per row (a named track, or every live track in id order) its id,
 * its world point Track::get_landmark_point() -- the anchor (lowest) frame's camera pose applied to [z_anchor; 1] / rho,
 * a plane track at the inverse depth set_planes gave it -- its role (-1, -2 or the plane index), and optionally the
 * point's 3 x 3 covariance and the track's Var(rho): the covariance of pvio_b200_batch_window_covariance (the anchor
 * frame's pose, rho and their cross-covariance, which that call does not return) propagated to first order through
 * Track::get_landmark_point().
 *  - point_cov / inv_depth_var: for the rows the solve treats as landmarks (role < 0, >= 2 observations); NaN for a
 *    plane track or a track with one observation.  inv_depth_var equals pvio_b200_batch_window_covariance's bit for
 *    bit.  point_cov NULL: no covariance and no covariance launches for the record (inv_depth_var must be NULL too).
 *  - status: PVIO_B200_OK, or PVIO_B200_ENUMERIC when the slot's scaled H is not positive definite (as the covariance
 *    call defines it): then every point_cov and inv_depth_var of the record is NaN; the points are still written.
 * Rejected (PVIO_B200_EINVAL, no output changed): a slot out of range, not resident, named twice or without frames; a
 * track count below -1 or above the live tracks; an unknown or repeated track; a capacity smaller than the slot's live
 * tracks (n_tracks == -1); a missing array.  The call changes no slot.  Points only: one host -> device copy, one kernel
 * launch, one device -> host copy and one synchronisation; with covariances four launches more (the covariance call's
 * linearise and Schur sweeps and cov_kernel over the slots that ask, and a landmark kernel), whatever n is.  With
 * n_tracks == -1 the host does no per-track work: the rows are those of the slot's mirror. */
typedef struct pvio_b200_window_landmarks {
    int32_t slot;
    int32_t n_tracks;         /* -1: every live track of the slot in id order; else 0 .. live tracks, named below     */
    const int32_t *tracks;    /* [n_tracks] live track ids of the slot, distinct (ignored when n_tracks == -1)        */
    int32_t capacity;         /* rows the outputs hold when n_tracks == -1                                             */
    int32_t *track_id;        /* out [rows] (may be NULL)                                                              */
    double *point;            /* out [rows][3] world point                                                             */
    int32_t *role;            /* out [rows] -1, -2 or the plane index (may be NULL); int32_t like the roles
                                 pvio_b200_window_planes takes                                                        */
    double *point_cov;        /* out [rows][9] row-major, or NULL: no covariance                                       */
    double *inv_depth_var;    /* out [rows] (may be NULL)                                                              */
    int32_t n_rows;           /* out: rows written                                                                     */
    int32_t status;           /* out: PVIO_B200_OK or PVIO_B200_ENUMERIC                                               */
} pvio_b200_window_landmarks; /* 72 bytes on LP64 */
int pvio_b200_batch_window_landmarks(pvio_b200_handle h, int n, pvio_b200_window_landmarks *records);
/* The state of each named inertial slot at any times inside its window, from the solved frames and the IMU samples its
 * factors keep on the device (pvio_b200_batch_window_set_imu, track_camera / mirror_frame with keep_samples).  Factor k
 * couples window frames k and k + 1; its samples s_0 .. s_{m-1} start at frame k's time (or up to 1e-5 s after it) and
 * its t_end is frame k + 1's time.
 *  - A time t is taken by the largest k whose factor holds samples and whose s_0.t <= t, when t <= that factor's t_end
 *    or factor k + 1 holds samples too (the last increment then runs past t_end, over the gap before s_0 of k + 1).
 *    Then  x(t) = PreIntegrator::predict(frame k's current state, delta),  delta = PreIntegrator::integrate(t, bg_k,
 *    ba_k) over the factor's samples at or before t (the last one up to t), at frame k's current biases: the arithmetic
 *    of pvio_b200_preintegrate and of the re-integration before a solve.  At t = s_0.t the state is frame k's, bit for
 *    bit; at t = t_end, delta is the factor's full re-integration.
 *  - This is a forward propagation from the preceding frame, not an interpolation between frames k and k + 1: at frame
 *    k + 1 the trajectory jumps by the factor's residual at the solution.
 *  - frame: the window frame k used; -1 for a time no factor with samples covers (before the first sample, past a
 *    factor's t_end, over a factor without samples, after the newest frame: pvio_b200_batch_imu_stream_predict's
 *    job).  Such a row has a zero state and a NaN covariance; it is not a rejection.
 *  - state_cov (NULL: no covariance launches): Phi Sigma_k Phi^T + Psi Sigma_delta(t) Psi^T in the coordinates of
 *    pvio_b200_batch_window_covariance ([dtheta dp dv dbg dba], q perturbed on the right), Sigma_k frame k's marginal
 *    covariance as that call defines it, Phi and Psi those of pvio_b200_batch_imu_stream_set_covariance's FACTOR seed,
 *    Sigma_delta(t) the partial integration's covariance itself; exactly symmetric.  status: PVIO_B200_ENUMERIC when the
 *    slot's scaled H is not positive definite, with every covariance of the record NaN (the states are still written).
 * Rejected (PVIO_B200_EINVAL, no output changed): n < 0; a slot out of range, not resident, visual-only or named twice;
 * n_times < 0; times, states or frame NULL when n_times > 0; a time that is not finite or that decreases.  The call
 * changes no slot.  Whatever n is: one host -> device copy, one kernel launch, one device -> host copy and one
 * synchronisation; with covariances three launches more (the covariance call's linearise and Schur sweeps and
 * cov_kernel over the records that ask for one). */
typedef struct pvio_b200_window_trajectory {
    int32_t slot;             /* resident inertial slot                                       */
    int32_t n_times;          /* >= 0                                                         */
    const double *times;      /* [n_times] finite, non-decreasing                             */
    double *states;           /* out [n_times][16] q xyzw, p, v, bg, ba                       */
    double *state_cov;        /* out [n_times][225] or NULL: no covariance launches           */
    int32_t *frame;           /* out [n_times]: the window frame k used, -1: t not covered    */
    int32_t status;           /* out: PVIO_B200_OK or PVIO_B200_ENUMERIC                      */
    int32_t pad;
} pvio_b200_window_trajectory; /* 48 bytes on LP64 */
int pvio_b200_batch_window_trajectory(pvio_b200_handle h, int n, pvio_b200_window_trajectory *records);
/* The smoothed state of each named inertial slot at any times inside its window: each state conditioned on both solved
 * frames around it, so that the trajectory meets frame k + 1 instead of jumping there.  The records, the factor each
 * time is taken by, the rejections, the ENUMERIC rule and "frame -1" are exactly those of
 * pvio_b200_batch_window_trajectory; the call changes no slot.  For a time t that factor k takes (frames k, k + 1,
 * samples s_0 .. s_{m-1}, t_end = frame k + 1's time), at frame k's current biases:
 *  - Delta(t), Sigma(t): the forward call's partial increment and its covariance, block-diagonal C(t) (9 x 9, [dtheta
 *    dp dv], rotation perturbed on the right), cbg(t), cba(t); e(t) its 15-dimensional error [dtheta dp dv | dbg dba].
 *    Delta(T), Sigma(T): the whole factor's re-integration, which the forward call reaches at t_end.
 *  - Phi(t2, t1): the transition of e along the chain, the product of the per-sample 9 x 9 A = [[exp(w dt)^T, 0, 0],
 *    [-dt^2/2 R hat(a), I, dt I], [-dt R hat(a), 0, I]] that pre-integration applies to C (R the chain's rotation at
 *    the step's start), the identity on the bias blocks.  From a t inside sample j's interval the chain runs the rest
 *    of sample j over [t, s_{j+1}] (or [t, t_end]), from the partial increment's rotation, then the whole samples.
 *  - Delta*: the increment PreIntegrator::predict maps from frame k onto frame k + 1 exactly, T = Delta(T)'s dt:
 *    q_k^-1 q_{k+1};  R_k^T (p_{k+1} - p_k - v_k T - g T^2 / 2);  R_k^T (v_{k+1} - v_k - g T);  b_{k+1} - b_k.
 *    r = Delta* (-) Delta(T) (15): r_theta = log(Delta_q(T)^-1 Delta*_q), the other parts differences.
 *  - Cov(e(t), e(T)) = Sigma(t) Phi(T, t)^T for t <= t_end; in the gap past t_end (<= 1e-5 s, which the forward rules
 *    give to factor k) Phi(t, T) Sigma(T), Phi(t, T) the last sample's step from t_end on to t.
 *  - K(t) = Cov(e(t), e(T)) Sigma(T)^-1;  Delta_s(t) = Delta(t) (+) K r (rotation on the right, the rest added);
 *    x_s(t) = PreIntegrator::predict(frame k, Delta_s(t)) with the bias part of K r added to frame k's biases (the
 *    Brownian bridge between b_k and b_{k+1}).
 *  - At t = s_0.t the state is frame k's, bit for bit; at t = t_end it is frame k + 1's to rounding; when r = 0 it is
 *    the forward state.
 *  - state_cov: J Sigma_{k,k+1} J^T + Psi Sigma_c(t) Psi^T, exactly symmetric, in the coordinates of
 *    pvio_b200_batch_window_covariance.  Sigma_{k,k+1} is the 30 x 30 joint covariance of frames k and k + 1 as that
 *    call defines it; Sigma_c(t) = Sigma(t) - K(t) Cov(e(T), e(t)); J = [dx_s/dx_k, dx_s/dx_{k+1}] to first order with
 *    K(t) held fixed and Delta(t), Delta(T) moving with frame k's biases through their bias Jacobians:
 *    Phi + Psi G K dr/dx_k and Psi G K dr/dx_{k+1}, with Phi and Psi those of
 *    pvio_b200_batch_imu_stream_set_covariance's FACTOR seed at Delta_s(t) (its dq_dbg carried through
 *    exp(u_theta)^T, u = K r) and G = diag(Jr(u_theta), I) the Jacobian of (+).
 *  - frame -2: the factor's Sigma(T) is not positive definite, taken as a pivot of its Cholesky factor (as
 *    pre-integration's sqrt_inv_cov forms it) at or below 1e-10 times its diagonal entry.  A one-sample factor is the
 *    known case: its C(T) has rank 6.  Such a row has a zero state and a NaN covariance; it is not a rejection.
 * Whatever n is: one host -> device copy, one kernel launch, one device -> host copy and one synchronisation; with
 * covariances three launches more (the covariance call's linearise and Schur sweeps and cov_kernel, over the frames
 * k and k + 1 of every factor with samples). */
int pvio_b200_batch_window_smoothed_trajectory(pvio_b200_handle h, int n, pvio_b200_window_trajectory *records);
/* Device -> host in one copy, per named slot i: n_frames [n], frames [n][frames_stride] ([N][16]), n_tracks [n] (live
 * tracks), and for each live track in id order at [i * track_stride + r]: id, inverse depth, anchor frame, observation
 * count, and the post-pass valid / quality of the last solve (0 / 0 for a track that did not take part in it).  Any
 * output pointer may be NULL. */
int pvio_b200_batch_window_download(pvio_b200_handle h, int n, const int32_t *slots, int32_t *n_frames, double *frames,
                                    int64_t frames_stride, int32_t *n_tracks, int64_t track_stride, int32_t *track_id,
                                    double *inv_depth, int32_t *anchor_frame, int32_t *n_observations, uint8_t *valid,
                                    double *quality);
/* The per-camera-frame half of SlidingWindowTracker::track (sliding_window_tracker.cpp:76-88) on resident slots, before
 * the edit that appends the new frame: visual_inertial_pnp of the new frame against the slot (pnp.cpp:32-100), then
 * Track::triangulate of the tracks born in the new frame (track.cpp:83-106).  The slot's newest frame plays
 * map->last_frame().  The call reads the slots and writes none of them; its results feed pvio_b200_batch_window_edit.
 *  - PnP points: an observation takes part only if its track is observed in the slot's newest frame.  Its world point
 *    is the given one when obs_point's row is finite (the plane-cast point of a TF_PLANE track, pnp.cpp:62-83),
 *    otherwise Track::get_landmark_point() from the slot: the anchor frame's camera pose applied to
 *    [z_anchor; 1] / inverse depth.  A track of role -2 or p >= 0 must come with a point.  Residual blocks follow the
 *    order of obs_track.  Extrinsics, sqrt_inv_cov and cauchy_a are the slot's; the newest frame is the constant
 *    last frame of the IMU factor.  The solve is pvio_b200_batch_pnp_solve's kernel on a record staged as that call
 *    stages it, so a record agrees with pvio_b200_batch_pnp_solve of the same problem in a batch of the same n to
 *    rounding: the kernel's per-warp sums meet in shared-memory atomics, whose order can change from run to run.
 *  - Triangulation of each new track over two views: the camera of the slot's newest frame (keypoint new_z_last) and
 *    the camera of the new frame at the solved state (keypoint new_z), with the parallax / depth < 100 checks of
 *    pvio_b200_triangulate.  new_inv_depth: the inverse depth in the newest slot frame (set_landmark_point), for a new
 *    track anchored there (a keyframe edit); new_inv_depth_next: the same re-expressed in the new frame (track.cpp:42-49),
 *    for a new track anchored in the new frame when the edit replaces the newest frame (replace_last).  Both are NaN
 *    for an invalid track.
 * Only tracks whose inverse depth is set (TF_VALID) should be named: a landmark point is not checked on the device.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no output has changed.  Rejected: a slot out
 * of range, not resident, named twice or without frames; an unknown or dead track, or one named twice in a record; a
 * non-finite keypoint; a point row neither finite nor NaN; a missing array; an inertial record without an IMU record; a
 * track of role -2 or p >= 0 that takes part without a point.  n == 0 is a no-op.  One host -> device copy, three
 * kernel launches whatever n is (gather, PnP, triangulation), one device -> host copy, one synchronisation; the staging
 * is pvio_b200_batch_pnp_solve's, grown to the largest call seen. */
typedef struct pvio_b200_window_localize {
    int32_t slot;
    int32_t use_inertial;
    const double *imu_record;   /* [PVIO_B200_IMU_STRIDE] the new frame's factor from the slot's newest frame; NULL when
                                   !use_inertial */
    double *state;              /* [16] in: the predicted state; out: the PnP solution */
    int32_t n_obs;              /* the new frame's keypoints on live tracks of the slot */
    const int32_t *obs_track;   /* [n_obs] track ids */
    const double *obs_z;        /* [n_obs][2] normalised keypoints in the new frame */
    const double *obs_point;    /* [n_obs][3] or NULL: a finite row is the world point; a NaN row or NULL: from the slot */
    double *points_out;         /* [n_obs][3] or NULL: the world point used, NaN for an observation left out */
    int32_t n_new;              /* tracks born in the new frame: keypoint in the slot's newest frame and in the new one */
    const double *new_z_last;   /* [n_new][2] */
    const double *new_z;        /* [n_new][2] */
    uint8_t *new_valid;         /* [n_new] out: Track::triangulate's result (TF_VALID) */
    double *new_inv_depth;      /* [n_new] out: inverse depth in the slot's newest frame, NaN if invalid */
    double *new_inv_depth_next; /* [n_new] or NULL, out: the same in the new frame, NaN if invalid */
    pvio_b200_summary *summary; /* or NULL: solve_seconds is the device time of the PnP launch */
} pvio_b200_window_localize;    /* 120 bytes on LP64 */
/* n records, each naming a different resident slot; opt (may be NULL) is shared. */
int pvio_b200_batch_window_localize(pvio_b200_handle h, int n, pvio_b200_window_localize *records,
                                    const pvio_b200_options *opt);
/* The raw IMU samples of a slot's factors, kept on the device with the factor, so that the slot re-integrates it before
 * every solve as BundleAdjustor::solve does (bundle_adjustor.cpp:220-231): without a first-order bias correction in the
 * factor (alias_bias), the factor follows the biases only through this re-integration.
 *  - Which factors are re-integrated: a factor that holds samples is re-integrated before every
 *    pvio_b200_batch_window_solve and pvio_b200_window_solve that names its slot, at the biases its first frame holds
 *    on the device at that moment.  The new record overwrites the old one, bg0 / ba0 included, and is bit-identical to
 *    what pvio_b200_preintegrate returns for the same samples, t_end, biases and noise.  A factor without samples keeps
 *    the record its edit gave it.
 *  - How samples follow their factor: drop_victim: the factor of old frame 1 leaves (map.cpp:86) and every other factor
 *    shifts down with its frame; replace_last: the replaced frame's samples leave, the new frame's factor holds only its
 *    edit record until a set_imu names it; pvio_b200_batch_window_reset clears every factor's samples, and so does
 *    anything that ends the slot's residency.
 *  - drop_victim's marginaliser reads the records of the last solve (as marginalize_frame reads the factors of the last
 *    solve); localize is unchanged.
 *  - Every record is checked before anything is staged: on PVIO_B200_EINVAL nothing has changed and nothing was
 *    launched.  Rejected: a slot out of range, not resident or visual-only; a frame outside 1 .. N - 1; a (slot, frame)
 *    pair named twice; n_samples < 1; a missing array; a non-finite sample, t_end or noise entry.
 *  - A set_imu call makes one host -> device copy and one kernel launch whatever n is.  A solve whose named slots hold
 *    no samples makes the launches and copies it makes without them; otherwise one more launch whatever n is, before
 *    the trust-region chain (summary.solve_seconds still times the chain only).
 * The device keeps, per slot and window frame, the samples, t_end and noise; its sample stride grows to the longest
 * list seen (every slot's samples are copied across on the device). */
typedef struct pvio_b200_window_imu {
    int32_t slot;
    int32_t frame;             /* window index j >= 1: the factor (j - 1, j) */
    int32_t n_samples;         /* >= 1 (integrate() returns false on none, preintegrator.cpp:86) */
    const double *samples;     /* [n_samples][7] t, w xyz, a xyz: frame_j->preintegration.data, as stored (after a
                                  non-keyframe merge, sliding_window_tracker.cpp:116-117, the merged list) */
    double t_end;              /* frame_j->image->t */
    const double *noise_cov;   /* [4][9] cov_w, cov_a, cov_bg, cov_ba, as pvio_b200_preintegrate takes it */
} pvio_b200_window_imu;        /* 40 bytes on LP64 */
/* n records; a slot may be named by several records, each (slot, frame) once. */
int pvio_b200_batch_window_set_imu(pvio_b200_handle h, int n, const pvio_b200_window_imu *records);
/* Device -> host, one copy: records [n][records_stride], the N_i - 1 IMU records of each named slot (resident, with
 * motion states, named once), in frame order. */
int pvio_b200_batch_window_imu_records(pvio_b200_handle h, int n, const int32_t *slots, double *records,
                                       int64_t records_stride);
/* The whole per-camera-frame start of SlidingWindowTracker::track (sliding_window_tracker.cpp:75-81, 116-118) on
 * resident inertial slots, before the frame edit; the slot's newest frame plays map->last_frame().  Per record, in the
 * reference's order:
 *  1. integrate the new frame's samples up to t_end at the newest frame's device biases (state doubles 10 .. 15):
 *     bit-identical to pvio_b200_preintegrate of the same samples, biases and noise;
 *  2. predict the new frame's state from the newest frame's device state and that record (preintegrator.cpp:102-109):
 *     biases copied, v = v_i + g dt + q_i dv, p = p_i + g dt^2 / 2 + v_i dt + q_i dp, q = q_i dq (not normalised),
 *     g = (0, 0, -9.80665);
 *  3. localize from the predicted state: the PnP and the triangulation of pvio_b200_batch_window_localize, with the
 *     same observation, point and new-track rules and the same kernels;
 *  4. keyframe_check (:255-296): frame_i is the slot's latest keyframe -- its newest frame when newest_is_keyframe,
 *     otherwise frame N - 2 (a slot holds at most one non-keyframe, its newest).  qij = (cam_q^* imu_q dq imu_q^*
 *     cam_q)^* with dq the step-1 record's.  Each named track with a keypoint in frame_i adds
 *     |apply_k(hnormalized(qij [z_i; 1])) - apply_k(z_j)| (fx, fy the slot's, cx, cy the record's): an observed track
 *     with its keypoint in frame_i from the slot, a new track with new_z_last when frame_i is the newest frame.  Fewer
 *     than 50 entries: a keyframe; otherwise entry m * 4 / 5 of the ascending list (exact for any m), a keyframe above
 *     50 px, else ++skipped; skipped > 10 forces a keyframe, a keyframe resets skipped to 0;
 *  5. when the newest frame is not a keyframe: integrate merge_samples ++ samples up to t_end at the newest frame's
 *     biases (:116-118), bit-identical to pvio_b200_preintegrate of the concatenated list.
 * imu_record is the factor the frame edit appends: step 1's record when the newest frame is a keyframe, otherwise step
 * 5's.  The call reads the slots and writes none of them.  Every record is checked before anything is staged: on
 * PVIO_B200_EINVAL no output has changed and nothing was launched.  Rejected: every localize rejection; a visual-only
 * slot; n_samples < 1; a non-finite sample, t_end, noise entry, cx or cy; newest_is_keyframe not 0 or 1; a non-keyframe
 * newest frame with N < 2 or without a merge list; a merge list with a keyframe newest frame; a missing array;
 * skipped_frames NULL or negative.  n == 0 is a no-op.  One host -> device copy, five kernel launches whatever n is
 * (integrate + predict, gather, PnP, triangulation, keyframe check), one device -> host copy, one synchronisation; the
 * staging is localize's. */
typedef struct pvio_b200_window_track_frame {
    int32_t slot;
    int32_t newest_is_keyframe;       /* 1: the slot's newest frame is a keyframe; 0: it is not (the next edit replaces it) */
    int32_t n_samples;                /* >= 1 */
    int32_t n_merge;                  /* newest_is_keyframe == 0: >= 1; otherwise 0 */
    const double *samples;            /* [n_samples][7] t, w xyz, a xyz: the new frame's own samples */
    const double *merge_samples;      /* [n_merge][7] the newest frame's own samples, or NULL with a keyframe newest frame */
    double t_end;                     /* the new frame's time */
    const double *noise_cov;          /* [4][9] cov_w, cov_a, cov_bg, cov_ba, as pvio_b200_preintegrate takes it */
    double cx, cy;                    /* principal point of the camera matrix the parallax is measured with */
    int32_t *skipped_frames;          /* in / out: the tracker's skipped-frame counter, >= 0 */
    double *state;                    /* [16] out: the PnP solution */
    double *predicted;                /* [16] or NULL, out: the predicted state */
    double *imu_record;               /* [PVIO_B200_IMU_STRIDE] out: the factor of the frame edit */
    uint8_t *keyframe;                /* out: 1 if the new frame is a keyframe */
    double *parallax;                 /* or NULL, out: the 80th-percentile parallax in px, NaN with fewer than 50 pairs */
    int32_t *n_parallax;              /* or NULL, out: the pairs in the parallax list */
    int32_t n_obs;                    /* as pvio_b200_window_localize */
    const int32_t *obs_track;
    const double *obs_z;
    const double *obs_point;
    double *points_out;
    int32_t n_new;
    const double *new_z_last;
    const double *new_z;
    uint8_t *new_valid;
    double *new_inv_depth;
    double *new_inv_depth_next;
    pvio_b200_summary *summary;
} pvio_b200_window_track_frame;       /* 216 bytes on LP64 */
/* n records, each naming a different resident slot; opt (may be NULL) is shared by the PnP solves. */
int pvio_b200_batch_window_track_frame(pvio_b200_handle h, int n, pvio_b200_window_track_frame *records,
                                       const pvio_b200_options *opt);
/* Plane detection on resident slots, from each slot's own track table: per record one Ransac<3, PlaneState,
 * PlaneSolver, PlaneEvaluator> (utility/ransac.h) over the points of its candidate tracks, then the inliers' plane.
 *  - mode PVIO_B200_PLANE_EXTRACT is PlaneExtractor::work (plane_extractor.cpp:40-81): a candidate's point is
 *    Track::get_landmark_point() from the slot row (the arithmetic of pvio_b200_batch_window_localize); threshold 0.03;
 *    the RANSAC runs on 3 or more points.
 *  - mode PVIO_B200_PLANE_REFIT is Plane::update_parameter(true) (plane.cpp:64-114): a candidate's point is
 *    Track::try_triangulate over the row's observations in the window (track.cpp:61-81: [R | T] per observing frame,
 *    R = q_cam^*, T = -R p_cam, the parallax / depth < 100 checks of pvio_b200_triangulate); threshold 0.05; fewer than
 *    50 points run no RANSAC (plane.cpp:74).  A track whose triangulation fails, or that has fewer than two window
 *    observations, is left out (the reference pushes an uninitialised point, plane.cpp:69-72).
 *  - Candidates: the caller's track ids in the caller's order, which is the RANSAC's index space: Map order for an
 *    extraction (not id order: Map::recycle_track swaps with the back), plane->tracks order (id order) for a refit.  The
 *    caller applies the rules only the map knows: TF_VALID, !TF_PLANE, life >= 10 and quality < 2.0 for an extraction
 *    (plane_extractor.cpp:45-47); TF_VALID and life >= 15 for a refit (plane.cpp:67).  The device applies
 *    PlaneExtractor::enough_baseline (plane_extractor.cpp:197-200): Track::compute_baseline over the row's observing
 *    frames in window order from their body positions (state doubles 4 .. 6), and the row's inverse depth.
 *  - Everything else is PVIO's: seed 0, confidence 0.999, 1000 iterations (every one evaluated, the serial acceptance
 *    rule replayed on the host, as pvio_b200_batch_two_view), accepted on more than 30 inliers.  PlaneSolver:
 *    n = (p2 - p0) x (p1 - p0), Eigen's stableNormalize (a zero cross product stays zero and then counts every point),
 *    d = p0 . n; an inlier has |p . n - d| <= threshold.
 *  - plane [7]: normal, distance, reference point.  Accepted: the inliers' centroid (summed serially in candidate order)
 *    is the reference point, the covariance's eigenvector of smallest eigenvalue the normal, d = n . centroid
 *    (plane_extractor.cpp:58-77, plane.cpp:78-97); the normal's sign is fixed: d >= 0, and its component of largest
 *    magnitude positive when d == 0 (the reference leaves the sign to Eigen's QR iterations).  A rejected refit returns
 *    the winning iteration's raw model, which the reference assigns whatever the count (plane.cpp:77), with a NaN
 *    reference point.  Otherwise all NaN.
 * The call reads the slots and writes none of them.  Every record is checked before anything is staged: on
 * PVIO_B200_EINVAL no output has changed and nothing was launched.  Rejected: more than 65535 records; a slot out of
 * range or not resident; a mode other than the two; n_tracks < 0; a missing array; an unknown or dead track, or one named
 * twice in a record.  A slot may be named by several records.  n == 0 is a no-op.  One host -> device copy, three
 * kernel launches whatever n is (gather and schedule, hypotheses, finish), a download of the counts and one
 * synchronisation, the replay, one more host -> device copy of the records, one device -> host copy of the results and
 * one synchronisation; the staging is the slots' (pvio_b200_batch_window_*), grown to the largest call seen. */
#define PVIO_B200_PLANE_EXTRACT 0
#define PVIO_B200_PLANE_REFIT 1
#define PVIO_B200_PLANE_ACCEPTED 0   /* more than 30 inliers                                          */
#define PVIO_B200_PLANE_FEW_POINTS 1 /* fewer used points than the mode's minimum: no RANSAC          */
#define PVIO_B200_PLANE_REJECTED 2   /* 30 inliers or fewer                                           */
typedef struct pvio_b200_window_plane_ransac {
    int32_t slot;
    int32_t mode;               /* PVIO_B200_PLANE_EXTRACT or PVIO_B200_PLANE_REFIT */
    int32_t n_tracks;
    const int32_t *tracks;      /* [n_tracks] candidate track ids of the slot, in the caller's order */
    int32_t *info;              /* [5] out: status, points that entered the RANSAC, inliers, iterations run, winning
                                   iteration (-1: none) */
    double *plane;              /* [7] out: normal, distance, reference point */
    uint8_t *used;              /* [n_tracks] out: 1 if the candidate's point entered the RANSAC */
    uint8_t *inlier;            /* [n_tracks] out: 1 if it is an inlier of the winning model */
    double *points;             /* [n_tracks][3] or NULL, out: the point used, NaN where the track was left out */
    int32_t *schedule;          /* [1000][3] or NULL, out: the sample drawn for every evaluated iteration (indices into
                                   the used points), -1 without a RANSAC */
    int32_t *counts;            /* [1000] or NULL, out: every evaluated iteration's inlier count, -1 without a RANSAC */
} pvio_b200_window_plane_ransac; /* 80 bytes on LP64 */
int pvio_b200_batch_window_plane_ransac(pvio_b200_handle h, int n, const pvio_b200_window_plane_ransac *records);
/* The link between a resident slot's newest frame and the tracker slot of pvio_b200_batch_feature_track that holds that
 * frame's keypoints: which keypoint each live track has there.  With the link set, pvio_b200_batch_window_mirror_frame
 * takes the next camera frame straight from the tracker slot.  A record replaces the slot's link: the tracker slot, the
 * tracker frame_id of the slot's newest window frame, (track, keypoint index) pairs for the live tracks observed in that
 * frame (the other tracks have no keypoint there), whether that frame is a keyframe, and the tracker's skipped-frame
 * counter (sliding_window_tracker.cpp:286).  A shim calls it after seating an initialised window (every frame a
 * keyframe, initializer.cpp:91-98) and after any host edit that writes the newest frame.
 * What keeps or clears a link: removal-only edits (prune_tracks), solve, set_planes, set_imu, set_prior and drop_victim
 * keep it, and each row keeps its keypoint index through the compactions; reset clears it, and so does every other edit
 * (replace_last, a new frame, new tracks, observations added from the host).  A link names the tracker slot's current
 * sequence: once batch_feature_track restarts the slot (map_frames == 0), mirror_frame rejects the slot until
 * set_keypoints links it again, even where frame ids repeat.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no slot has changed.  Rejected: a slot out of
 * range, not resident, without frames or named twice; a tracker slot outside 0 .. 65535; frame_id 0 or not one of the
 * tracker slot's two newest frames (of its current sequence); n < 0; a missing array; an unknown or dead track, one not observed in the newest frame, or one named twice; a keypoint index below 0 or
 * named twice; newest_is_keyframe not 0 or 1; a negative skipped_frames.  n == 0 is a no-op.  One host -> device copy,
 * one kernel launch whatever n is, one synchronisation. */
typedef struct pvio_b200_window_keypoints {
    int32_t slot;
    int32_t tracker_slot;             /* the slot of pvio_b200_batch_feature_track holding the newest frame's keypoints */
    uint64_t frame_id;                /* that frame's id in the tracker slot, != 0 */
    int32_t n;
    const int32_t *track;             /* [n] live track ids observed in the newest frame */
    const int32_t *keypoint;          /* [n] their keypoint index in that frame */
    int32_t newest_is_keyframe;       /* 0 or 1 */
    int32_t skipped_frames;           /* >= 0 */
} pvio_b200_window_keypoints;         /* 48 bytes on LP64 */
int pvio_b200_batch_window_set_keypoints(pvio_b200_handle h, int n, const pvio_b200_window_keypoints *records);
/* SlidingWindowTracker::mirror_frame (sliding_window_tracker.cpp:52-73), then the whole per-camera-frame start of
 * SlidingWindowTracker::track (:75-121) and the frame edit, on linked resident inertial slots, right after
 * pvio_b200_batch_feature_track advanced their tracker slots.  The host mirrors no keypoint.  Per record:
 *  1. mirror: the new frame's keypoints kj in order; prev_index[kj] = ki with a row at ki continues that row's track; a
 *     ki without a row is a new-track candidate (keypoint z_i[ki] in the newest frame, z_j[kj] in the new one); -1 is a
 *     fresh detection and stays without a track.  The PnP observations and the parallax list follow kj
 *     (frame->keypoint_num() order, pnp.cpp:56, :269); the candidates follow ki (mirror_frame creates tracks walking
 *     frame i, :66-71), and the slot's next ids go to the valid ones in that order.
 *  2. track_frame's steps with these lists and its kernels: integrate and predict from the newest frame, PnP,
 *     triangulation of the candidates, keyframe check, the merged record behind a non-keyframe newest frame.  PnP
 *     points: a row of role -1 always takes part, from the slot or from its given point; a row of role -2 or p >= 0
 *     only with a given point (the plane-cast point, pnp.cpp:62-85), otherwise it is left out.  The one difference from
 *     track_frame: every continued track and every candidate enters the parallax list (keyframe_check walks every
 *     track of frame j, :269-277), not only those the PnP uses.  The merge list behind a non-keyframe newest frame is
 *     the newest factor's samples, which the slot keeps (keep_samples of the call that appended that frame).
 *  3. the frame edit: replace_last when the slot's newest frame is not a keyframe; the new frame at the PnP state with
 *     the edit's IMU record, not fixed; an observation in the new frame for every continued track (a track observed in
 *     the replaced frame only ends with it, and its keypoint stays without a track); every valid candidate a new track
 *     anchored in the newest frame (new_inv_depth) with its observation in the new frame, or anchored in the new frame
 *     (new_inv_depth_next) after replace_last.  keep_samples: the new factor keeps its samples (the merged list after a
 *     non-keyframe) as pvio_b200_batch_window_set_imu would.  The slot's link moves to the new frame with the keyframe
 *     decision and the skipped-frame counter.
 * Outputs: state, predicted, imu_record, keyframe, parallax, n_parallax, skipped_frames and summary as track_frame;
 * kp_track [n_keypoints of the new frame]: the track each keypoint now observes, or -1; counts [4]: continued tracks,
 * PnP observations, new-track candidates, new tracks added.
 * Every record is checked before anything is changed: on PVIO_B200_EINVAL no slot, no tracker slot and no output has
 * changed.  Rejected: every track_frame rejection that applies (a slot out of range, not resident, visual-only, named
 * twice; n_samples < 1; a non-finite sample, t_end, noise entry, cx or cy; a missing array); an unknown or dead given
 * track, one named twice, a non-finite given point; a slot without a link; a tracker slot not the link's, named twice,
 * or restarted since the link, or whose previous frame is not the slot's newest frame (a frontend that skipped frames, feature_tracker.cpp:70-75:
 * the shim falls back to track_frame + edit + set_keypoints); max_keypoints below the tracker's keypoint count;
 * keep_samples not 0 or 1; a non-keyframe newest frame with N < 2 or whose factor holds no samples; a window that the
 * new frame would take past max_frames; and, after the mirror, a window that would exceed max_landmarks or max_obs if
 * every candidate turned out valid.  n == 0 is a no-op.  The kernel launches do not depend on n: mirror, integrate +
 * predict, gather, PnP, triangulation, keyframe check, a download of the counts and the continued rows and one
 * synchronisation, the capacity check, then append, edit, re-layout, the kept samples (when a record keeps them),
 * the link, one download of the results and a second synchronisation.  Growing the device sample store (a kept list
 * longer than any kept before, done before anything is staged) or the plane tables (after the capacity check) adds a
 * device copy and a synchronisation each. */
typedef struct pvio_b200_window_mirror {
    int32_t slot;
    int32_t tracker_slot;             /* the tracker slot just advanced by pvio_b200_batch_feature_track */
    int32_t n_samples;                /* >= 1 */
    int32_t keep_samples;             /* 1: the new factor keeps its samples on the device (as set_imu) */
    const double *samples;            /* [n_samples][7] t, w xyz, a xyz: the new frame's own samples */
    double t_end;                     /* the new frame's time */
    const double *noise_cov;          /* [4][9] cov_w, cov_a, cov_bg, cov_ba */
    double cx, cy;                    /* principal point of the camera matrix the parallax is measured with */
    int32_t n_given;
    const int32_t *given_track;       /* [n_given] live track ids with a given world point */
    const double *given_point;        /* [n_given][3] */
    int32_t max_keypoints;            /* capacity of kp_track, >= the new frame's keypoint count */
    int32_t *kp_track;                /* [max_keypoints] out */
    int32_t *counts;                  /* [4] or NULL, out */
    double *state;                    /* [16] out: the PnP solution */
    double *predicted;                /* [16] or NULL, out */
    double *imu_record;               /* [PVIO_B200_IMU_STRIDE] or NULL, out: the factor of the frame edit */
    uint8_t *keyframe;                /* out: 1 if the new frame is a keyframe */
    double *parallax;                 /* or NULL, out */
    int32_t *n_parallax;              /* or NULL, out */
    int32_t *skipped_frames;          /* or NULL, out: the counter after this frame */
    pvio_b200_summary *summary;       /* or NULL */
} pvio_b200_window_mirror;            /* 168 bytes on LP64 */
/* n records, each naming a different resident slot and a different tracker slot; opt (may be NULL) is shared by the
 * PnP solves. */
int pvio_b200_batch_window_mirror_frame(pvio_b200_handle h, int n, pvio_b200_window_mirror *records,
                                        const pvio_b200_options *opt);
/* One new camera frame of linked resident inertial slots in one call: what pvio_b200_batch_feature_track with a
 * host-given predict_q followed by pvio_b200_batch_window_mirror_frame with the same samples gives, with the IMU
 * keypoint prediction of FeatureTracker::work (feature_tracker.cpp:77-91, frame.cpp:98) made on the device.
 * Lockstep is assumed: the tracker slot's newest frame is the window slot's newest frame (the frontend's latest
 * optimised frame), so the re-prediction loop of feature_tracker.cpp:57-76 is empty.  Per record:
 *  1. PreIntegrator::integrate over samples at the biases of the slot's newest frame, then predict from that frame's
 *     state (post-solve when the slot was solved after the previous frame): `predicted`, the feature tracker's
 *     latest_state (:87-90), from which a shim's Core::predict_pose propagates.
 *  2. delta_key_q = (cam_q^* imu_q dq imu_q^* cam_q)^* from that integration's dq and the slot constants' extrinsics,
 *     each product in Eigen's scalar order, uncontracted; written to predict_q when given.
 *  3. batch_feature_track's frame with that prediction on tracker_slot (map_frames > 0), then mirror_frame's steps with
 *     the new frame's keypoints; the PnP starts from the state of step 1.
 * samples are the list mirror_frame takes: the frame's preintegration.data after the prepend rule of
 * feature_tracker.cpp:78-84, which the caller applies (it holds the previous frame's samples).
 * Rejected: every batch_feature_track and mirror_frame rejection that applies (the tracker slot is checked as it stands
 * before the call: its newest frame must be the slot's newest frame), a visual-only slot, map_frames == 0 (a sequence
 * start goes through batch_feature_track), fx or fy other than the slot constants' (the reference's Frame::K serves
 * both), and, after the gather, more keypoints than the bound or mirror_frame's capacity check.  A rejected call
 * changes no window slot, no tracker slot and no output; the tracker slot's host state (newest buffer, counts, frame
 * ids, counters) commits only after the capacity check.  Its one side effect: the tracker slot's older cached pyramid,
 * which no call reads, may have been evicted.
 * Launches, copies and synchronisations do not depend on n: batch_feature_track's and mirror_frame's together plus two
 * launches (the step-1 integration ahead of the feature stages, the delta_key_q composition), with one host -> device
 * copy more (the new frames into the mirror's records) and one device -> host copy fewer (counts and continued rows
 * in one).  n == 0 is a no-op. */
typedef struct pvio_b200_window_camera {
    int32_t slot;                     /* resident inertial slot, linked to tracker_slot */
    int32_t tracker_slot;             /* its tracker slot of pvio_b200_batch_feature_track */
    uint64_t frame_id;                /* the new frame's id, != 0 */
    int32_t width, height, stride;
    int32_t map_frames;               /* > 0: the tracker map's frame_num() before this frame is put */
    const uint8_t *image;             /* raw pixels */
    double fx, fy, cx, cy;            /* the frame's K; fx, fy as the slot constants' */
    int32_t max_keypoints;            /* capacity of kp_track, keypoints, prev_index: >= cells + 2000 */
    int32_t n_samples;                /* >= 1 */
    const double *samples;            /* [n_samples][7] t, w xyz, a xyz: the frame's samples after the prepend rule */
    double t_end;                     /* the new frame's time */
    const double *noise_cov;          /* [4][9] cov_w, cov_a, cov_bg, cov_ba */
    int32_t keep_samples;             /* 1: the new factor keeps its samples on the device (as set_imu) */
    int32_t n_given;
    const int32_t *given_track;       /* [n_given] live track ids with a given (plane-cast) world point */
    const double *given_point;        /* [n_given][3] */
    int32_t *n_keypoints;             /* out: the new frame's keypoint count */
    int32_t *kp_track;                /* [max_keypoints] out, as mirror_frame */
    int32_t *counts;                  /* [4] or NULL, out, as mirror_frame */
    double *state;                    /* [16] out: the PnP solution */
    double *predicted;                /* [16] or NULL, out: step 1's state */
    double *imu_record;               /* [PVIO_B200_IMU_STRIDE] or NULL, out: the factor of the frame edit */
    uint8_t *keyframe;                /* out */
    double *parallax;                 /* or NULL, out */
    int32_t *n_parallax;              /* or NULL, out */
    int32_t *skipped_frames;          /* or NULL, out */
    pvio_b200_summary *summary;       /* or NULL */
    double *keypoints;                /* [max_keypoints][2] or NULL, out: as batch_feature_track */
    int32_t *prev_index;              /* [max_keypoints] or NULL, out: as batch_feature_track */
    int32_t *feature_counts;          /* [4] or NULL, out: batch_feature_track's counts */
    int32_t *info;                    /* [4] or NULL, out: batch_feature_track's info */
    double *predict_q;                /* [4] or NULL, out: the delta_key_q used, x y z w */
} pvio_b200_window_camera;            /* 256 bytes on LP64 */
/* n records, each naming a different resident slot and a different tracker slot; the tracker options are
 * pvio_b200_batch_feature_track's, opt (may be NULL) is shared by the PnP solves. */
int pvio_b200_batch_window_track_camera(pvio_b200_handle h, int n, pvio_b200_window_camera *records, int max_level,
                                        int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                                        int border, double ransac_threshold, double ransac_confidence,
                                        double keypoint_distance, const pvio_b200_options *opt);
/* Snapshots: a live sequence saved to host memory and restored into any slot of any handle, so that it can outlive its
 * handle, move to another handle or device, or be forked or rolled back.  A record names a window slot, a tracker slot
 * of pvio_b200_batch_feature_track, or both (-1: none).  The blob holds the source-of-truth state only, compacted to
 * what is used: the window's constants (with the origin its solves use), counts, fixed mask, next id, prior size, keyframe flag and skipped-frame
 * counter; per live track its id, frame mask, role, inverse depth, post-pass flags, keypoint index in the newest frame
 * and fp64 keypoint per window frame; the frame states, IMU records, prior (S, e, state0), the factors' samples, t_end
 * and noise, the plane parameters; of the tracker slot the keypoints of its two newest frames (keypoint, birth,
 * prev_index; newest first), its counters, frame ids and K, and the pyramid of its newest frame with its CLAHE clip.
 * Packed tables (the solve's landmark and observation records, the frame-major table, the prior's Lambda, the plane
 * tables) are rebuilt on restore.  A blob names no slot, pointer, capacity or sequence generation, its padding is zero,
 * so save -> restore -> save gives the same bytes in any slot of any handle.
 *  - save: a resident window slot and / or a live tracker slot.  data == NULL asks for the size only (no device work);
 *    otherwise capacity must hold `size` bytes.  size is written on success.  The window's link to a tracker slot is
 *    saved only when the record names that tracker slot too and the link still names one of its two newest frames
 *    (of its current sequence) with every keypoint index inside that frame's keypoints, as mirror_frame needs it;
 *    otherwise the blob holds no link (every keypoint index -1), and such a blob restores unlinked.
 *  - restore: capacity is the blob's byte count.  A record restores the parts it names (the blob must hold them) and
 *    skips the others.  The window part replaces the target slot as a reset followed by seating the state; the tracker
 *    part replaces the target tracker slot, starts a new sequence there (a window linked to it before must be linked
 *    again) with only its newest frame cached.  The link comes back only when both parts are restored, re-pointed at the
 *    target tracker slot; otherwise the window comes back unlinked and pvio_b200_batch_window_set_keypoints links it.
 *  - Not restored: the tracker slot's lens (configuration: set it with pvio_b200_batch_set_lens on the target, as at the
 *    start of a sequence), its older pyramid, the single-call tracker and detector caches.  A blob restored into a handle
 *    of the other precision (fp32 or fp64 Jacobians) solves with that handle's pipeline.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no slot, tracker slot or output has changed.
 * Rejected: n < 0; a record naming neither part; a slot out of range (save: not resident); a tracker slot outside
 * 0 .. 65535 (save: not live); a slot or a tracker slot named twice; save capacity below the size; a restore blob with
 * the wrong magic or version, a declared size other than its byte count, a part the record names but the blob lacks,
 * or contents out of range: more frames than max_frames, more live tracks than max_landmarks, the observation, chunk and
 * 16-observation limits of the other calls, ids not strictly increasing or not below the next id, a frame mask 0 or
 * outside the window's frames, a role not -1, -2 or a plane of the blob, a prior over more frames than the window or on
 * a visual-only window, samples on a visual-only window, a keypoint index or prev_index outside its keypoint count, a
 * pyramid shape the tracker would not build.  Buffers grow as the other calls grow them.
 * Launches, whatever n is: save one pack kernel, one device -> host copy, one synchronisation; restore one host ->
 * device copy, one unpack kernel, the re-layout of the window slots and the write-back of their saved origins (4
 * launches, when a record restores a window) and one synchronisation.  A restored window solves, drops and edits
 * exactly as its source would have. */
#define PVIO_B200_SNAPSHOT_MAGIC 1314084432  /* "PVSN" as a little-endian uint32 */
#define PVIO_B200_SNAPSHOT_VERSION 1
typedef struct pvio_b200_window_snapshot {
    int32_t slot;                     /* window slot, or -1 */
    int32_t tracker_slot;             /* tracker slot of pvio_b200_batch_feature_track, or -1 */
    uint8_t *data;                    /* save: room for capacity bytes, NULL: size query only; restore: the saved bytes */
    int64_t capacity;                 /* bytes at data */
    int64_t size;                     /* save, out: the bytes the record needs / wrote */
} pvio_b200_window_snapshot;          /* 32 bytes on LP64 */
int pvio_b200_batch_window_save(pvio_b200_handle h, int n, pvio_b200_window_snapshot *records);
int pvio_b200_batch_window_restore(pvio_b200_handle h, int n, const pvio_b200_window_snapshot *records);

/* IMU stream slots: the IMU side of PVIO::Core for many sequences, one stream slot per sequence (slots 0 .. 65535,
 * independent of window and tracker slots).  A record gives a sequence's new events in arrival order, each a row
 * (kind, t, x, y, z): a gyroscope reading (rad/s), an accelerometer reading (m/s^2) or a camera timestamp (x, y, z
 * unused).  The call restates, event by event, Core::track_gyroscope / track_accelerometer (core.cpp:59-107), the frame
 * enqueue of Core::track_camera (:109-127), Core::track_imu (:129-141) and Core::predict_pose (:143-164) with
 * propagate_state (:32-39), and applies FeatureTracker::work's prepend rule (feature_tracker.cpp:78-84) to each frame
 * it releases, against the previously released frame's list, which the slot keeps.
 *  - poses: each consumed event's OutputPose, q = state.q * output_q and p = state.p + state.q * output_p (q xyzw, p),
 *    the slot's latest state propagated over its kept samples with t <= the event's t; all zero while the slot has no
 *    latest state.
 *  - released frames: when a sample releases pending camera frames (track_imu's else branch), each frame's timestamp
 *    frame_t[k], its row count frame_rows[k] and its rows, back to back in rows ([t, w xyz, a xyz]) with the prepend
 *    rule applied: the list pvio_b200_window_camera / pvio_b200_window_mirror take as samples.
 *  - Lockstep rule (the reference's frontend runs asynchronously; this makes it deterministic): a record's events are
 *    consumed up to and including the first event that releases a frame, and n_consumed says how many.  The caller
 *    runs the released frames through the frontend (pvio_b200_batch_window_track_camera, or batch_feature_track before
 *    initialisation), then calls again with the rest and the new latest state.  The releasing event's own pose uses
 *    the latest state from before the release (the frontend has only just been handed the frame).
 *  - Latest state: state_op PVIO_B200_IMU_STREAM_SET gives the slot a new latest state before the events, the 16-double
 *    `predicted` of track_camera / mirror_frame / track_frame with its frame time; CLEAR removes it
 *    (feature_tracker.cpp:74); KEEP leaves it.  The next pose computed with a new state first drops the kept samples with
 *    t <= state_time, as predict_pose does.
 *    While the slot has no state, each release drops the kept samples with t <= the released frame's time: the next
 *    state is that frame's or a later one's (DESIGN 4.7h).
 *  - Size query: a call in which any record's rows is NULL writes need_frames / need_rows of every record and does
 *    nothing else.  need_rows bounds the released rows: unreleased samples + queued accelerometer readings + the
 *    record's accelerometer readings + need_frames (pending frames + the record's camera events).
 *  - Deviation from the reference: a gyroscope or accelerometer time below that stream's previous one is rejected (the
 *    reference's output then depends on the order of its unsorted sample queue).
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no stream slot and no output has changed.
 * Rejected: n < 0; a slot out of range, named twice or never reset; n_events < 0; a NULL events or poses with events;
 * an unknown kind, state_op or a value that is not finite; a gyroscope or accelerometer time below that stream's
 * previous one; a SET state with a NULL state, or older than a frame released while the slot had no state; a queue that
 * could exceed PVIO_B200_IMU_STREAM_MAX_QUEUE entries (its size plus the record's readings that could enter it: the
 * reference's queues grow without bound on a gyroscope stream with no accelerometer and on samples before the first
 * camera frame); max_frames or max_rows below need_frames / need_rows.
 * Launches, whatever n is: one host -> device copy, one kernel (one thread per record), one device -> host copy, one
 * synchronisation; a call that grows the slots' queues first copies them into the larger buffers.  fp64, no fused
 * multiply-adds, Eigen's scalar evaluation order (DESIGN 4.7h).
 * reset: n stream slots (each once) emptied, latest state cleared, with their output extrinsic (Config
 * output_to_body_rotation [4] xyzw / translation [3] per slot). */
#define PVIO_B200_IMU_EVENT_GYROSCOPE 0
#define PVIO_B200_IMU_EVENT_ACCELEROMETER 1
#define PVIO_B200_IMU_EVENT_CAMERA 2
#define PVIO_B200_IMU_STREAM_KEEP 0
#define PVIO_B200_IMU_STREAM_SET 1
#define PVIO_B200_IMU_STREAM_CLEAR 2
#define PVIO_B200_IMU_STREAM_MAX_QUEUE 65536
typedef struct pvio_b200_imu_stream_record {
    int32_t slot;
    int32_t n_events;
    const double *events;             /* [n_events][5] kind, t, x, y, z */
    int32_t state_op;                 /* PVIO_B200_IMU_STREAM_KEEP / SET / CLEAR, applied before the events */
    double state_time;                /* SET: the state's frame time */
    const double *state;              /* SET: [16] q xyzw, p, v, bg, ba */
    double *poses;                    /* out [n_events][7] q xyzw, p: the first n_consumed rows */
    int32_t max_frames;               /* room at frame_t / frame_rows */
    int64_t max_rows;                 /* rows of room at rows */
    double *frame_t;                  /* out [max_frames] */
    int32_t *frame_rows;              /* out [max_frames] */
    double *rows;                     /* out [max_rows][7] t, w xyz, a xyz; NULL: size query */
    int32_t n_consumed;               /* out */
    int32_t n_frames;                 /* out: frames released */
    int32_t need_frames;              /* out: the room the record needs */
    int64_t need_rows;                /* out */
} pvio_b200_imu_stream_record;        /* 112 bytes on LP64 */
int pvio_b200_batch_imu_stream_reset(pvio_b200_handle h, int n, const int32_t *slots, const double *output_q,
                                     const double *output_p);
int pvio_b200_batch_imu_stream(pvio_b200_handle h, int n, pvio_b200_imu_stream_record *records);

/* Snapshots of IMU stream slots: save a stream slot to host memory and restore it into any stream slot of any handle,
 * to move a live sequence to another handle or GPU, fork it, or roll it back.  A blob is the slot's whole state between
 * two calls: the output extrinsic; the latest state with its time and whether a pose still has to drop the kept samples
 * up to it; the previously released frame's time and last row (the prepend rule reads them); the leading unreleased
 * samples given to the front frame; the last gyroscope and accelerometer times and the newest frame released without a
 * state (what rejecting a later record reads); and the live rows of the gyroscope, accelerometer, unreleased-sample,
 * pending-frame and kept-sample queues, oldest first.  What the caller holds itself (events it has not yet passed, a
 * `predicted` it has not yet fed back) is not in it.  A blob names no slot, pointer or queue capacity, its padding is
 * zero, so save -> restore -> save gives the same bytes in any stream slot of any handle.  Separate from the window
 * blobs of pvio_b200_batch_window_save: a sequence moved with its window and tracker slots takes both.
 *  - save: stream slots that were reset (and not marked unset by the internal-error path of batch_imu_stream).
 *    data == NULL asks for the size only (no device work); otherwise capacity must hold `size` bytes.  size is written
 *    on success.
 *  - restore: capacity is the blob's byte count.  The target slot takes the blob's state and counts as reset; its
 *    queues and the handle's stream slots grow as batch_imu_stream grows them.  One blob restored into several slots
 *    of one call forks the sequence.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no stream slot and no output has changed.
 * Rejected: n < 0; a slot out of range or named twice (save: never reset); save capacity below the size; a restore blob
 * with the wrong magic or version, a declared size other than its byte count or than its counts imply, a queue count
 * above PVIO_B200_IMU_STREAM_MAX_QUEUE, more leading samples than unreleased ones, a flag outside 0 / 1, a pending drop
 * without a state, a non-empty previous list without a previous frame, a state older than a frame released without
 * one, a value that is not finite, times that decrease within the gyroscope, accelerometer, unreleased-sample or
 * kept-sample queue, a queued reading newer than its stream's last time, or a non-empty queue of a stream never seen.
 * Launches, whatever n is: save one host -> device copy of the records, one pack kernel, one device -> host copy, one
 * synchronisation; restore one host -> device copy, one unpack kernel, one synchronisation (a restore that grows the
 * stream slots or their queues first copies them into the larger buffers). */
#define PVIO_B200_IMU_STREAM_SNAPSHOT_MAGIC 1397315152  /* "PVIS" as a little-endian uint32 */
#define PVIO_B200_IMU_STREAM_SNAPSHOT_VERSION 1
typedef struct pvio_b200_imu_stream_snapshot {
    int32_t slot;                     /* stream slot */
    int32_t pad;                      /* 0 */
    uint8_t *data;                    /* save: room for capacity bytes, NULL: size query only; restore: the saved bytes */
    int64_t capacity;                 /* bytes at data */
    int64_t size;                     /* save, out: the bytes the record needs / wrote */
} pvio_b200_imu_stream_snapshot;      /* 32 bytes on LP64 */
int pvio_b200_batch_imu_stream_save(pvio_b200_handle h, int n, pvio_b200_imu_stream_snapshot *records);
int pvio_b200_batch_imu_stream_restore(pvio_b200_handle h, int n, const pvio_b200_imu_stream_snapshot *records);

/* The covariance of a stream slot's latest state, for the IMU-rate pose's covariance (pvio_b200_batch_imu_stream_predict).
 * Coordinates are those of pvio_b200_batch_window_covariance: [dtheta dp dv dbg dba], q perturbed on the right,
 * q (x) exp(dtheta).  A record seeds its slot's current latest state, whose time must be state_time:
 *  - PVIO_B200_IMU_STREAM_COV_DIRECT: cov is that state's covariance.
 *  - PVIO_B200_IMU_STREAM_COV_FACTOR: the state is the `predicted` of track_camera / mirror_frame / track_frame
 *    (PreIntegrator::predict from the window's newest frame through the new frame's factor), cov is the covariance of
 *    that source frame (pvio_b200_batch_window_covariance after the solve) and imu_record the factor returned with
 *    `predicted`.  The device forms Phi cov Phi^T + Psi Sigma_d Psi^T: Phi the Jacobian of predict(integrate) with
 *    respect to the source state, its bias columns through the record's dq_dbg .. dv_dba; Sigma_d = (U^T U)^-1 with U the
 *    record's sqrt_inv_cov (upper triangular; its strict lower part is not read); Psi = diag(I, R, R, I, I), so the
 *    factor's bias random walk enters the predicted biases.  R, the source rotation, is that of q_state (x) dq^-1.
 * noise_cov [4][9] (cov_w, cov_a, cov_bg, cov_ba, 3 x 3 row-major) is what predict propagates with.  The device keeps the
 * symmetrised matrix.  A seed holds until the slot's latest state changes: any later SET record (even of the same
 * state), CLEAR, pvio_b200_batch_imu_stream_reset or pvio_b200_batch_imu_stream_restore of the slot drops it.  Seeds are
 * not part of the stream blobs: after a restore the caller seeds the slot again.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no seed has changed.
 * Rejected: n < 0; a slot out of range, named twice or never reset; a slot without a latest state or whose state time
 * is not state_time; an unknown mode; a NULL cov, noise_cov or (FACTOR) imu_record; a value that is not finite; a cov
 * that is not symmetric to 1e-12 of its largest entry or has a negative diagonal; (FACTOR) a zero diagonal in
 * sqrt_inv_cov.
 * Launches, whatever n is: one host -> device copy, one kernel (one warp per record), one synchronisation. */
#define PVIO_B200_IMU_STREAM_COV_DIRECT 0
#define PVIO_B200_IMU_STREAM_COV_FACTOR 1
typedef struct pvio_b200_imu_stream_cov_seed {
    int32_t slot;
    int32_t mode;                     /* PVIO_B200_IMU_STREAM_COV_DIRECT / FACTOR */
    double state_time;                /* the slot's latest-state time */
    const double *cov;                /* [225] row-major: the state's (DIRECT) or the source frame's (FACTOR) */
    const double *imu_record;         /* FACTOR: [PVIO_B200_IMU_STRIDE] the factor returned with `predicted` */
    const double *noise_cov;          /* [4][9] cov_w, cov_a, cov_bg, cov_ba */
} pvio_b200_imu_stream_cov_seed;      /* 40 bytes on LP64 */
int pvio_b200_batch_imu_stream_set_covariance(pvio_b200_handle h, int n, const pvio_b200_imu_stream_cov_seed *records);

/* The IMU-rate pose of stream slots at any times, with its covariance; changes no slot.  Per record, n_times
 * non-decreasing times; for each time t:
 *  - poses: the OutputPose the slot's predict_pose(t) gives as the slot stands, bit for bit (the latest state propagated
 *    with propagate_state over the kept samples with t_k <= t, then the output extrinsic).  A state that no pose has
 *    read yet skips, rather than drops, the kept samples up to its time.
 *  - states (or NULL): the propagated body state [16] q xyzw, p, v, bg, ba.
 *  - state_cov (or NULL): the seeded covariance propagated to first order along the same chain.  The sample at t_k drives
 *    the interval (t_{k-1}, t_k]; PreIntegrator::increment's noise discretisation: cov_w / max(dt, 1e-7) through
 *    dt Jr((w - bg) dt) into dtheta, cov_a / max(dt, 1e-7) through dt R and dt^2 R / 2 into dv and dp, cov_bg dt and
 *    cov_ba dt into the bias blocks.
 *  - pose_cov (or NULL): [dtheta_out dp_out] of the OutputPose, q_out = q q_ob and p_out = p + q p_ob perturbed as q:
 *    dtheta_out = R_ob^T dtheta, dp_out = dp - R hat(p_ob) dtheta.
 *  - status: PVIO_B200_OK; PVIO_B200_IMU_STREAM_NO_STATE (no latest state: zero poses and states, NaN covariances);
 *    PVIO_B200_IMU_STREAM_NO_COVARIANCE (no seed for the current state: poses and states, NaN covariances).
 * Covariance outputs are exactly symmetric.
 * Every record is checked before anything is staged: on PVIO_B200_EINVAL no output has changed.
 * Rejected: n < 0; a slot out of range, named twice or never reset; n_times < 0; a NULL times or poses with n_times > 0;
 * a time that is not finite; decreasing times.
 * Launches, whatever n is: one host -> device copy, one kernel (one warp per record), one device -> host copy, one
 * synchronisation. */
#define PVIO_B200_IMU_STREAM_NO_STATE 1
#define PVIO_B200_IMU_STREAM_NO_COVARIANCE 2
typedef struct pvio_b200_imu_stream_predict {
    int32_t slot;
    int32_t n_times;
    const double *times;              /* [n_times], non-decreasing */
    double *poses;                    /* out [n_times][7] q xyzw, p */
    double *states;                   /* out [n_times][16] or NULL */
    double *pose_cov;                 /* out [n_times][36] or NULL */
    double *state_cov;                /* out [n_times][225] or NULL */
    int32_t status;                   /* out */
    int32_t pad;
} pvio_b200_imu_stream_predict;       /* 56 bytes on LP64 */
int pvio_b200_batch_imu_stream_predict(pvio_b200_handle h, int n, pvio_b200_imu_stream_predict *records);

int pvio_b200_sync(pvio_b200_handle h);
/* CUDA-event timing on the handle's stream (bench.py): start / stop return ms. */
int pvio_b200_timer_start(pvio_b200_handle h);
int pvio_b200_timer_stop(pvio_b200_handle h, float *ms);
/* device-side time (ms) of the linearise + Schur stage from CUDA events around its launches: which = 0 the most recent
 * stage, 1 the mean stage since the last reset, 2 / 3 the mean of the linearise / Schur kernel alone, -1 reset.  Always
 * the whole batch's: when batch_gn_step runs it as overlapping sub-batches, 2 ends with the batch's last linearise sweep
 * and 3 is the Schur time left after it (DESIGN §7) */
int pvio_b200_last_kernel_ms(pvio_b200_handle h, int which, float *ms);

/* ---- visual-inertial PnP (SURVEY 8f rank 2) ------------------------------------------------ */
/* Replaces the ceres::Solve of visual_inertial_pnp, pvio/src/pvio/estimation/pnp.cpp:32-100: the new
 * frame's pose (and v, bg, ba when use_inertial) against PreIntegrationPriorCost
 * (ceres/preintegration_error_cost.h:167-206; last_frame is constant) and pose-only reprojection
 * blocks on constant world points (ceres/reprojection_error_cost.h:128-203, CauchyLoss(1.0)):
 * Track::get_landmark_point() for ordinary tracks, the plane-cast point for TF_PLANE tracks. */
typedef struct pvio_b200_pnp_problem {
    int32_t n_points;
    int32_t use_inertial;
    const double *points;        /* [n][3] world points                                        */
    const double *z;             /* [n][2] normalised keypoints in the new frame               */
    double cam_q_cs[4], cam_p_cs[3], imu_q_cs[4], imu_p_cs[3];
    double sqrt_inv_cov[4];
    double cauchy_a;
    const double *last_frame;    /* [16] map->last_frame() state (constant)          pnp.cpp:44 */
    const double *imu_data;      /* [PVIO_B200_IMU_STRIDE] frame->preintegration (bg0/ba0 ignored:
                                    they alias last_frame's biases)                             */
} pvio_b200_pnp_problem;

/* frame: [16] in/out (q xyzw, p, v, bg, ba).  One kernel launch runs the whole trust-region solve. */
int pvio_b200_pnp_solve(pvio_b200_handle h, const pvio_b200_pnp_problem *problem, double *frame,
                        const pvio_b200_options *opt, pvio_b200_summary *summary);

/* visual_inertial_pnp (pnp.cpp:32-100) for n independent problems, e.g. the new frame of n sequences, in ONE kernel
 * launch, one CTA per problem.  problems [n]: as for pvio_b200_pnp_solve; each problem has its own points,
 * extrinsics, sqrt_inv_cov, last frame and IMU record.  frames: n rows of frames_stride (>= 16) doubles, in/out.
 * opt: shared by all problems.  summaries [n] (may be NULL): one per problem; solve_seconds = device time of the
 * batched launch.  Every problem is checked before anything is copied: on PVIO_B200_EINVAL no frame has changed.
 * n == 0 is a no-op.  Independent of the capacities given to pvio_b200_create.  A problem solved in a batch matches
 * its pvio_b200_pnp_solve to rounding, not bit for bit (the per-point sums are combined in a different order). */
int pvio_b200_batch_pnp_solve(pvio_b200_handle h, int n, const pvio_b200_pnp_problem *problems, double *frames,
                              int64_t frames_stride, const pvio_b200_options *opt, pvio_b200_summary *summaries);

/* Same, from the RAW 8-bit frames: CLAHE (cv::createCLAHE(clahe_clip, Size(tiles_x, tiles_y))->apply,
 * pvio-extra/src/pvio/extra/opencv_image.cpp:138-143: clip 6.0, 8 x 8 tiles) runs on the device between the upload and
 * the pyramid build, bit-exact with OpenCV.  width / height must be multiples of tiles_x / tiles_y (752x480 and
 * 512x512 are).  prev_eq / next_eq (optional, [height][width]): the equalised frames, e.g. to hand to GFTT. */
int pvio_b200_klt_track_raw(pvio_b200_handle h, const uint8_t *prev, const uint8_t *next,
                            int width, int height, int stride, const float *prev_pts,
                            float *next_pts, uint8_t *status, float *err, int n_points,
                            int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                            uint8_t *prev_eq, uint8_t *next_eq);

/* The call OpenCvImage::track_keypoints maps to in a running tracker (opencv_image.cpp:88-136, caller
 * core/feature_tracker.cpp:92: prev is always the previous call's next): frames carry ids (!= 0) and the handle keeps the
 * finished pyramids (CLAHE output + 4 levels) of the last two frames on the device, so a steady-state call uploads and
 * builds ONE pyramid; an image whose id is cached may be passed as NULL.  clahe_clip > 0: raw frames, CLAHE on the
 * device; 0: frames are already equalised.  border > 0: the 20-pixel border rejection of :106-108 runs on the device. */
int pvio_b200_klt_track_cached(pvio_b200_handle h, uint64_t prev_id, const uint8_t *prev, uint64_t next_id, const uint8_t *next,
                               int width, int height, int stride, const float *prev_pts, float *next_pts, uint8_t *status,
                               float *err, int n_points, int max_level, int max_iter, double eps, double clahe_clip,
                               int tiles_x, int tiles_y, int border);

/* OpenCvImage::detect_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:54-86): GFTT with the Harris response
 * (GFTTDetector::create(1000, 1e-3, 20, 3, true), :183) on the preprocessed frame, PVIO's Poisson-disk filter
 * (utility/poisson_disk_filter.h) against the `existing` keypoints [n_existing][2] with radius keypoint_distance, 20-pixel
 * border.  The frame is taken from the pyramid cache of pvio_b200_klt_track_cached when frame_id is cached there
 * (image may then be NULL); otherwise `image` is uploaded (clahe_clip > 0: raw frame, equalised on the device first).
 * keypoints_out [max_out][2] pixel coordinates in the reference's order (decreasing response), *n_out their number.
 * gftt_out [1000][2] / n_gftt (may be NULL): the corners before the Poisson filter, for parity checks against
 * cv::goodFeaturesToTrack. */
int pvio_b200_detect_keypoints(pvio_b200_handle h, uint64_t frame_id, const uint8_t *image, int width, int height, int stride,
                               double clahe_clip, int tiles_x, int tiles_y, const double *existing, int n_existing,
                               double keypoint_distance, int max_out, double *keypoints_out, int *n_out,
                               float *gftt_out, int *n_gftt);

/* The F-matrix outlier rejection of OpenCvImage::track_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:121-129):
 * cv::findFundamentalMat(p, q, cv::FM_RANSAC, threshold, confidence, mask) with OpenCV's semantics -- n >= 15: RANSAC on
 * 7-point models, at most max_iters (OpenCV: 1000) iterations with the adaptive iteration count; 8 <= n < 15: OpenCV's
 * LMedS branch; n == 7: mask all ones; n < 7: mask zero.  p, q: [n][2] pixel coordinates (the cv::Point2f values).
 * schedule == NULL: the samples are the ones OpenCV itself draws (cv::RNG((uint64)-1) and getSubset restated), so the
 * mask is cv2's; otherwise int32 [n_schedule][7] injected sample indices (a row starting with -1 ends the run).
 * Every iteration of the schedule is evaluated on the device at once; the host replays OpenCV's acceptance rule over
 * the inlier counts (see csrc/fmat.cu).  mask: [n] 0/1.  F (may be NULL): the winning model, row-major 3x3.
 * info (may be NULL): int32[4] = iterations the serial loop runs, winning iteration, winning model, method (1 RANSAC,
 * 2 LMedS, 3 seven points). */
int pvio_b200_find_fundamental_mask(pvio_b200_handle h, int n, const float *p, const float *q, double threshold, double confidence,
                                    int max_iters, const int32_t *schedule, int n_schedule, uint8_t *mask, double *F, int32_t *info);

/* Host only (no device, no handle): the sample schedule the call above uses when schedule == NULL, i.e. the subsets
 * cv::findFundamentalMat draws for these n >= 8 matches with cv::RNG((uint64)-1): int32 [iters][7].  Returns the number of
 * iterations that have a subset (< iters only if getSubset gives up: degenerate, collinear input), or a negative error. */
int pvio_b200_fm_sample_schedule(int n, const float *p, const float *q, int iters, int32_t *schedule);

/* OpenCvImage::track_keypoints as a whole (opencv_image.cpp:88-136): pvio_b200_klt_track_cached (LK on the cached pyramids,
 * 20-pixel border on the device) followed by the F-matrix rejection above over the surviving matches when there are at
 * least 8 (:121).  next_pts holds the initial guess on entry (:91-96: the caller's next_keypoints, or a copy of prev_pts);
 * on return status[i] != 0 marks the matches the reference keeps and next_pts[i] their positions. */
int pvio_b200_track_keypoints(pvio_b200_handle h, uint64_t prev_id, const uint8_t *prev, uint64_t next_id, const uint8_t *next,
                              int width, int height, int stride, const float *prev_pts, float *next_pts, uint8_t *status,
                              int n_points, int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                              int border, double ransac_threshold, double ransac_confidence);

/* One frame pair of pvio_b200_batch_track_keypoints: the next frame of one sequence. */
typedef struct pvio_b200_klt_pair {
    int32_t slot;                  /* the sequence's cache slot, 0 .. 65535, distinct within one call                 */
    int32_t width, height, stride;
    uint64_t prev_id, next_id;     /* frame ids WITHIN the sequence, != 0                                             */
    const uint8_t *prev, *next;    /* pixels (raw when clahe_clip > 0); NULL allowed when the id is cached in this    */
                                   /* slot                                                                            */
    int32_t n_points;
    const float *prev_pts;         /* [n][2]                                                                          */
    float *next_pts;               /* [n][2] in: initial guess (opencv_image.cpp:91-96), out: tracked positions       */
    uint8_t *status;               /* [n] out: the matches the reference keeps                                        */
    float *err;                    /* [n] out, may be NULL: LK error, as pvio_b200_klt_track_cached gives it          */
    int32_t *info;                 /* [4] out, may be NULL: as pvio_b200_find_fundamental_mask's info;                */
                                   /* {0, -1, -1, 0} when fewer than 8 matches survive                                */
} pvio_b200_klt_pair;              /* 96 bytes on LP64 */

/* pvio_b200_track_keypoints for n independent sequences in one call, e.g. the new camera frame of each.  Each pair
 * gets bit for bit what pvio_b200_track_keypoints gives on a handle whose cache holds that sequence's frames: LK on
 * the two pyramids, the border test, and findFundamentalMat(FM_RANSAC) with OpenCV's own sample schedule over the
 * survivors (LMedS below 15) when at least 8 survive.  The options are shared; the image shape may differ per pair,
 * and each pair's level count follows OpenCV's small-image rule for its own shape.
 * Cache: slot s keeps the finished pyramids of the last two frames of its sequence, keyed by (id, clahe_clip); ids
 * are looked up in their own slot only, so two slots may use the same ids for different images.  A slot's buffers
 * are rebuilt, and its cache dropped, only when its shape or level count changes.  Slots are created on demand,
 * independent of the window capacities, and separate from the cache of the single calls (which
 * pvio_b200_detect_keypoints reads): neither path reads or evicts the other's frames.  Unlike the single call, a pair
 * with n_points == 0 still caches its next frame, so a sequence that lost every track continues with prev = NULL.
 * Every pair is checked before anything is staged: on PVIO_B200_EINVAL no output and no slot has changed.  n == 0 is
 * a no-op.  A call whose previous frames are all cached runs CLAHE, pyrDown, LK, the schedules, the hypotheses and
 * the masks as at most 7 + max_level kernel launches whatever n is, with two synchronisations. */
int pvio_b200_batch_track_keypoints(pvio_b200_handle h, int n, const pvio_b200_klt_pair *pairs,
                                    int max_level, int max_iter, double eps, double clahe_clip,
                                    int tiles_x, int tiles_y, int border,
                                    double ransac_threshold, double ransac_confidence);

/* One frame of pvio_b200_batch_detect_keypoints: the arguments of one pvio_b200_detect_keypoints call. */
typedef struct pvio_b200_detect_request {
    int32_t slot;                  /* a sequence slot of pvio_b200_batch_track_keypoints, 0 .. 65535                  */
    int32_t width, height, stride; /* width, height >= 8; stride >= width when the pixels are uploaded                */
    uint64_t frame_id;             /* the frame's id within its slot's sequence (0: never cached)                     */
    const uint8_t *image;          /* pixels (raw when clahe_clip > 0); NULL allowed when frame_id is cached in slot  */
    const double *existing;        /* [n_existing][2] the frame's existing keypoints, pixels                          */
    int32_t n_existing;
    int32_t max_out;
    double keypoint_distance;      /* Poisson-disk radius, > 0                                                        */
    double *keypoints_out;         /* [max_out][2] out: the new keypoints in the reference's order                    */
    int32_t *n_out;                /* out: their number                                                               */
    float *gftt_out;               /* [1000][2] out, may be NULL: the GFTT corners before the Poisson filter          */
    int32_t *n_gftt;               /* out, may be NULL: their number                                                  */
} pvio_b200_detect_request;        /* 88 bytes on LP64 */

/* pvio_b200_detect_keypoints for n frames in one call, e.g. the frame each sequence of a batched tracker call has just
 * tracked into.  Each request gets bit for bit what pvio_b200_detect_keypoints gives for that frame: the same keypoints
 * and GFTT corners in the same order.  clahe_clip and the tile grid are shared.
 * Frame source: level 0 of the pyramid in the request's slot of pvio_b200_batch_track_keypoints is used when
 * (frame_id, clahe_clip) is cached in that slot -- either of the slot's two cached frames -- and the shape matches;
 * otherwise `image` is uploaded, and equalised on the device when clahe_clip > 0 (the size must then be a multiple of
 * the tile grid).  The call changes no cache, neither the slots nor the single calls' cache, so several requests may
 * name the same slot.
 * Every request is checked before anything is staged: on an argument error PVIO_B200_EINVAL is returned and no output
 * has changed.  A request whose keypoints do not fit gets its first max_out keypoints and *n_out = its full count (at
 * most 1000), as the single call, and the call returns PVIO_B200_EINVAL after every request has its results.  n == 0 is
 * a no-op.  A call runs CLAHE (uploaded frames only), Harris, non-maximum suppression, a segmented sort and the two
 * greedy passes as at most 6 kernel launches whatever n is, with one upload, one download and one synchronisation. */
int pvio_b200_batch_detect_keypoints(pvio_b200_handle h, int n, const pvio_b200_detect_request *requests,
                                     double clahe_clip, int tiles_x, int tiles_y);

/* One camera frame of pvio_b200_batch_feature_track: the next frame of one sequence. */
typedef struct pvio_b200_feature_frame {
    int32_t slot;                  /* a sequence slot of pvio_b200_batch_track_keypoints, 0 .. 65535, distinct        */
    int32_t width, height, stride;
    uint64_t frame_id;             /* the frame's id within the sequence, != 0                                        */
    const uint8_t *image;          /* raw pixels (undistorted on the device when the slot has a lens)                 */
    double fx, fy, cx, cy;         /* the frame's K                                                                   */
    int32_t map_frames;            /* the tracker map's frame_num() before this frame is put (0: a new sequence)      */
    int32_t max_keypoints;         /* capacity of keypoints / prev_index (see the bound below)                       */
    const double *predict_q;       /* [4] x, y, z, w: delta_key_q of frame.cpp:98; NULL: no prediction              */
    double *keypoints;             /* [max_keypoints][2] out: the frame's keypoints, normalised (Frame::keypoints)    */
    int32_t *prev_index;           /* [max_keypoints] out: the previous frame's keypoint each one continues, or -1   */
    int32_t *n_keypoints;          /* out: their number                                                               */
    int32_t *counts;               /* [4] out, may be NULL: kept after LK and the border test, after F-RANSAC, after */
                                   /* the track-length thinning, and the number of new detections                    */
    int32_t *info;                 /* [4] out, may be NULL: as pvio_b200_klt_pair::info                               */
} pvio_b200_feature_frame;         /* 120 bytes on LP64 */

/* The per-frame step of FeatureTracker::work (feature_tracker.cpp:77-99) for n sequences in one call: Frame::track_keypoints
 * of the previous frame into this one (frame.cpp:88-138) -- the initial guesses, pvio_b200_batch_track_keypoints' LK,
 * border test and F-RANSAC, then the track-length-ordered Poisson-disk thinning -- followed by Frame::detect_keypoints
 * (frame.cpp:72-86) on the new frame.  Each slot keeps its newest frame's keypoints on the device, so nothing but the
 * new pixels goes up and the new keypoints come down.  The options are pvio_b200_batch_track_keypoints' plus
 * keypoint_distance (Config::feature_tracker_min_keypoint_distance, > 0).
 * Slot rules:
 *  - map_frames == 0 starts the sequence: the slot drops its keypoints, and the frame is only equalised, cached and
 *    detected, as the reference does for a map's first frame.
 *  - map_frames > 0 continues it: the slot's newest frame must still be in its pyramid cache (same shape and
 *    clahe_clip); a request whose frame another call has evicted is rejected, as is a frame_id equal to that frame's.
 *  - A slot named twice is rejected.
 *  - max_keypoints below cells + 2000 is rejected, cells = (floor(w / (r / sqrt 2)) + 1) (floor(h / (r / sqrt 2)) + 1)
 *    with r = keypoint_distance: the thinned keypoints are at least r apart (at most one per cell), and at most 1000
 *    untracked survivors and 1000 detections are added.
 *  - Every request is checked before anything is staged: on PVIO_B200_EINVAL no output and no slot has changed.
 *  - pvio_b200_batch_track_keypoints and pvio_b200_batch_detect_keypoints leave a slot's keypoints alone (they may
 *    evict its frames).
 * A keypoint's track length is min(frames since it was detected + 1, map_frames); keypoints the previous frame detected
 * have no track yet and skip the thinning.  n == 0 is a no-op.  With clahe_clip > 0 the launches, copies and
 * synchronisations of a call do not depend on n (DESIGN.md §4.7f). */
int pvio_b200_batch_feature_track(pvio_b200_handle h, int n, const pvio_b200_feature_frame *frames,
                                  int max_level, int max_iter, double eps, double clahe_clip,
                                  int tiles_x, int tiles_y, int border,
                                  double ransac_threshold, double ransac_confidence, double keypoint_distance);

/* ---- two-view initialisation ------------------------------------------------------------- */
/* The two-view step of Initializer::init_sfm (pvio/src/pvio/core/initializer.cpp:102-161) that seeds a sequence: the
 * match-count and parallax gates, find_homography_matrix and find_essential_matrix (Ransac<> of utility/ransac.h,
 * threshold 0.7 / fx), decompose_homography and decompose_essential, and triangulate_from_rt_scored over the 8 pose
 * candidates.  status is the first of init_sfm's early returns that applies, in its order: */
#define PVIO_B200_TWO_VIEW_OK 0
#define PVIO_B200_TWO_VIEW_FEW_MATCHES 1      /* n_matches < min_matches, or n_matches < 5                      */
#define PVIO_B200_TWO_VIEW_LOW_PARALLAX 2     /* mean parallax (pixels) < min_parallax                          */
#define PVIO_B200_TWO_VIEW_PURE_ROTATION 3    /* decompose_homography found a pure rotation                     */
#define PVIO_B200_TWO_VIEW_FEW_TRIANGULATED 4 /* the chosen candidate triangulates fewer than min_triangulation */

/* One problem of pvio_b200_batch_two_view: the matches of frames i and j of one sequence.  Every output may be NULL. */
typedef struct pvio_b200_two_view {
    int32_t n_matches;
    int32_t seed;                  /* Config::random(); PVIO's default 648                                            */
    const double *p1, *p2;         /* [n][2] normalised keypoints of frames i and j (initializer.cpp:117-127)         */
    double fx, fy;                 /* frame i's focal lengths: the parallax in pixels and the threshold 0.7 / fx      */
    int32_t min_matches;           /* Config::initializer_min_matches (50)                                            */
    int32_t min_triangulation;     /* Config::initializer_min_triangulation (20)                                      */
    double min_parallax;           /* Config::initializer_min_parallax (10)                                           */
    double confidence;             /* 0.999                                                                           */
    int32_t max_iteration;         /* 1000                                                                            */
    int32_t *info;                 /* [10] out: status, H inliers, H iterations run, H winning iteration,             */
                                   /* E inliers, E iterations run, E winning iteration, E winning model,              */
                                   /* chosen candidate (0..7 in init_sfm's Rs / Ts order), triangulated count;        */
                                   /* winners and candidate -1 when there are none                                    */
    double *parallax;              /* out: the mean parallax                                                          */
    double *H, *E;                 /* [9] out, row-major: the two RANSACs' models (0 without a winner)                */
    double *R, *T;                 /* [9], [3] out: init_R, init_T (the chosen candidate)                             */
    uint8_t *h_mask, *e_mask;      /* [n] out: the inlier masks of the two winners                                    */
    double *points;                /* [n][3] out: the chosen candidate's points in frame i (0 where not triangulated) */
    uint8_t *point_status;         /* [n] out: init_point_status                                                      */
    int32_t *h_schedule;           /* [max_iteration][4] out: the H RANSAC's sample schedule                          */
    int32_t *e_schedule;           /* [max_iteration][5] out: the E RANSAC's sample schedule                          */
    int32_t *h_counts;             /* [max_iteration] out: the inliers of each iteration's homography                 */
    int32_t *e_counts;             /* [max_iteration][11] out: each iteration's model count, then each model's inliers */
} pvio_b200_two_view;              /* 184 bytes on LP64 */

/* init_sfm's two-view step for n sequences in one call.  Both RANSACs evaluate every iteration of their sample schedule
 * (drawn on the device as Ransac::solve draws it, from a LotBox seeded with `seed`) and the serial acceptance rule,
 * early stop included, is replayed on the host: each problem gets the serial loop's result for that schedule.  One
 * deviation: the E models of one iteration are taken in ascending order of their action-matrix eigenvalue (the reference
 * takes Eigen's real-Schur order), which matters only when two models of one iteration tie on the winning count.
 * decompose_essential's SVD leaves the sign of T and the order of R1, R2 to rounding (an essential matrix has two equal
 * singular values); here T's component of largest magnitude is positive and R1 has the larger trace.  The
 * RANSACs and the triangulation run whatever the gates say, except below 5 matches; the diagnostic outputs (schedules,
 * counts) are written for the iterations evaluated, none below 5 matches.
 * Every record is checked before anything is staged: PVIO_B200_EINVAL, with no output changed, for n < 0, n > 65535,
 * a negative n_matches or one above 2^24, more than 2^31 - 1 matches in all, NULL keypoints with n_matches > 0, fx or
 * fy not positive, confidence not positive, max_iteration < 1 or a negative minimum.  n == 0 is a no-op.  A call is 4
 * kernel launches and 2 synchronisations whatever n is; its buffers grow to the largest call and are then reused. */
int pvio_b200_batch_two_view(pvio_b200_handle h, int n, const pvio_b200_two_view *records);

/* ---- lens distortion ------------------------------------------------------------------- */
/* The undistortion PVIO's dataset readers run on every raw frame before CLAHE:
 *  PVIO_B200_LENS_RADTAN       cv::undistort(img, out, K, D) with K and D as cv::Mat_<float> (EurocDatasetReader::read_image,
 *                              pvio-pc/src/euroc_dataset_reader.cpp:70-74; OpenCvImage::correct_distortion,
 *                              pvio-extra/src/pvio/extra/opencv_image.cpp:162-175): coefficients k1 k2 p1 p2, new camera
 *                              matrix K.  fx, fy, cx, cy and the coefficients are first rounded to float32.
 *  PVIO_B200_LENS_EQUIDISTANT  ImageUndistorter (pvio-extra/include/pvio/extra/image_undistorter.h:28-95, as
 *                              tum_dataset_reader.cpp:71-81 uses it): distort_pixel in double, a float map converted by
 *                              cv::convertMaps to CV_16SC2, cv::remap(INTER_LINEAR, BORDER_CONSTANT).  Coefficients k1..k4.
 * The undistorted frame has the raw frame's shape.  Both are a bilinear remap with OpenCV's fixed-point weights, bit for
 * bit what OpenCV gives. */
#define PVIO_B200_LENS_RADTAN 1
#define PVIO_B200_LENS_EQUIDISTANT 2

/* Host only (no device, no handle): the map of one lens for width x height frames, built in fp64 on the host as OpenCV
 * builds it (cv::undistort's 4096-pixel stripes included).  fx_fy_cx_cy [4], coeffs [4] as above.  Out: OpenCV's CV_16SC2
 * pair, m1 int16 [height][width][2] the integer source pixel (x, y), m2 uint16 [height][width] the fraction index
 * (v & 31) * 32 + (u & 31) of the 1/32-pixel coordinates (u, v).  PVIO_B200_EINVAL for an unknown model, width or height
 * below 8 or above 32767 (cv::remap's limit), a parameter that is not finite, fx <= 0 or fy <= 0, or a map coordinate
 * that is not finite. */
int pvio_b200_undistort_map(int model, int width, int height, const double *fx_fy_cx_cy, const double *coeffs,
                            int16_t *m1, uint16_t *m2);

/* The lens of one sequence slot of pvio_b200_batch_track_keypoints. */
typedef struct pvio_b200_lens {
    int32_t slot;                  /* a sequence slot of pvio_b200_batch_track_keypoints, 0 .. 65535                  */
    int32_t model;                 /* 0 none (clears the slot's lens), PVIO_B200_LENS_RADTAN, PVIO_B200_LENS_EQUIDISTANT */
    int32_t width, height;         /* the raw frame's shape; the undistorted frame has the same shape                */
    double fx, fy, cx, cy;
    double coeffs[4];              /* radtan: k1 k2 p1 p2; equidistant: k1 k2 k3 k4                                   */
} pvio_b200_lens;                  /* 80 bytes on LP64 */

/* Sets (or, model 0, clears) the lens of n slots, once per sequence.  Each slot's map is built on the host
 * (pvio_b200_undistort_map) and kept on the device, one map per slot at 6 bytes per pixel: 2.2 MB for 752 x 480, so 528
 * slots hold 1.1 GB.  Slots never share a map.  From then on a frame that pvio_b200_batch_track_keypoints or
 * pvio_b200_batch_detect_keypoints uploads for a slot with a lens is the RAW frame: it is undistorted on the device
 * before CLAHE, and the results are bit for bit those of the same call on frames undistorted by OpenCV.  Frames read
 * from a slot's cache are used as cached (already undistorted).  A tracker pair whose slot has a lens must have the
 * lens's shape.  Setting or clearing a lens drops the slot's two cached frames.  Slots are created on demand; a lens
 * outlives the tracker's rebuild of its slot on a shape change.  Every record is checked, and every map built, before a
 * slot changes: PVIO_B200_EINVAL for each rejection of pvio_b200_undistort_map, a slot out of range or a slot named
 * twice.  n == 0 is a no-op. */
int pvio_b200_batch_set_lens(pvio_b200_handle h, int n, const pvio_b200_lens *records);

/* One frame of pvio_b200_batch_undistort. */
typedef struct pvio_b200_undistort_request {
    int32_t slot;                  /* a slot with a lens                                                              */
    int32_t width, height, stride; /* the lens's shape; stride >= width                                               */
    const uint8_t *src;            /* the raw frame                                                                   */
    uint8_t *dst;                  /* [height][width] out: the undistorted frame                                      */
} pvio_b200_undistort_request;     /* 32 bytes on LP64 */

/* The undistorted frames of n slots (several requests may name one slot), for callers that need the image itself: one
 * upload, one kernel launch, one download.  The call reads no cache and changes none.  Every request is checked first:
 * PVIO_B200_EINVAL for a slot out of range or without a lens, a shape other than the lens's, stride < width, or a NULL
 * pointer; no output has changed then. */
int pvio_b200_batch_undistort(pvio_b200_handle h, int n, const pvio_b200_undistort_request *requests);

/* CLAHE of one frame (same kernels); dst is [height][width]. */
int pvio_b200_clahe(pvio_b200_handle h, const uint8_t *src, int width, int height, int stride, double clip_limit,
                    int tiles_x, int tiles_y, uint8_t *dst);

/* ---- IMU pre-integration ---------------------------------------------------------------- */
/* PreIntegrator::integrate(t, bg, ba, true, true) (pvio/src/pvio/estimation/preintegrator.cpp:85-98) for
 * n_factors independent factors, one warp each.  samples: rows (t, w xyz, a xyz) of every factor back to
 * back, begin[n_factors + 1] the CSR offsets; the last sample of a factor is integrated up to t_end[i].
 * bias: [n_factors][6] (bg, ba) -- the biases of the factor's FIRST frame (bundle_adjustor.cpp:228).
 * noise_cov: [4][9] row-major 3x3 cov_w, cov_a, cov_bg, cov_ba (preintegrator.h:63-66).
 * records: [n_factors][PVIO_B200_IMU_STRIDE], the layout pvio_b200_window::imu_data takes. */
int pvio_b200_preintegrate(pvio_b200_handle h, int n_factors, const int32_t *begin, const double *samples,
                           const double *t_end, const double *bias, const double *noise_cov, double *records);

/* ---- triangulation of new tracks ---------------------------------------------------------- */
/* Track::triangulate (pvio/src/pvio/map/track.cpp:83-106): multi-view DLT (stereo.h:67-75) and the parallax /
 * depth checks of triangulate_point_scored (stereo.h:104-128), one thread per track.
 * P: [n_frames][12] row-major 3x4 [R | T] of the CAMERA in each frame (R = q_wc^-1, T = -R p_wc, track.cpp:90-95).
 * begin / obs_frame / obs_z: CSR list of ALL keypoints of each track (>= 2 views).
 * points: [n_tracks][3] (q.hnormalized() when valid; otherwise the unit direction, whose sign is that of the
 * singular vector and as unspecified as in the reference, stereo.h:122-126);
 * valid: has_parallax; score: mean squared reprojection error in normalised coordinates. */
int pvio_b200_triangulate(pvio_b200_handle h, int n_frames, const double *P, int n_tracks, const int32_t *begin,
                          const int32_t *obs_frame, const double *obs_z, double *points, uint8_t *valid, double *score);

/* ---- diagnostics ---------------------------------------------------------------------- */
/* Device self-test of the Lie-group helpers (geometry/lie_algebra.h:25-42, lie_algebra.cpp:22-59,
 * quaternion_parameterization.h:28-31): w [n][3] rotation vectors; out [n][32] = expmap(w) (4, xyzw),
 * logmap(expmap(w)) (3), right_jacobian(w) (9, row-major), its inverse (9), Plus(expmap(w), w) (4), 3 spare.
 * Not part of the reference interface. */
int pvio_b200_selftest_lie(pvio_b200_handle h, int n, const double *w, double *out);
/* Device self-test of the marginaliser's eigen-solver (the factorisation of bundle_adjustor.cpp:583-590): n problems in
 * one launch of the same kernel, with the launch shape pvio_b200_ba_marginalize gives a window of the largest dk.
 * Problem i: dk[i] in {15, 30, ..., 165}, a dk[i] x dk[i] symmetric row-major matrix A_i and a vector b_i, stored back to
 * back in A and b.  Out, in the same layout: S_i = sqrt(lambda+) V^T and e_i = sqrt(1 / lambda+) V^T b_i, where lambda+
 * keeps the eigenvalues above 1e-8 (the rows of the others are 0).  PVIO_B200_EINVAL for n < 1 or a dk outside that set.
 * Not part of the reference interface. */
int pvio_b200_selftest_eig(pvio_b200_handle h, int n, const int32_t *dk, const double *A, const double *b, double *S_out,
                           double *e_out);
/* Device self-test of the reduced-system Cholesky solve of the Gauss-Newton step: n systems in one launch, one CTA per
 * system, packed as the solve kernels pack a window's reduced system (4 x 4 tiles, D padded to 4 nb with identity rows).
 * System i: D[i] unknowns, a D[i] x D[i] symmetric row-major matrix A_i (its lower triangle is read) and a right-hand
 * side b_i, stored back to back in A and b.  mode 0: the factorisation of the batched visual-only kernel (64 threads);
 * 1: the one the single-window kernel chooses for the block count (256 threads); 2: its tiled fallback, forced.
 * Out: x_i (same layout as b; 0 where the factorisation failed) and ok_i = 1 where every pivot was positive and finite.
 * PVIO_B200_EINVAL for n < 1, an unknown mode, a D[i] < 1, a system that needs more shared memory than the mode's
 * production kernel gets (48 KB for mode 0, 220 KB otherwise) or, in mode 1, more than 64 block rows.
 * Not part of the reference interface. */
int pvio_b200_selftest_chol(pvio_b200_handle h, int n, int mode, const int32_t *D, const double *A, const double *b,
                            double *x_out, int32_t *ok_out);

/* ---- KLT ----------------------------------------------------------------------------- */
/* Pyramidal Lucas-Kanade with OpenCV's semantics: winSize 21x21, maxLevel levels above
 * level 0, criteria COUNT+EPS (max_iter, eps), OPTFLOW_USE_INITIAL_FLOW (next_pts holds
 * the guess on entry), minEigThreshold 1e-4.  prev/next: 8-bit single-channel images
 * (post-CLAHE).  status[i] = 1 if found; err[i] as cv (mean abs patch difference). */
int pvio_b200_klt_track(pvio_b200_handle h, const uint8_t *prev, const uint8_t *next,
                        int width, int height, int stride, const float *prev_pts,
                        float *next_pts, uint8_t *status, float *err, int n_points,
                        int max_level, int max_iter, double eps);

#ifdef __cplusplus
}
#endif
#endif /* PVIO_B200_H */
