"""ctypes binding of libpvio_b200.so (the C-ABI in include/pvio_b200.h): the header's constants, its structs as ctypes
classes, one signature table that load() applies to every entry point, and the typed pointer helpers.  This is the
only module that declares the ABI; tests/test_abi_bindings.py holds it to the header.

There is NO CPU fallback: if the shared library is missing or no CUDA device is present the
product path raises.  The library is built in-tree by `python -m pvio_b200.build`
(__graft_entry__.build())."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpvio_b200.so")
if os.environ.get("PVIO_B200_TUNE_LIB"):        # tools/ only: a tuning build of the same sources (pvio_b200.build, defines=...)
    LIB_PATH = os.environ["PVIO_B200_TUNE_LIB"]

# ---- the header's constants (PVIO_B200_<name>) ----------------------------------------------------------------------
OK, ENODEV, EINVAL, ENOMEM, ECUDA, ENUMERIC = 0, -1, -2, -3, -4, -5
FRAME_STRIDE = 16
IMU_STRIDE = 288
IMU_DT, IMU_DQ, IMU_DP, IMU_DV, IMU_SQRT_INV_COV = 0, 1, 5, 8, 11
IMU_DQ_DBG, IMU_DP_DBG, IMU_DP_DBA, IMU_DV_DBG, IMU_DV_DBA, IMU_BG0, IMU_BA0 = 236, 245, 254, 263, 272, 281, 284
TERM_CONVERGENCE, TERM_NO_CONVERGENCE, TERM_FAILURE = 0, 1, 2
TWO_VIEW_OK, TWO_VIEW_FEW_MATCHES, TWO_VIEW_LOW_PARALLAX, TWO_VIEW_PURE_ROTATION, TWO_VIEW_FEW_TRIANGULATED = 0, 1, 2, 3, 4
LENS_RADTAN, LENS_EQUIDISTANT = 1, 2
PLANE_EXTRACT, PLANE_REFIT = 0, 1
PLANE_ACCEPTED, PLANE_FEW_POINTS, PLANE_REJECTED = 0, 1, 2
SNAPSHOT_MAGIC, SNAPSHOT_VERSION = 1314084432, 1
IMU_EVENT_GYROSCOPE, IMU_EVENT_ACCELEROMETER, IMU_EVENT_CAMERA = 0, 1, 2
IMU_STREAM_KEEP, IMU_STREAM_SET, IMU_STREAM_CLEAR = 0, 1, 2
IMU_STREAM_MAX_QUEUE = 65536
IMU_STREAM_SNAPSHOT_MAGIC, IMU_STREAM_SNAPSHOT_VERSION = 1397315152, 1
IMU_STREAM_COV_DIRECT, IMU_STREAM_COV_FACTOR = 0, 1
IMU_STREAM_NO_STATE, IMU_STREAM_NO_COVARIANCE = 1, 2

c_i32p = C.POINTER(C.c_int32)
c_u8p = C.POINTER(C.c_uint8)
c_f64p = C.POINTER(C.c_double)
c_f32p = C.POINTER(C.c_float)


class CWindow(C.Structure):
    _fields_ = [
        ("n_frames", C.c_int32), ("n_landmarks", C.c_int32), ("n_obs", C.c_int32), ("use_inertial", C.c_int32),
        ("frame_fixed", c_u8p),
        ("cam_q_cs", C.c_double * 4), ("cam_p_cs", C.c_double * 3),
        ("imu_q_cs", C.c_double * 4), ("imu_p_cs", C.c_double * 3),
        ("sqrt_inv_cov", C.c_double * 4),
        ("fx", C.c_double), ("fy", C.c_double), ("cauchy_a", C.c_double),
        ("lm_anchor", c_i32p), ("lm_z_ref", c_f64p), ("lm_obs_begin", c_i32p), ("lm_in_victim", c_u8p),
        ("obs_frame", c_i32p), ("obs_z", c_f64p),
        ("n_imu", C.c_int32), ("imu_frame_i", c_i32p), ("imu_frame_j", c_i32p), ("imu_data", c_f64p),
        ("n_prior", C.c_int32), ("prior_frames", c_i32p), ("prior_S", c_f64p), ("prior_e", c_f64p),
        ("prior_state0", c_f64p),
        ("n_planes", C.c_int32), ("plane_param", c_f64p), ("plane_sqrt_inv_cov", C.c_double),
        ("n_plane_tracks", C.c_int32), ("pt_plane", c_i32p), ("pt_obs_begin", c_i32p), ("pt_obs_frame", c_i32p),
        ("pt_obs_z", c_f64p),
    ]


class CState(C.Structure):
    _fields_ = [("frames", c_f64p), ("inv_depth", c_f64p)]


class COptions(C.Structure):
    _fields_ = [("max_iterations", C.c_int32), ("max_time", C.c_double), ("alias_bias", C.c_int32),
                ("run_postpass", C.c_int32), ("initial_trust_region_radius", C.c_double)]


class CSummary(C.Structure):
    _fields_ = [("iterations", C.c_int32), ("accepted_steps", C.c_int32), ("termination", C.c_int32),
                ("usable", C.c_int32), ("initial_cost", C.c_double), ("final_cost", C.c_double),
                ("final_radius", C.c_double), ("final_mu", C.c_double), ("solve_seconds", C.c_double)]


class CPnpProblem(C.Structure):
    _fields_ = [("n_points", C.c_int32), ("use_inertial", C.c_int32), ("points", c_f64p), ("z", c_f64p),
                ("cam_q_cs", C.c_double * 4), ("cam_p_cs", C.c_double * 3), ("imu_q_cs", C.c_double * 4),
                ("imu_p_cs", C.c_double * 3), ("sqrt_inv_cov", C.c_double * 4), ("cauchy_a", C.c_double),
                ("last_frame", c_f64p), ("imu_data", c_f64p)]


class CKltPair(C.Structure):
    _fields_ = [("slot", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32),
                ("prev_id", C.c_uint64), ("next_id", C.c_uint64), ("prev", c_u8p), ("next", c_u8p),
                ("n_points", C.c_int32), ("prev_pts", c_f32p), ("next_pts", c_f32p), ("status", c_u8p),
                ("err", c_f32p), ("info", c_i32p)]


class CDetectRequest(C.Structure):
    _fields_ = [("slot", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32),
                ("frame_id", C.c_uint64), ("image", c_u8p), ("existing", c_f64p), ("n_existing", C.c_int32),
                ("max_out", C.c_int32), ("keypoint_distance", C.c_double), ("keypoints_out", c_f64p), ("n_out", c_i32p),
                ("gftt_out", c_f32p), ("n_gftt", c_i32p)]


class CFeatureFrame(C.Structure):
    _fields_ = [("slot", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32),
                ("frame_id", C.c_uint64), ("image", c_u8p), ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double),
                ("cy", C.c_double), ("map_frames", C.c_int32), ("max_keypoints", C.c_int32), ("predict_q", c_f64p),
                ("keypoints", c_f64p), ("prev_index", c_i32p), ("n_keypoints", c_i32p), ("counts", c_i32p),
                ("info", c_i32p)]


class CWindowEdit(C.Structure):
    _fields_ = [("slot", C.c_int32), ("replace_last", C.c_int32), ("state", c_f64p), ("fixed", C.c_int32),
                ("imu_record", c_f64p), ("n_new_tracks", C.c_int32), ("new_frame", c_i32p), ("new_z", c_f64p),
                ("new_inv_depth", c_f64p), ("new_ids", c_i32p), ("n_obs", C.c_int32), ("obs_track", c_i32p),
                ("obs_frame", c_i32p), ("obs_z", c_f64p), ("n_remove", C.c_int32), ("remove", c_i32p)]


class CWindowPlanes(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_planes", C.c_int32), ("plane_param", c_f64p), ("n_set", C.c_int32),
                ("track", c_i32p), ("role", c_i32p), ("inv_depth", c_f64p)]


class CWindowLocalize(C.Structure):
    _fields_ = [("slot", C.c_int32), ("use_inertial", C.c_int32), ("imu_record", c_f64p), ("state", c_f64p),
                ("n_obs", C.c_int32), ("obs_track", c_i32p), ("obs_z", c_f64p), ("obs_point", c_f64p),
                ("points_out", c_f64p), ("n_new", C.c_int32), ("new_z_last", c_f64p), ("new_z", c_f64p),
                ("new_valid", c_u8p), ("new_inv_depth", c_f64p), ("new_inv_depth_next", c_f64p),
                ("summary", C.POINTER(CSummary))]


class CWindowImu(C.Structure):
    _fields_ = [("slot", C.c_int32), ("frame", C.c_int32), ("n_samples", C.c_int32), ("samples", c_f64p),
                ("t_end", C.c_double), ("noise_cov", c_f64p)]


class CWindowTrackFrame(C.Structure):
    _fields_ = [("slot", C.c_int32), ("newest_is_keyframe", C.c_int32), ("n_samples", C.c_int32), ("n_merge", C.c_int32),
                ("samples", c_f64p), ("merge_samples", c_f64p), ("t_end", C.c_double), ("noise_cov", c_f64p),
                ("cx", C.c_double), ("cy", C.c_double), ("skipped_frames", c_i32p), ("state", c_f64p),
                ("predicted", c_f64p), ("imu_record", c_f64p), ("keyframe", c_u8p), ("parallax", c_f64p),
                ("n_parallax", c_i32p), ("n_obs", C.c_int32), ("obs_track", c_i32p), ("obs_z", c_f64p),
                ("obs_point", c_f64p), ("points_out", c_f64p), ("n_new", C.c_int32), ("new_z_last", c_f64p),
                ("new_z", c_f64p), ("new_valid", c_u8p), ("new_inv_depth", c_f64p), ("new_inv_depth_next", c_f64p),
                ("summary", C.POINTER(CSummary))]


class CWindowPlaneRansac(C.Structure):
    _fields_ = [("slot", C.c_int32), ("mode", C.c_int32), ("n_tracks", C.c_int32), ("tracks", c_i32p), ("info", c_i32p),
                ("plane", c_f64p), ("used", c_u8p), ("inlier", c_u8p), ("points", c_f64p), ("schedule", c_i32p),
                ("counts", c_i32p)]


class CWindowCovariance(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_frames", C.c_int32), ("frames", c_i32p), ("cov", c_f64p), ("n_tracks", C.c_int32),
                ("tracks", c_i32p), ("inv_depth_var", c_f64p), ("status", C.c_int32)]


class CWindowLandmarks(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_tracks", C.c_int32), ("tracks", c_i32p), ("capacity", C.c_int32),
                ("track_id", c_i32p), ("point", c_f64p), ("role", c_i32p), ("point_cov", c_f64p),
                ("inv_depth_var", c_f64p), ("n_rows", C.c_int32), ("status", C.c_int32)]


class CWindowTrajectory(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_times", C.c_int32), ("times", c_f64p), ("states", c_f64p), ("state_cov", c_f64p),
                ("frame", c_i32p), ("status", C.c_int32), ("pad", C.c_int32)]


class CWindowKeypoints(C.Structure):
    _fields_ = [("slot", C.c_int32), ("tracker_slot", C.c_int32), ("frame_id", C.c_uint64), ("n", C.c_int32),
                ("track", c_i32p), ("keypoint", c_i32p), ("newest_is_keyframe", C.c_int32), ("skipped_frames", C.c_int32)]


class CWindowMirror(C.Structure):
    _fields_ = [("slot", C.c_int32), ("tracker_slot", C.c_int32), ("n_samples", C.c_int32), ("keep_samples", C.c_int32),
                ("samples", c_f64p), ("t_end", C.c_double), ("noise_cov", c_f64p), ("cx", C.c_double), ("cy", C.c_double),
                ("n_given", C.c_int32), ("given_track", c_i32p), ("given_point", c_f64p), ("max_keypoints", C.c_int32),
                ("kp_track", c_i32p), ("counts", c_i32p), ("state", c_f64p), ("predicted", c_f64p),
                ("imu_record", c_f64p), ("keyframe", c_u8p), ("parallax", c_f64p), ("n_parallax", c_i32p),
                ("skipped_frames", c_i32p), ("summary", C.POINTER(CSummary))]


class CWindowCamera(C.Structure):
    _fields_ = [("slot", C.c_int32), ("tracker_slot", C.c_int32), ("frame_id", C.c_uint64), ("width", C.c_int32),
                ("height", C.c_int32), ("stride", C.c_int32), ("map_frames", C.c_int32), ("image", c_u8p),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("max_keypoints", C.c_int32), ("n_samples", C.c_int32), ("samples", c_f64p), ("t_end", C.c_double),
                ("noise_cov", c_f64p), ("keep_samples", C.c_int32), ("n_given", C.c_int32), ("given_track", c_i32p),
                ("given_point", c_f64p), ("n_keypoints", c_i32p), ("kp_track", c_i32p), ("counts", c_i32p),
                ("state", c_f64p), ("predicted", c_f64p), ("imu_record", c_f64p), ("keyframe", c_u8p),
                ("parallax", c_f64p), ("n_parallax", c_i32p), ("skipped_frames", c_i32p),
                ("summary", C.POINTER(CSummary)), ("keypoints", c_f64p), ("prev_index", c_i32p),
                ("feature_counts", c_i32p), ("info", c_i32p), ("predict_q", c_f64p)]


class CWindowSnapshot(C.Structure):
    _fields_ = [("slot", C.c_int32), ("tracker_slot", C.c_int32), ("data", c_u8p), ("capacity", C.c_int64),
                ("size", C.c_int64)]


class CImuStreamRecord(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_events", C.c_int32), ("events", c_f64p), ("state_op", C.c_int32),
                ("state_time", C.c_double), ("state", c_f64p), ("poses", c_f64p), ("max_frames", C.c_int32),
                ("max_rows", C.c_int64), ("frame_t", c_f64p), ("frame_rows", c_i32p), ("rows", c_f64p),
                ("n_consumed", C.c_int32), ("n_frames", C.c_int32), ("need_frames", C.c_int32), ("need_rows", C.c_int64)]


class CImuStreamSnapshot(C.Structure):
    _fields_ = [("slot", C.c_int32), ("pad", C.c_int32), ("data", c_u8p), ("capacity", C.c_int64), ("size", C.c_int64)]


class CImuStreamCovSeed(C.Structure):
    _fields_ = [("slot", C.c_int32), ("mode", C.c_int32), ("state_time", C.c_double), ("cov", c_f64p),
                ("imu_record", c_f64p), ("noise_cov", c_f64p)]


class CImuStreamPredict(C.Structure):
    _fields_ = [("slot", C.c_int32), ("n_times", C.c_int32), ("times", c_f64p), ("poses", c_f64p), ("states", c_f64p),
                ("pose_cov", c_f64p), ("state_cov", c_f64p), ("status", C.c_int32), ("pad", C.c_int32)]


class CLens(C.Structure):
    _fields_ = [("slot", C.c_int32), ("model", C.c_int32), ("width", C.c_int32), ("height", C.c_int32),
                ("fx", C.c_double), ("fy", C.c_double), ("cx", C.c_double), ("cy", C.c_double),
                ("coeffs", C.c_double * 4)]


class CUndistortRequest(C.Structure):
    _fields_ = [("slot", C.c_int32), ("width", C.c_int32), ("height", C.c_int32), ("stride", C.c_int32),
                ("src", c_u8p), ("dst", c_u8p)]


class CTwoView(C.Structure):
    _fields_ = [("n_matches", C.c_int32), ("seed", C.c_int32), ("p1", c_f64p), ("p2", c_f64p), ("fx", C.c_double),
                ("fy", C.c_double), ("min_matches", C.c_int32), ("min_triangulation", C.c_int32),
                ("min_parallax", C.c_double), ("confidence", C.c_double), ("max_iteration", C.c_int32), ("info", c_i32p),
                ("parallax", c_f64p), ("H", c_f64p), ("E", c_f64p), ("R", c_f64p), ("T", c_f64p), ("h_mask", c_u8p),
                ("e_mask", c_u8p), ("points", c_f64p), ("point_status", c_u8p), ("h_schedule", c_i32p),
                ("e_schedule", c_i32p), ("h_counts", c_i32p), ("e_counts", c_i32p)]


# ---- the signature table: name -> (restype, argtypes), in the header's order -----------------------------------------
_int, _i32, _i64, _u64, _f64, _h = C.c_int, C.c_int32, C.c_int64, C.c_uint64, C.c_double, C.c_void_p
_P = C.POINTER
_intp = _P(C.c_int)
SIGNATURES = {
    "pvio_b200_create": (_int, [_int, _int, _int, _int, _int, _P(_h)]),
    "pvio_b200_destroy": (None, [_h]),
    "pvio_b200_last_error": (C.c_char_p, [_h]),
    "pvio_b200_kernel_launches": (_i64, [_h]),
    "pvio_b200_version": (C.c_char_p, []),
    "pvio_b200_ba_solve": (_int, [_h, _P(CWindow), _P(CState), _P(COptions), _P(CSummary), c_u8p, c_f64p]),
    "pvio_b200_ba_gn_step": (_int, [_h, _P(CWindow), _P(CState), _f64, c_f64p, c_f64p, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_ba_marginalize": (_int, [_h, _P(CWindow), _P(CState), _int, c_f64p, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_window_reset": (_int, [_h, _P(CWindow)]),
    "pvio_b200_window_append_frame": (_int, [_h, c_f64p, _int, c_f64p]),
    "pvio_b200_window_add_tracks": (_int, [_h, _int, c_i32p, c_f64p, c_f64p, c_i32p]),
    "pvio_b200_window_add_observations": (_int, [_h, _int, c_i32p, c_i32p, c_f64p]),
    "pvio_b200_window_remove_track": (_int, [_h, _i32]),
    "pvio_b200_window_set_prior": (_int, [_h, _int, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_window_solve": (_int, [_h, _P(COptions), _P(CSummary)]),
    "pvio_b200_window_drop_victim": (_int, [_h]),
    "pvio_b200_window_get": (_int, [_h, c_i32p, c_f64p, _int, c_i32p, c_f64p, c_i32p, c_i32p]),
    "pvio_b200_reprojection_error": (_int, [_h, _P(CWindow), _P(CState), c_f64p]),
    "pvio_b200_batch_set_window": (_int, [_h, _int, _P(CWindow), _P(CState)]),
    "pvio_b200_batch_replicate": (_int, [_h, _int]),
    "pvio_b200_batch_upload": (_int, [_h, _int]),
    "pvio_b200_batch_gn_step": (_int, [_h, _int, _f64, _int]),
    "pvio_b200_batch_download": (_int, [_h, _int, c_f64p, _i64, c_f64p]),
    "pvio_b200_batch_gn_step_host": (_int, [_h, _int, _f64, c_f64p, _i64, c_f64p]),
    "pvio_b200_batch_solve": (_int, [_h, _int, _P(COptions)]),
    "pvio_b200_batch_download_state": (_int, [_h, _int, c_f64p, _i64, c_f64p, _i64, _P(CSummary)]),
    "pvio_b200_batch_solve_host": (_int, [_h, _int, _P(COptions), c_f64p, _i64, c_f64p, _i64, _P(CSummary)]),
    "pvio_b200_batch_marginalize": (_int, [_h, _int, c_f64p, _i64, c_f64p, _i64]),
    "pvio_b200_batch_window_reset": (_int, [_h, _int, _P(CWindow)]),
    "pvio_b200_batch_window_set_prior": (_int, [_h, _int, _int, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_batch_window_edit": (_int, [_h, _int, _P(CWindowEdit)]),
    "pvio_b200_batch_window_set_planes": (_int, [_h, _int, _P(CWindowPlanes)]),
    "pvio_b200_batch_window_solve": (_int, [_h, _int, c_i32p, _P(COptions), _P(CSummary)]),
    "pvio_b200_batch_window_drop_victim": (_int, [_h, _int, c_i32p, c_f64p, _i64, c_f64p, _i64]),
    "pvio_b200_batch_window_covariance": (_int, [_h, _int, _P(CWindowCovariance)]),
    "pvio_b200_batch_window_landmarks": (_int, [_h, _int, _P(CWindowLandmarks)]),
    "pvio_b200_batch_window_trajectory": (_int, [_h, _int, _P(CWindowTrajectory)]),
    "pvio_b200_batch_window_smoothed_trajectory": (_int, [_h, _int, _P(CWindowTrajectory)]),
    "pvio_b200_batch_window_download": (_int, [_h, _int, c_i32p, c_i32p, c_f64p, _i64, c_i32p, _i64, c_i32p, c_f64p,
                                               c_i32p, c_i32p, c_u8p, c_f64p]),
    "pvio_b200_batch_window_localize": (_int, [_h, _int, _P(CWindowLocalize), _P(COptions)]),
    "pvio_b200_batch_window_set_imu": (_int, [_h, _int, _P(CWindowImu)]),
    "pvio_b200_batch_window_imu_records": (_int, [_h, _int, c_i32p, c_f64p, _i64]),
    "pvio_b200_batch_window_track_frame": (_int, [_h, _int, _P(CWindowTrackFrame), _P(COptions)]),
    "pvio_b200_batch_window_plane_ransac": (_int, [_h, _int, _P(CWindowPlaneRansac)]),
    "pvio_b200_batch_window_set_keypoints": (_int, [_h, _int, _P(CWindowKeypoints)]),
    "pvio_b200_batch_window_mirror_frame": (_int, [_h, _int, _P(CWindowMirror), _P(COptions)]),
    "pvio_b200_batch_window_track_camera": (_int, [_h, _int, _P(CWindowCamera), _int, _int, _f64, _f64, _int, _int, _int,
                                                   _f64, _f64, _f64, _P(COptions)]),
    "pvio_b200_batch_window_save": (_int, [_h, _int, _P(CWindowSnapshot)]),
    "pvio_b200_batch_window_restore": (_int, [_h, _int, _P(CWindowSnapshot)]),
    "pvio_b200_batch_imu_stream_reset": (_int, [_h, _int, c_i32p, c_f64p, c_f64p]),
    "pvio_b200_batch_imu_stream": (_int, [_h, _int, _P(CImuStreamRecord)]),
    "pvio_b200_batch_imu_stream_save": (_int, [_h, _int, _P(CImuStreamSnapshot)]),
    "pvio_b200_batch_imu_stream_restore": (_int, [_h, _int, _P(CImuStreamSnapshot)]),
    "pvio_b200_batch_imu_stream_set_covariance": (_int, [_h, _int, _P(CImuStreamCovSeed)]),
    "pvio_b200_batch_imu_stream_predict": (_int, [_h, _int, _P(CImuStreamPredict)]),
    "pvio_b200_sync": (_int, [_h]),
    "pvio_b200_timer_start": (_int, [_h]),
    "pvio_b200_timer_stop": (_int, [_h, c_f32p]),
    "pvio_b200_last_kernel_ms": (_int, [_h, _int, c_f32p]),
    "pvio_b200_pnp_solve": (_int, [_h, _P(CPnpProblem), c_f64p, _P(COptions), _P(CSummary)]),
    "pvio_b200_batch_pnp_solve": (_int, [_h, _int, _P(CPnpProblem), c_f64p, _i64, _P(COptions), _P(CSummary)]),
    "pvio_b200_klt_track_raw": (_int, [_h, c_u8p, c_u8p, _int, _int, _int, c_f32p, c_f32p, c_u8p, c_f32p, _int, _int,
                                       _int, _f64, _f64, _int, _int, c_u8p, c_u8p]),
    "pvio_b200_klt_track_cached": (_int, [_h, _u64, c_u8p, _u64, c_u8p, _int, _int, _int, c_f32p, c_f32p, c_u8p, c_f32p,
                                          _int, _int, _int, _f64, _f64, _int, _int, _int]),
    "pvio_b200_detect_keypoints": (_int, [_h, _u64, c_u8p, _int, _int, _int, _f64, _int, _int, c_f64p, _int, _f64, _int,
                                          c_f64p, _intp, c_f32p, _intp]),
    "pvio_b200_find_fundamental_mask": (_int, [_h, _int, c_f32p, c_f32p, _f64, _f64, _int, c_i32p, _int, c_u8p, c_f64p,
                                               c_i32p]),
    "pvio_b200_fm_sample_schedule": (_int, [_int, c_f32p, c_f32p, _int, c_i32p]),
    "pvio_b200_track_keypoints": (_int, [_h, _u64, c_u8p, _u64, c_u8p, _int, _int, _int, c_f32p, c_f32p, c_u8p, _int,
                                         _int, _int, _f64, _f64, _int, _int, _int, _f64, _f64]),
    "pvio_b200_batch_track_keypoints": (_int, [_h, _int, _P(CKltPair), _int, _int, _f64, _f64, _int, _int, _int, _f64,
                                               _f64]),
    "pvio_b200_batch_detect_keypoints": (_int, [_h, _int, _P(CDetectRequest), _f64, _int, _int]),
    "pvio_b200_batch_feature_track": (_int, [_h, _int, _P(CFeatureFrame), _int, _int, _f64, _f64, _int, _int, _int, _f64,
                                             _f64, _f64]),
    "pvio_b200_batch_two_view": (_int, [_h, _int, _P(CTwoView)]),
    "pvio_b200_undistort_map": (_int, [_int, _int, _int, c_f64p, c_f64p, _P(C.c_int16), _P(C.c_uint16)]),
    "pvio_b200_batch_set_lens": (_int, [_h, _int, _P(CLens)]),
    "pvio_b200_batch_undistort": (_int, [_h, _int, _P(CUndistortRequest)]),
    "pvio_b200_clahe": (_int, [_h, c_u8p, _int, _int, _int, _f64, _int, _int, c_u8p]),
    "pvio_b200_preintegrate": (_int, [_h, _int, c_i32p, c_f64p, c_f64p, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_triangulate": (_int, [_h, _int, c_f64p, _int, c_i32p, c_i32p, c_f64p, c_f64p, c_u8p, c_f64p]),
    "pvio_b200_selftest_lie": (_int, [_h, _int, c_f64p, c_f64p]),
    "pvio_b200_selftest_eig": (_int, [_h, _int, c_i32p, c_f64p, c_f64p, c_f64p, c_f64p]),
    "pvio_b200_selftest_chol": (_int, [_h, _int, _int, c_i32p, c_f64p, c_f64p, c_f64p, c_i32p]),
    "pvio_b200_klt_track": (_int, [_h, c_u8p, c_u8p, _int, _int, _int, c_f32p, c_f32p, c_u8p, c_f32p, _int, _int, _int,
                                   _f64]),
}
EXPORTS = list(SIGNATURES)          # the header's entry points
# not in the header: force batch_gn_step's sub-batch count (tests/test_gpu_step_split.py, tools/step_overlap.py)
SIGNATURES["pvio_b200_internal_set_step_split"] = (_int, [_h, _int])
# tuning builds only (-DPVIO_SOLVE_STAMPS / -DPVIO_MARG_STAMPS, loaded through PVIO_B200_TUNE_LIB): bound when present
TUNING_SIGNATURES = {
    "pvio_b200_debug_solve_stamps": (_int, [_P(C.c_longlong)]),
    "pvio_b200_debug_marg_stamps": (_int, [_P(C.c_longlong)]),
}

_lib = None


def load():
    """Load the shared library and declare every entry point (raises if it was not built: no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -m pvio_b200.build` (nvcc, sm_90a). "
                           "pvio_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    for name, (restype, argtypes) in TUNING_SIGNATURES.items():
        if hasattr(lib, name):
            fn = getattr(lib, name)
            fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


# ---- typed pointers ---------------------------------------------------------------------------------------------------
_CTYPE = {np.dtype(np.float64): C.c_double, np.dtype(np.float32): C.c_float, np.dtype(np.int64): C.c_int64,
          np.dtype(np.int32): C.c_int32, np.dtype(np.int16): C.c_int16, np.dtype(np.uint16): C.c_uint16,
          np.dtype(np.uint8): C.c_uint8}


def ptr(a):
    """A pointer to the data of array `a`, typed by its dtype (None: NULL).  Raises on an array that is not
    C-contiguous; never copies."""
    if a is None:
        return None
    if not a.flags.c_contiguous:
        raise ValueError(f"a {a.dtype} array of shape {a.shape} is not C-contiguous")
    ct = _CTYPE.get(a.dtype)
    if ct is None:
        raise TypeError(f"no C type for a {a.dtype} array")
    return a.ctypes.data_as(C.POINTER(ct))


def _ptr(a, ctype):
    """ptr(a) for callers that name the element type; raises TypeError when a's dtype is not that type."""
    if a is not None and _CTYPE.get(a.dtype) is not ctype:
        raise TypeError(f"a {a.dtype} array is not a {ctype.__name__} array")
    return ptr(a)


def set_ptrs(rec, **arrays):
    """Point the pointer fields of struct `rec` at the arrays (None: NULL), each through ptr(); raises TypeError when
    an array's dtype is not the field's declared element type (ctypes refuses the assignment).  Returns rec."""
    for name, a in arrays.items():
        try:
            setattr(rec, name, ptr(a))
        except TypeError as e:
            raise TypeError(f"{type(rec).__name__}.{name} does not take a {a.dtype} array: {e}") from None
    return rec


def check_rows(a, n, stride, name):
    """Raises unless `a` is a C-contiguous float64 [n, stride] array: a caller's output buffer of a strided call."""
    if a.dtype != np.float64 or not a.flags.c_contiguous or a.shape != (n, stride):
        raise ValueError(f"{name} must be a C-contiguous float64 array of shape {(n, stride)}, "
                         f"not {a.dtype} {a.shape}{'' if a.flags.c_contiguous else ' (strided)'}")


def summary(sm):
    """A CSummary as a dict of its fields."""
    return {k: getattr(sm, k) for k, _ in CSummary._fields_}


def imu_records(dt, dq, dp, dv, sqrt_inv_cov, dq_dbg, dp_dbg, dp_dba, dv_dbg, dv_dba, bg0=None, ba0=None):
    """IMU factor records [n, IMU_STRIDE] in the header's layout (PVIO_B200_IMU_*) from the PreIntegrator outputs of n
    factors: dt [n], dq [n, 4] (x, y, z, w), dp, dv [n, 3], sqrt_inv_cov [n, 15, 15], the five bias Jacobians [n, 3, 3],
    and the bias linearisation point bg0, ba0 [n, 3] (None: left 0)."""
    n = np.size(dt)
    rec = np.zeros((n, IMU_STRIDE))
    rec[:, IMU_DT] = dt
    rec[:, IMU_DQ:IMU_DQ + 4] = dq
    rec[:, IMU_DP:IMU_DP + 3] = dp
    rec[:, IMU_DV:IMU_DV + 3] = dv
    rec[:, IMU_SQRT_INV_COV:IMU_SQRT_INV_COV + 225] = np.asarray(sqrt_inv_cov).reshape(n, 225)
    for o, m in ((IMU_DQ_DBG, dq_dbg), (IMU_DP_DBG, dp_dbg), (IMU_DP_DBA, dp_dba), (IMU_DV_DBG, dv_dbg),
                 (IMU_DV_DBA, dv_dba)):
        rec[:, o:o + 9] = np.asarray(m).reshape(n, 9)
    if bg0 is not None:
        rec[:, IMU_BG0:IMU_BG0 + 3] = bg0
        rec[:, IMU_BA0:IMU_BA0 + 3] = ba0
    return rec


def window_constants(win):
    """A CWindow holding only the constants of win (use_inertial, extrinsics, noise model, intrinsics); no arrays."""
    cw = CWindow()
    cw.use_inertial = 1 if win.use_inertial else 0
    cw.cam_q_cs[:] = list(win.cam_q_cs); cw.cam_p_cs[:] = list(win.cam_p_cs)
    cw.imu_q_cs[:] = list(win.imu_q_cs); cw.imu_p_cs[:] = list(win.imu_p_cs)
    cw.sqrt_inv_cov[:] = list(np.asarray(win.sqrt_inv_cov, dtype=np.float64).reshape(4))
    cw.fx, cw.fy, cw.cauchy_a = win.K_fx, win.K_fy, win.cauchy_a
    cw.plane_sqrt_inv_cov = getattr(win, "plane_sqrt_inv_cov", 0.0)
    return cw


class PackedArgs:
    """Keeps the contiguous NumPy arrays alive while a CWindow / CState points into them."""

    def __init__(self, win, st):
        k = self.keep = {}

        def arr(name, a, dt):
            k[name] = np.ascontiguousarray(a, dtype=dt)
            return k[name]

        cw = window_constants(win)
        cw.n_frames, cw.n_landmarks, cw.n_obs = win.N, win.M, win.K
        set_ptrs(cw, frame_fixed=arr("fixed", win.frame_fixed, np.uint8), lm_anchor=arr("anchor", win.lm_anchor, np.int32),
                 lm_z_ref=arr("zref", win.lm_z_ref, np.float64), lm_obs_begin=arr("ob", win.lm_obs_begin, np.int32),
                 lm_in_victim=arr("victim", win.lm_in_victim if len(win.lm_in_victim) == win.M else np.zeros(win.M),
                                  np.uint8),
                 obs_frame=arr("of", win.obs_frame, np.int32), obs_z=arr("oz", win.obs_z, np.float64))
        cw.n_imu = win.n_imu if win.use_inertial else 0
        if cw.n_imu > 0:
            rec = imu_records(win.imu_dt, win.imu_dq, win.imu_dp, win.imu_dv, win.imu_sqrt_inv_cov, win.imu_dq_dbg,
                              win.imu_dp_dbg, win.imu_dp_dba, win.imu_dv_dbg, win.imu_dv_dba, win.imu_bg0, win.imu_ba0)
            set_ptrs(cw, imu_data=arr("imu", rec, np.float64), imu_frame_i=arr("imui", win.imu_frame_i, np.int32),
                     imu_frame_j=arr("imuj", win.imu_frame_j, np.int32))
        cw.n_prior = win.n_prior if win.use_inertial else 0
        if cw.n_prior > 0:
            x0 = np.concatenate([win.prior_q0, win.prior_p0, win.prior_v0, win.prior_bg0, win.prior_ba0], axis=1)
            set_ptrs(cw, prior_frames=arr("pf", win.prior_frames, np.int32), prior_S=arr("pS", win.prior_S, np.float64),
                     prior_e=arr("pe", win.prior_e, np.float64), prior_state0=arr("px0", x0, np.float64))
        cw.n_planes = win.n_planes
        cw.n_plane_tracks = win.n_ptracks
        if win.n_ptracks > 0:
            pp = np.concatenate([win.plane_normal, win.plane_distance[:, None]], axis=1)
            set_ptrs(cw, plane_param=arr("pp", pp, np.float64), pt_plane=arr("ptp", win.pt_plane, np.int32),
                     pt_obs_begin=arr("ptb", win.pt_obs_begin, np.int32),
                     pt_obs_frame=arr("ptf", win.pt_obs_frame, np.int32), pt_obs_z=arr("ptz", win.pt_obs_z, np.float64))
        self.cw = cw
        frames = np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)
        self.cs = set_ptrs(CState(), frames=arr("frames", frames, np.float64),
                           inv_depth=arr("rho", np.array(st.rho, dtype=np.float64, copy=True), np.float64))
