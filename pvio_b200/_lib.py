"""ctypes loader for libpvio_b200.so (the C-ABI in include/pvio_b200.h).

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

IMU_STRIDE = 288
FRAME_STRIDE = 16

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


EXPORTS = [
    "pvio_b200_create", "pvio_b200_destroy", "pvio_b200_last_error", "pvio_b200_kernel_launches",
    "pvio_b200_version", "pvio_b200_ba_solve", "pvio_b200_ba_gn_step", "pvio_b200_ba_marginalize",
    "pvio_b200_reprojection_error", "pvio_b200_batch_set_window", "pvio_b200_batch_replicate",
    "pvio_b200_batch_upload", "pvio_b200_batch_gn_step", "pvio_b200_batch_download",
    "pvio_b200_batch_gn_step_host", "pvio_b200_sync", "pvio_b200_timer_start", "pvio_b200_timer_stop",
    "pvio_b200_last_kernel_ms", "pvio_b200_klt_track", "pvio_b200_pnp_solve", "pvio_b200_preintegrate",
    "pvio_b200_triangulate", "pvio_b200_klt_track_raw", "pvio_b200_clahe", "pvio_b200_batch_solve",
    "pvio_b200_batch_download_state", "pvio_b200_batch_solve_host", "pvio_b200_selftest_lie", "pvio_b200_klt_track_cached",
    "pvio_b200_window_reset", "pvio_b200_window_append_frame", "pvio_b200_window_add_tracks",
    "pvio_b200_window_add_observations", "pvio_b200_window_remove_track", "pvio_b200_window_set_prior",
    "pvio_b200_window_solve", "pvio_b200_window_drop_victim", "pvio_b200_window_get", "pvio_b200_detect_keypoints",
    "pvio_b200_find_fundamental_mask", "pvio_b200_track_keypoints", "pvio_b200_fm_sample_schedule",
    "pvio_b200_batch_marginalize", "pvio_b200_batch_pnp_solve", "pvio_b200_batch_track_keypoints",
    "pvio_b200_batch_detect_keypoints", "pvio_b200_selftest_eig", "pvio_b200_batch_window_reset",
    "pvio_b200_batch_window_set_prior", "pvio_b200_batch_window_edit", "pvio_b200_batch_window_solve",
    "pvio_b200_batch_window_drop_victim", "pvio_b200_batch_window_download", "pvio_b200_batch_window_set_planes",
    "pvio_b200_batch_window_localize", "pvio_b200_batch_window_set_imu", "pvio_b200_batch_window_imu_records",
    "pvio_b200_batch_window_track_frame", "pvio_b200_undistort_map", "pvio_b200_batch_set_lens", "pvio_b200_batch_undistort",
    "pvio_b200_batch_two_view",
]

_lib = None


def load():
    """Load the shared library (raises if it was not built: no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `python -m pvio_b200.build` (nvcc, sm_90a). "
                           "pvio_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    lib.pvio_b200_create.argtypes = [C.c_int] * 5 + [C.POINTER(vp)]
    lib.pvio_b200_create.restype = C.c_int
    lib.pvio_b200_destroy.argtypes = [vp]
    lib.pvio_b200_destroy.restype = None
    lib.pvio_b200_last_error.argtypes = [vp]
    lib.pvio_b200_last_error.restype = C.c_char_p
    lib.pvio_b200_kernel_launches.argtypes = [vp]
    lib.pvio_b200_kernel_launches.restype = C.c_int64
    lib.pvio_b200_version.restype = C.c_char_p
    lib.pvio_b200_ba_solve.argtypes = [vp, C.POINTER(CWindow), C.POINTER(CState), C.POINTER(COptions),
                                       C.POINTER(CSummary), c_u8p, c_f64p]
    lib.pvio_b200_ba_gn_step.argtypes = [vp, C.POINTER(CWindow), C.POINTER(CState), C.c_double, c_f64p, c_f64p,
                                         c_f64p, c_f64p, c_f64p]
    lib.pvio_b200_ba_marginalize.argtypes = [vp, C.POINTER(CWindow), C.POINTER(CState), C.c_int, c_f64p, c_f64p,
                                             c_f64p, c_f64p]
    lib.pvio_b200_reprojection_error.argtypes = [vp, C.POINTER(CWindow), C.POINTER(CState), c_f64p]
    lib.pvio_b200_batch_set_window.argtypes = [vp, C.c_int, C.POINTER(CWindow), C.POINTER(CState)]
    lib.pvio_b200_batch_replicate.argtypes = [vp, C.c_int]
    lib.pvio_b200_batch_upload.argtypes = [vp, C.c_int]
    lib.pvio_b200_batch_gn_step.argtypes = [vp, C.c_int, C.c_double, C.c_int]
    lib.pvio_b200_batch_download.argtypes = [vp, C.c_int, c_f64p, C.c_int64, c_f64p]
    lib.pvio_b200_batch_gn_step_host.argtypes = [vp, C.c_int, C.c_double, c_f64p, C.c_int64, c_f64p]
    lib.pvio_b200_batch_solve.argtypes = [vp, C.c_int, C.POINTER(COptions)]
    lib.pvio_b200_batch_download_state.argtypes = [vp, C.c_int, c_f64p, C.c_int64, c_f64p, C.c_int64, C.POINTER(CSummary)]
    lib.pvio_b200_batch_solve_host.argtypes = [vp, C.c_int, C.POINTER(COptions), c_f64p, C.c_int64, c_f64p, C.c_int64,
                                               C.POINTER(CSummary)]
    lib.pvio_b200_batch_marginalize.argtypes = [vp, C.c_int, c_f64p, C.c_int64, c_f64p, C.c_int64]
    lib.pvio_b200_selftest_lie.argtypes = [vp, C.c_int, c_f64p, c_f64p]
    lib.pvio_b200_selftest_eig.argtypes = [vp, C.c_int, c_i32p, c_f64p, c_f64p, c_f64p, c_f64p]
    lib.pvio_b200_sync.argtypes = [vp]
    lib.pvio_b200_timer_start.argtypes = [vp]
    lib.pvio_b200_timer_stop.argtypes = [vp, c_f32p]
    lib.pvio_b200_last_kernel_ms.argtypes = [vp, C.c_int, c_f32p]
    # internal, not in the header: force batch_gn_step's sub-batch count (tests/test_gpu_step_split.py, tools/)
    lib.pvio_b200_internal_set_step_split.argtypes = [vp, C.c_int]
    lib.pvio_b200_internal_set_step_split.restype = C.c_int
    lib.pvio_b200_pnp_solve.argtypes = [vp, C.POINTER(CPnpProblem), c_f64p, C.POINTER(COptions), C.POINTER(CSummary)]
    lib.pvio_b200_batch_pnp_solve.argtypes = [vp, C.c_int, C.POINTER(CPnpProblem), c_f64p, C.c_int64,
                                              C.POINTER(COptions), C.POINTER(CSummary)]
    lib.pvio_b200_batch_track_keypoints.argtypes = [vp, C.c_int, C.POINTER(CKltPair), C.c_int, C.c_int, C.c_double,
                                                    C.c_double, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double]
    lib.pvio_b200_batch_detect_keypoints.argtypes = [vp, C.c_int, C.POINTER(CDetectRequest), C.c_double, C.c_int, C.c_int]
    lib.pvio_b200_undistort_map.argtypes = [C.c_int, C.c_int, C.c_int, c_f64p, c_f64p, C.POINTER(C.c_int16),
                                            C.POINTER(C.c_uint16)]
    lib.pvio_b200_batch_set_lens.argtypes = [vp, C.c_int, C.POINTER(CLens)]
    lib.pvio_b200_batch_undistort.argtypes = [vp, C.c_int, C.POINTER(CUndistortRequest)]
    lib.pvio_b200_batch_two_view.argtypes = [vp, C.c_int, C.POINTER(CTwoView)]
    lib.pvio_b200_klt_track.argtypes = [vp, c_u8p, c_u8p, C.c_int, C.c_int, C.c_int, c_f32p, c_f32p, c_u8p, c_f32p,
                                        C.c_int, C.c_int, C.c_int, C.c_double]
    for name in EXPORTS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("pvio_b200_create",):
            fn.restype = C.c_int
    _lib = lib
    return lib


def _ptr(a, ctype):
    return a.ctypes.data_as(C.POINTER(ctype))


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
        cw.frame_fixed = _ptr(arr("fixed", win.frame_fixed, np.uint8), C.c_uint8)
        cw.lm_anchor = _ptr(arr("anchor", win.lm_anchor, np.int32), C.c_int32)
        cw.lm_z_ref = _ptr(arr("zref", win.lm_z_ref, np.float64), C.c_double)
        cw.lm_obs_begin = _ptr(arr("ob", win.lm_obs_begin, np.int32), C.c_int32)
        cw.lm_in_victim = _ptr(arr("victim", win.lm_in_victim if len(win.lm_in_victim) == win.M
                                   else np.zeros(win.M), np.uint8), C.c_uint8)
        cw.obs_frame = _ptr(arr("of", win.obs_frame, np.int32), C.c_int32)
        cw.obs_z = _ptr(arr("oz", win.obs_z, np.float64), C.c_double)
        cw.n_imu = win.n_imu if win.use_inertial else 0
        if cw.n_imu > 0:
            rec = np.zeros((win.n_imu, IMU_STRIDE))
            rec[:, 0] = win.imu_dt
            rec[:, 1:5] = win.imu_dq
            rec[:, 5:8] = win.imu_dp
            rec[:, 8:11] = win.imu_dv
            rec[:, 11:236] = win.imu_sqrt_inv_cov.reshape(win.n_imu, 225)
            rec[:, 236:245] = win.imu_dq_dbg.reshape(win.n_imu, 9)
            rec[:, 245:254] = win.imu_dp_dbg.reshape(win.n_imu, 9)
            rec[:, 254:263] = win.imu_dp_dba.reshape(win.n_imu, 9)
            rec[:, 263:272] = win.imu_dv_dbg.reshape(win.n_imu, 9)
            rec[:, 272:281] = win.imu_dv_dba.reshape(win.n_imu, 9)
            rec[:, 281:284] = win.imu_bg0
            rec[:, 284:287] = win.imu_ba0
            cw.imu_data = _ptr(arr("imu", rec, np.float64), C.c_double)
            cw.imu_frame_i = _ptr(arr("imui", win.imu_frame_i, np.int32), C.c_int32)
            cw.imu_frame_j = _ptr(arr("imuj", win.imu_frame_j, np.int32), C.c_int32)
        cw.n_prior = win.n_prior if win.use_inertial else 0
        if cw.n_prior > 0:
            x0 = np.concatenate([win.prior_q0, win.prior_p0, win.prior_v0, win.prior_bg0, win.prior_ba0], axis=1)
            cw.prior_frames = _ptr(arr("pf", win.prior_frames, np.int32), C.c_int32)
            cw.prior_S = _ptr(arr("pS", win.prior_S, np.float64), C.c_double)
            cw.prior_e = _ptr(arr("pe", win.prior_e, np.float64), C.c_double)
            cw.prior_state0 = _ptr(arr("px0", x0, np.float64), C.c_double)
        cw.n_planes = win.n_planes
        cw.n_plane_tracks = win.n_ptracks
        if win.n_ptracks > 0:
            pp = np.concatenate([win.plane_normal, win.plane_distance[:, None]], axis=1)
            cw.plane_param = _ptr(arr("pp", pp, np.float64), C.c_double)
            cw.pt_plane = _ptr(arr("ptp", win.pt_plane, np.int32), C.c_int32)
            cw.pt_obs_begin = _ptr(arr("ptb", win.pt_obs_begin, np.int32), C.c_int32)
            cw.pt_obs_frame = _ptr(arr("ptf", win.pt_obs_frame, np.int32), C.c_int32)
            cw.pt_obs_z = _ptr(arr("ptz", win.pt_obs_z, np.float64), C.c_double)
        self.cw = cw
        frames = np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)
        cs = CState()
        cs.frames = _ptr(arr("frames", frames, np.float64), C.c_double)
        cs.inv_depth = _ptr(arr("rho", np.array(st.rho, dtype=np.float64, copy=True), np.float64), C.c_double)
        self.cs = cs
