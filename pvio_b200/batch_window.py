"""Resident sliding windows of many sequences (include/pvio_b200.h "resident batched windows", csrc/batch_window.cu): each
slot keeps one sequence's window on the device; per camera frame the caller sends only the edits, solves and
marginalises the slots that take a keyframe, and reads back states, inverse depths and post-pass flags in one copy."""
import ctypes as C

import numpy as np

from . import _lib

_constants = _lib.window_constants            # the CWindow a reset takes: the window's constants only


class Edit:
    """One camera frame of one slot (pvio_b200_window_edit), built up by the caller:
    replace_last, frame(state16, fixed, imu_record), new tracks (frame, z, inv_depth), observations (id, frame, z),
    removals (ids)."""

    def __init__(self, slot, replace_last=False):
        self.slot, self.replace_last = int(slot), bool(replace_last)
        self.state, self.fixed, self.imu = None, False, None
        self.new, self.obs, self.remove = [], [], []

    def frame(self, state16, fixed=False, imu_record=None):
        self.state, self.fixed = np.ascontiguousarray(state16, dtype=np.float64), bool(fixed)
        self.imu = None if imu_record is None else np.ascontiguousarray(imu_record, dtype=np.float64)
        return self


# roles of a track (pvio_b200_window_planes): a landmark; a landmark kept out of the marginaliser's victim set (TF_PLANE
# on a plane with fewer than 20 tracks); a plane index p >= 0 makes the track a plane track of plane p
LANDMARK, SMALL_PLANE = -1, -2


class Planes:
    """The plane factors of one slot (pvio_b200_window_planes), built up by the caller: the slot's planes (None: keep
    them), and per track a role (LANDMARK, SMALL_PLANE or a plane index) with an optional new inverse depth."""

    def __init__(self, slot, planes=None):
        self.slot = int(slot)
        self.planes = None if planes is None else np.ascontiguousarray(planes, dtype=np.float64).reshape(-1, 4)
        self.tracks, self.roles, self.rho = [], [], []

    def role(self, track, role, inv_depth=np.nan):
        self.tracks.append(int(track)); self.roles.append(int(role)); self.rho.append(float(inv_depth))
        return self


class Localize:
    """One new camera frame of one slot (pvio_b200_window_localize), before the edit that appends it: the predicted
    state, the IMU record from the slot's newest frame (None: a visual-only PnP), the frame's keypoints on live tracks
    of the slot (id, z, and a world point for a plane track), and the keypoint pairs of the tracks born in the frame
    (z in the slot's newest frame, z in the new frame)."""

    def __init__(self, slot, state16, imu_record=None):
        self.slot = int(slot)
        self.state = np.array(state16, dtype=np.float64, copy=True)
        self.imu = None if imu_record is None else np.ascontiguousarray(imu_record, dtype=np.float64)
        self.obs, self.new = [], []

    def observe(self, track, z, point=None):
        self.obs.append((int(track), z, point))
        return self

    def born(self, z_last, z):
        self.new.append((z_last, z))
        return self


class TrackFrame(Localize):
    """One new camera frame of one inertial slot (pvio_b200_window_track_frame): its raw samples [K][7] up to t_end with
    noise_cov (as Imu takes them), the principal point (cx, cy), whether the slot's newest frame is a keyframe, and
    otherwise the newest frame's own samples (merge_samples); the tracker's skipped-frame counter; the keypoints as
    Localize's observe / born.  The call integrates, predicts, solves the PnP, triangulates and checks for a keyframe."""

    def __init__(self, slot, samples, t_end, noise_cov, cx, cy, newest_is_keyframe=True, merge_samples=None,
                 skipped_frames=0):
        super().__init__(slot, np.full(16, np.nan))
        self.samples = np.ascontiguousarray(np.asarray(samples, dtype=np.float64).reshape(-1, 7))
        self.t_end, self.cx, self.cy = float(t_end), float(cx), float(cy)
        self.noise = np.ascontiguousarray(np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in noise_cov]))
        self.newest_is_keyframe = bool(newest_is_keyframe)
        self.merge = None if merge_samples is None else np.ascontiguousarray(
            np.asarray(merge_samples, dtype=np.float64).reshape(-1, 7))
        self.skipped = int(skipped_frames)


def _localize_fields(r, L, o, keep):
    """the observation and new-track fields of a localize / track_frame ctypes record r from L, outputs into dict o"""
    if L.obs:
        t = np.array([b[0] for b in L.obs], dtype=np.int32)
        z = np.ascontiguousarray([b[1] for b in L.obs], dtype=np.float64).reshape(-1, 2)
        x = np.array([np.full(3, np.nan) if b[2] is None else b[2] for b in L.obs], dtype=np.float64).reshape(-1, 3)
        keep += [t, z, x]
        r.n_obs = len(t)
        _lib.set_ptrs(r, obs_track=t, obs_z=z, obs_point=x, points_out=o["points"])
    if L.new:
        zl = np.ascontiguousarray([b[0] for b in L.new], dtype=np.float64).reshape(-1, 2)
        zn = np.ascontiguousarray([b[1] for b in L.new], dtype=np.float64).reshape(-1, 2)
        keep += [zl, zn]
        r.n_new = len(zl)
        _lib.set_ptrs(r, new_z_last=zl, new_z=zn, new_valid=o["valid"], new_inv_depth=o["inv_depth"],
                      new_inv_depth_next=o["inv_depth_next"])


def _localize_out(L):
    return dict(state=L.state.copy(), points=np.zeros((len(L.obs), 3)), valid=np.zeros(len(L.new), dtype=np.uint8),
                inv_depth=np.zeros(len(L.new)), inv_depth_next=np.zeros(len(L.new)))


class PlaneRansac:
    """One plane RANSAC on one slot (pvio_b200_window_plane_ransac): mode EXTRACT (PlaneExtractor::work, the candidates'
    landmark points) or REFIT (Plane::update_parameter(true), the candidates triangulated over their window views), and
    the candidate track ids in the caller's order (Map order for an extraction, plane->tracks order for a refit)."""

    EXTRACT, REFIT = _lib.PLANE_EXTRACT, _lib.PLANE_REFIT

    def __init__(self, slot, mode, tracks):
        self.slot, self.mode = int(slot), int(mode)
        self.tracks = np.ascontiguousarray(tracks, dtype=np.int32).reshape(-1)


class Imu:
    """The raw samples of one IMU factor of one slot (pvio_b200_window_imu): window frame j >= 1 (the factor (j - 1, j)),
    samples [K][7] (t, w xyz, a xyz), t_end (the time of frame j) and noise_cov (cov_w, cov_a, cov_bg, cov_ba, 3x3 each
    or [4][9]).  The slot re-integrates the factor from them before every solve that names it."""

    def __init__(self, slot, frame, samples, t_end, noise_cov):
        self.slot, self.frame, self.t_end = int(slot), int(frame), float(t_end)
        self.samples = np.ascontiguousarray(np.asarray(samples, dtype=np.float64).reshape(-1, 7))
        self.noise = np.ascontiguousarray(np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in noise_cov]))


class Mirror:
    """One new camera frame of one linked inertial slot (pvio_b200_window_mirror), right after batch_feature_track
    advanced its tracker slot: the raw samples [K][7] up to t_end with noise_cov, the principal point, whether the new
    factor keeps its samples, and the given world points {track id: point [3]} of plane tracks."""

    def __init__(self, slot, tracker_slot, samples, t_end, noise_cov, cx, cy, keep_samples=True, given=None):
        self.slot, self.tracker_slot = int(slot), int(tracker_slot)
        self.samples = np.ascontiguousarray(np.asarray(samples, dtype=np.float64).reshape(-1, 7))
        self.t_end, self.cx, self.cy, self.keep = float(t_end), float(cx), float(cy), bool(keep_samples)
        self.noise = np.ascontiguousarray(np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in noise_cov]))
        self.given = dict(given or {})


class Camera(Mirror):
    """One new camera frame of one linked inertial slot (pvio_b200_window_camera) for track_camera: the raw image
    (uint8 [h, w]) with frame_id, K (fx, fy, cx, cy; fx, fy as the slot's) and map_frames (> 0) for the tracker slot,
    and the Mirror fields; samples are the frame's list after the prepend rule of feature_tracker.cpp:78-84."""

    def __init__(self, slot, tracker_slot, frame_id, image, K, map_frames, samples, t_end, noise_cov,
                 keep_samples=True, given=None):
        super().__init__(slot, tracker_slot, samples, t_end, noise_cov, K[2], K[3], keep_samples, given)
        self.frame_id, self.map_frames = int(frame_id), int(map_frames)
        self.image = np.ascontiguousarray(image, dtype=np.uint8)
        self.K = tuple(float(v) for v in K)


def _mirror_out(max_keypoints):
    """the output arrays of one mirror_frame record (kp_track filled with -7, the rest zero)"""
    return dict(kp_track=np.full(max_keypoints, -7, dtype=np.int32), counts=np.zeros(4, dtype=np.int32),
                state=np.zeros(16), predicted=np.zeros(16), imu_record=np.zeros(_lib.IMU_STRIDE),
                keyframe=np.zeros(1, dtype=np.uint8), parallax=np.zeros(1), n_parallax=np.zeros(1, dtype=np.int32),
                skipped_frames=np.zeros(1, dtype=np.int32))


class BatchWindows:
    def __init__(self, ba):
        """ba: a BundleAdjustor (owns the device handle and its max_windows slots)."""
        self.ba, self.lib, self.h = ba, ba.lib, ba.h

    def reset(self, slot, win):
        """Start an empty resident window in `slot`; `win` carries the constants (its arrays are not used)."""
        self.ba._ck(self.lib.pvio_b200_batch_window_reset(self.h, int(slot), C.byref(_constants(win))))

    def set_prior(self, slot, S, e, state0):
        S = np.ascontiguousarray(S, dtype=np.float64); e = np.ascontiguousarray(e, dtype=np.float64)
        x0 = np.ascontiguousarray(state0, dtype=np.float64).reshape(-1, 16)
        self.ba._ck(self.lib.pvio_b200_batch_window_set_prior(self.h, int(slot), len(x0), _lib.ptr(S), _lib.ptr(e),
                                                              _lib.ptr(x0)))

    def edit(self, edits):
        """Apply a list of Edit (distinct slots) in one call; returns the new track ids of each edit."""
        keep, recs = [], (_lib.CWindowEdit * max(len(edits), 1))()
        ids = []
        for i, e in enumerate(edits):
            r = recs[i]
            r.slot, r.replace_last = e.slot, 1 if e.replace_last else 0
            if e.state is not None:
                keep += [e.state, e.imu]
                _lib.set_ptrs(r, state=e.state, imu_record=e.imu)
                r.fixed = 1 if e.fixed else 0
            out = np.zeros(max(len(e.new), 1), dtype=np.int32)
            ids.append(out)
            if e.new:
                f = np.array([t[0] for t in e.new], dtype=np.int32)
                z = np.ascontiguousarray([t[1] for t in e.new], dtype=np.float64).reshape(-1, 2)
                rho = np.array([t[2] for t in e.new], dtype=np.float64)
                keep += [f, z, rho]
                r.n_new_tracks = len(e.new)
                _lib.set_ptrs(r, new_frame=f, new_z=z, new_inv_depth=rho, new_ids=out)
            if e.obs:
                t = np.array([o[0] for o in e.obs], dtype=np.int32)
                f = np.array([o[1] for o in e.obs], dtype=np.int32)
                z = np.ascontiguousarray([o[2] for o in e.obs], dtype=np.float64).reshape(-1, 2)
                keep += [t, f, z]
                r.n_obs = len(e.obs)
                _lib.set_ptrs(r, obs_track=t, obs_frame=f, obs_z=z)
            if e.remove:
                rm = np.array(e.remove, dtype=np.int32)
                keep.append(rm)
                r.n_remove = len(rm)
                _lib.set_ptrs(r, remove=rm)
        self.ba._ck(self.lib.pvio_b200_batch_window_edit(self.h, len(edits), recs))
        return [o[:len(e.new)].copy() for o, e in zip(ids, edits)]

    def set_planes(self, records):
        """Apply a list of Planes (distinct slots) in one call."""
        keep, recs = [], (_lib.CWindowPlanes * max(len(records), 1))()
        for i, p in enumerate(records):
            r = recs[i]
            r.slot = p.slot
            if p.planes is None:
                r.n_planes = -1
            else:
                keep.append(p.planes)
                r.n_planes = len(p.planes)
                _lib.set_ptrs(r, plane_param=p.planes)
            if p.tracks:
                t, ro = np.array(p.tracks, dtype=np.int32), np.array(p.roles, dtype=np.int32)
                rho = np.array(p.rho, dtype=np.float64)
                keep += [t, ro, rho]
                r.n_set = len(t)
                _lib.set_ptrs(r, track=t, role=ro, inv_depth=rho)
        self.ba._ck(self.lib.pvio_b200_batch_window_set_planes(self.h, len(records), recs))

    def localize(self, records, max_iterations=10, initial_radius=0.0):
        """PnP and new-track triangulation of a list of Localize (distinct slots) in one call; the slots do not change.
        Per record a dict: state [16], summary, points [n_obs, 3] (NaN: left out of the PnP), and per new track valid,
        inv_depth (in the slot's newest frame) and inv_depth_next (in the new frame)."""
        keep, out, n = [], [], len(records)
        recs, sms = (_lib.CWindowLocalize * max(n, 1))(), (_lib.CSummary * max(n, 1))()
        for i, L in enumerate(records):
            r = recs[i]
            o = _localize_out(L)
            out.append(o)
            r.slot, r.summary = L.slot, C.pointer(sms[i])
            keep.append(L.imu)
            _lib.set_ptrs(r, state=o["state"], imu_record=L.imu)
            r.use_inertial = 0 if L.imu is None else 1
            _localize_fields(r, L, o, keep)
        opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
        self.ba._ck(self.lib.pvio_b200_batch_window_localize(self.h, n, recs, C.byref(opt)))
        for i, o in enumerate(out):
            o["summary"] = _lib.summary(sms[i])
            o["valid"] = o["valid"].astype(bool)
        return out

    def track_frame(self, records, max_iterations=10, initial_radius=0.0):
        """Integrate, predict, PnP, triangulate and keyframe-check a list of TrackFrame (distinct inertial slots) in one
        call; the slots do not change.  Per record what localize returns, plus predicted [16], imu_record [288] (the
        factor of the frame edit), keyframe, parallax (NaN with fewer than 50 pairs), n_parallax and skipped_frames."""
        recs, sms, out, keep = self.track_frame_records(records)
        opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
        self.ba._ck(self.lib.pvio_b200_batch_window_track_frame(self.h, len(records), recs, C.byref(opt)))
        for i, o in enumerate(out):
            o["summary"] = _lib.summary(sms[i])
            o["valid"] = o["valid"].astype(bool)
            o["keyframe"], o["parallax"] = bool(o["keyframe"][0]), float(o["parallax"][0])
            o["n_parallax"], o["skipped_frames"] = int(o["n_parallax"][0]), int(o["skipped_frames"][0])
        return out

    @staticmethod
    def track_frame_records(records):
        """the ctypes records of a list of TrackFrame: (records, summaries, output arrays per record, arrays to keep)"""
        keep, out, n = [], [], len(records)
        recs, sms = (_lib.CWindowTrackFrame * max(n, 1))(), (_lib.CSummary * max(n, 1))()
        for i, T in enumerate(records):
            r = recs[i]
            o = _localize_out(T)
            o.update(predicted=np.zeros(16), imu_record=np.zeros(_lib.IMU_STRIDE), keyframe=np.zeros(1, dtype=np.uint8),
                     parallax=np.zeros(1), n_parallax=np.zeros(1, dtype=np.int32),
                     skipped_frames=np.array([T.skipped], dtype=np.int32))
            out.append(o)
            r.slot, r.newest_is_keyframe = T.slot, 1 if T.newest_is_keyframe else 0
            r.n_samples, r.n_merge, r.t_end = len(T.samples), 0 if T.merge is None else len(T.merge), T.t_end
            r.cx, r.cy, r.summary = T.cx, T.cy, C.pointer(sms[i])
            _lib.set_ptrs(r, samples=T.samples, merge_samples=T.merge, noise_cov=T.noise,
                          skipped_frames=o["skipped_frames"], state=o["state"], predicted=o["predicted"],
                          imu_record=o["imu_record"], keyframe=o["keyframe"], parallax=o["parallax"],
                          n_parallax=o["n_parallax"])
            keep += [T.samples, T.noise] + ([] if T.merge is None else [T.merge])
            _localize_fields(r, T, o, keep)
        return recs, sms, out, keep

    def set_keypoints(self, slot, tracker_slot, frame_id, pairs, newest_is_keyframe=True, skipped_frames=0):
        """Link `slot`'s newest frame to frame `frame_id` of tracker slot `tracker_slot`: pairs {track id: keypoint
        index in that frame} for the live tracks observed there."""
        t = np.array(list(pairs), dtype=np.int32)
        k = np.array([pairs[i] for i in pairs], dtype=np.int32)
        r = _lib.CWindowKeypoints()
        r.slot, r.tracker_slot, r.frame_id, r.n = int(slot), int(tracker_slot), int(frame_id), len(t)
        r.newest_is_keyframe, r.skipped_frames = 1 if newest_is_keyframe else 0, int(skipped_frames)
        _lib.set_ptrs(r, track=t, keypoint=k)
        self.ba._ck(self.lib.pvio_b200_batch_window_set_keypoints(self.h, 1, C.byref(r)))

    def mirror_frame(self, records, max_keypoints, max_iterations=10, initial_radius=0.0):
        """mirror_frame + track_frame + the frame edit of a list of Mirror (distinct slots and tracker slots) in one
        call.  Per record a dict: kp_track [max_keypoints] (the track of each new-frame keypoint, -1: none; only the
        tracker's keypoint count is written), counts [4] (continued, PnP observations, candidates, new tracks), state,
        predicted, imu_record, keyframe, parallax, n_parallax, skipped_frames, summary."""
        recs, sms, out, keep = self.mirror_records(records, max_keypoints)
        opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
        self.ba._ck(self.lib.pvio_b200_batch_window_mirror_frame(self.h, len(records), recs, C.byref(opt)))
        for i, o in enumerate(out):
            o["summary"] = _lib.summary(sms[i])
            o["keyframe"], o["parallax"] = bool(o["keyframe"][0]), float(o["parallax"][0])
            o["n_parallax"], o["skipped_frames"] = int(o["n_parallax"][0]), int(o["skipped_frames"][0])
        return out

    def track_camera(self, records, max_keypoints, keypoint_distance=20.0, max_level=3, max_iter=30, eps=0.01,
                     clahe_clip=6.0, clahe_tiles=(8, 8), border=20, ransac_threshold=1.0, ransac_confidence=0.99,
                     max_iterations=10, initial_radius=0.0):
        """batch_feature_track with the IMU prediction made on the device, then mirror_frame, of a list of Camera
        (distinct slots and tracker slots) in one call.  Per record mirror_frame's dict plus n_keypoints, keypoints
        [n_keypoints][2], prev_index [n_keypoints], feature_counts [4], info [4] and predict_q [4] (the delta_key_q
        used)."""
        recs, sms, out, keep = self.camera_records(records, max_keypoints)
        opt = _lib.COptions(max_iterations, 1e6, 1, 0, initial_radius)
        self.ba._ck(self.lib.pvio_b200_batch_window_track_camera(
            self.h, len(records), recs, int(max_level), int(max_iter), float(eps), float(clahe_clip),
            int(clahe_tiles[0]), int(clahe_tiles[1]), int(border), float(ransac_threshold), float(ransac_confidence),
            float(keypoint_distance), C.byref(opt)))
        for i, o in enumerate(out):
            m = int(o["n_keypoints"][0])
            o["n_keypoints"], o["keypoints"], o["prev_index"] = m, o["keypoints"][:m], o["prev_index"][:m]
            o["summary"] = _lib.summary(sms[i])
            o["keyframe"], o["parallax"] = bool(o["keyframe"][0]), float(o["parallax"][0])
            o["n_parallax"], o["skipped_frames"] = int(o["n_parallax"][0]), int(o["skipped_frames"][0])
        return out

    @staticmethod
    def camera_records(records, max_keypoints):
        """the ctypes records of a list of Camera: (records, summaries, output arrays per record, arrays to keep)"""
        keep, out, n = [], [], len(records)
        recs, sms = (_lib.CWindowCamera * max(n, 1))(), (_lib.CSummary * max(n, 1))()
        for i, M in enumerate(records):
            r = recs[i]
            o = _mirror_out(max_keypoints)
            o.update(n_keypoints=np.full(1, -7, dtype=np.int32), keypoints=np.full((max_keypoints, 2), -7.0),
                     prev_index=np.full(max_keypoints, -7, dtype=np.int32), feature_counts=np.zeros(4, dtype=np.int32),
                     info=np.zeros(4, dtype=np.int32), predict_q=np.zeros(4))
            out.append(o)
            h, w = M.image.shape
            r.slot, r.tracker_slot, r.frame_id, r.width, r.height, r.stride = M.slot, M.tracker_slot, M.frame_id, w, h, w
            r.map_frames, (r.fx, r.fy, r.cx, r.cy), r.max_keypoints = M.map_frames, M.K, int(max_keypoints)
            r.n_samples, r.t_end, r.keep_samples, r.summary = len(M.samples), M.t_end, int(M.keep), C.pointer(sms[i])
            gt = np.array(list(M.given), dtype=np.int32)
            gp = np.ascontiguousarray([M.given[t] for t in M.given], dtype=np.float64).reshape(-1, 3)
            r.n_given = len(gt)
            keep += [M.image, M.samples, M.noise, gt, gp]
            _lib.set_ptrs(r, image=M.image, samples=M.samples, noise_cov=M.noise, given_track=gt if len(gt) else None,
                          given_point=gp if len(gt) else None, **{k: o[k] for k in o})
        return recs, sms, out, keep

    @staticmethod
    def mirror_records(records, max_keypoints):
        """the ctypes records of a list of Mirror: (records, summaries, output arrays per record, arrays to keep)"""
        keep, out, n = [], [], len(records)
        recs, sms = (_lib.CWindowMirror * max(n, 1))(), (_lib.CSummary * max(n, 1))()
        for i, M in enumerate(records):
            r = recs[i]
            o = _mirror_out(max_keypoints)
            out.append(o)
            r.slot, r.tracker_slot, r.n_samples, r.keep_samples = M.slot, M.tracker_slot, len(M.samples), int(M.keep)
            r.t_end, r.cx, r.cy, r.max_keypoints, r.summary = M.t_end, M.cx, M.cy, int(max_keypoints), C.pointer(sms[i])
            gt = np.array(list(M.given), dtype=np.int32)
            gp = np.ascontiguousarray([M.given[t] for t in M.given], dtype=np.float64).reshape(-1, 3)
            r.n_given = len(gt)
            keep += [M.samples, M.noise, gt, gp]
            _lib.set_ptrs(r, samples=M.samples, noise_cov=M.noise, given_track=gt if len(gt) else None,
                          given_point=gp if len(gt) else None, **{k: o[k] for k in o})
        return recs, sms, out, keep

    def plane_ransac(self, records, schedules=False):
        """Run a list of PlaneRansac in one call (a slot may be named by several); the slots do not change.  Per record
        a dict: status (PLANE_ACCEPTED, PLANE_FEW_POINTS or PLANE_REJECTED), n_points, inliers, iterations, best_it,
        normal [3], distance, reference [3], and per candidate used, inlier (bool) and point [3] (NaN: left out).
        schedules: also the sample schedule [1000, 3] and every iteration's inlier count [1000] (-1 without a RANSAC)."""
        n = len(records)
        recs, out = (_lib.CWindowPlaneRansac * max(n, 1))(), []
        for r, P in zip(recs, records):
            m = len(P.tracks)
            o = dict(info=np.zeros(5, dtype=np.int32), plane=np.zeros(7), used=np.zeros(m, dtype=np.uint8),
                     inlier=np.zeros(m, dtype=np.uint8), points=np.zeros((m, 3)), tracks=P.tracks)
            if schedules:
                o.update(schedule=np.zeros((1000, 3), dtype=np.int32), counts=np.zeros(1000, dtype=np.int32))
            out.append(o)
            r.slot, r.mode, r.n_tracks = P.slot, P.mode, m
            _lib.set_ptrs(r, tracks=P.tracks, info=o["info"], plane=o["plane"], used=o["used"], inlier=o["inlier"],
                          points=o["points"], schedule=o.get("schedule"), counts=o.get("counts"))
        self.ba._ck(self.lib.pvio_b200_batch_window_plane_ransac(self.h, n, recs))
        for o in out:
            i, p = o.pop("info"), o.pop("plane")
            o.pop("tracks")
            o.update(status=int(i[0]), n_points=int(i[1]), inliers=int(i[2]), iterations=int(i[3]), best_it=int(i[4]),
                     normal=p[:3].copy(), distance=float(p[3]), reference=p[4:].copy(),
                     used=o["used"].astype(bool), inlier=o["inlier"].astype(bool))
        return out

    def set_imu(self, records):
        """Keep the samples of a list of Imu on the device with their factors, in one call."""
        recs = (_lib.CWindowImu * max(len(records), 1))()
        for r, m in zip(recs, records):
            r.slot, r.frame, r.n_samples, r.t_end = m.slot, m.frame, len(m.samples), m.t_end
            _lib.set_ptrs(r, samples=m.samples, noise_cov=m.noise)
        self.ba._ck(self.lib.pvio_b200_batch_window_set_imu(self.h, len(records), recs))

    def imu_records(self, slots):
        """Per slot its N - 1 IMU records [N - 1, 288] as they stand on the device (after a solve: the records it used)."""
        s = np.ascontiguousarray(slots, dtype=np.int32)
        n = len(s)
        nf = np.zeros(max(n, 1), dtype=np.int32)
        self.ba._ck(self.lib.pvio_b200_batch_window_download(self.h, n, _lib.ptr(s), _lib.ptr(nf), None, 0, None, 0,
                                                             None, None, None, None, None, None))
        stride = _lib.IMU_STRIDE * max(self.ba.max_frames - 1, 1)
        out = np.zeros((max(n, 1), stride))
        self.ba._ck(self.lib.pvio_b200_batch_window_imu_records(self.h, n, _lib.ptr(s), _lib.ptr(out), stride))
        return [out[i, :_lib.IMU_STRIDE * max(int(nf[i]) - 1, 0)].reshape(-1, _lib.IMU_STRIDE).copy() for i in range(n)]

    def solve(self, slots, max_iterations=10, max_time=1e6, alias_bias=True, postpass=True):
        s = np.ascontiguousarray(slots, dtype=np.int32)
        opt = _lib.COptions(max_iterations, max_time, 1 if alias_bias else 0, 1 if postpass else 0, 0.0)
        sm = (_lib.CSummary * max(len(s), 1))()
        self.ba._ck(self.lib.pvio_b200_batch_window_solve(self.h, len(s), _lib.ptr(s), C.byref(opt), sm))
        return [_lib.summary(sm[i]) for i in range(len(s))]

    def drop_victim(self, slots, want=False, max_frames=None):
        """Map::marginalize_frame(0) on the slots; want: also return each slot's new prior (S, e)."""
        s = np.ascontiguousarray(slots, dtype=np.int32)
        if not want:
            self.ba._ck(self.lib.pvio_b200_batch_window_drop_victim(self.h, len(s), _lib.ptr(s), None, 0, None, 0))
            return None
        d = 15 * ((max_frames or self.ba.max_frames) - 1)
        S = np.zeros((max(len(s), 1), d * d)); e = np.zeros((max(len(s), 1), d))
        self.ba._ck(self.lib.pvio_b200_batch_window_drop_victim(self.h, len(s), _lib.ptr(s), _lib.ptr(S), d * d,
                                                                _lib.ptr(e), d))
        return S, e

    def covariance(self, slots, frames, tracks):
        """The covariance of each named slot's window at its current state, in the solve's local coordinates: per slot
        frames[i] (window indices) and tracks[i] (live track ids).  Per record a dict: cov [15 k, 15 k] (the named frames'
        joint block, [dtheta dp dv dbg dba] per frame; 0 where a frame has no such coordinate), inv_depth_var [len(tracks)]
        (NaN for a plane track or a track with one observation) and status (OK, or ENUMERIC with every output NaN)."""
        n = len(slots)
        recs, out = (_lib.CWindowCovariance * max(n, 1))(), []
        for r, s, f, t in zip(recs, slots, frames, tracks):
            f = np.ascontiguousarray(f, dtype=np.int32).reshape(-1)
            t = np.ascontiguousarray(t, dtype=np.int32).reshape(-1)
            o = dict(frames=f, tracks=t, cov=np.zeros((15 * len(f), 15 * len(f))), inv_depth_var=np.zeros(len(t)))
            out.append(o)
            r.slot, r.n_frames, r.n_tracks = int(s), len(f), len(t)
            _lib.set_ptrs(r, frames=f if len(f) else None, cov=o["cov"] if len(f) else None,
                          tracks=t if len(t) else None, inv_depth_var=o["inv_depth_var"] if len(t) else None)
        self.ba._ck(self.lib.pvio_b200_batch_window_covariance(self.h, n, recs))
        for r, o in zip(recs, out):
            del o["frames"], o["tracks"]
            o["status"] = int(r.status)
        return out

    def landmarks(self, slots, tracks=None, covariance=False, capacity=None):
        """The map of each named slot at its current state: per record the rows of tracks[i] (live track ids), or of every
        live track in id order when tracks (or tracks[i]) is None.  Per record a dict: ids [rows], point [rows, 3]
        (Track::get_landmark_point()), role [rows] (-1, -2 or the plane index) and status; with covariance also point_cov
        [rows, 3, 3] and inv_depth_var [rows], NaN for a plane track or a track with one observation, and NaN throughout
        when status is ENUMERIC.  capacity: rows reserved for an all-tracks record (None: the handle's max_landmarks)."""
        n = len(slots)
        cap = int(self.ba.max_landmarks if capacity is None else capacity)
        recs, out = (_lib.CWindowLandmarks * max(n, 1))(), []
        for i, (r, s) in enumerate(zip(recs, slots)):
            t = None if tracks is None else tracks[i]
            if t is not None:
                t = np.ascontiguousarray(t, dtype=np.int32).reshape(-1)
            rows = cap if t is None else len(t)
            o = dict(tracks=t, ids=np.zeros(rows, dtype=np.int32), point=np.zeros((rows, 3)),
                     role=np.zeros(rows, dtype=np.int32))
            if covariance:
                o["point_cov"], o["inv_depth_var"] = np.zeros((rows, 3, 3)), np.zeros(rows)
            out.append(o)
            r.slot, r.n_tracks, r.capacity = int(s), -1 if t is None else len(t), rows
            _lib.set_ptrs(r, tracks=t if t is not None and len(t) else None, track_id=o["ids"], point=o["point"],
                          role=o["role"], point_cov=o.get("point_cov"), inv_depth_var=o.get("inv_depth_var"))
        self.ba._ck(self.lib.pvio_b200_batch_window_landmarks(self.h, n, recs))
        for r, o in zip(recs, out):
            del o["tracks"]
            k = int(r.n_rows)
            for key in ("ids", "point", "role", "point_cov", "inv_depth_var"):
                if key in o:
                    o[key] = o[key][:k]
            o["status"] = int(r.status)
        return out

    def trajectory(self, slots, times, covariance=False, smoothed=False):
        """The state of each named inertial slot at the sorted times[i], forward from the window frame before each time
        through the part of that frame's IMU factor's kept samples up to it (pvio_b200_batch_window_trajectory).  Per
        record a dict: states [n, 16] (q xyzw, p, v, bg, ba), frame [n] (the window frame used, -1: a time no factor
        with samples covers, with a zero state) and status; with covariance also state_cov [n, 15, 15] in the
        coordinates of covariance(), NaN for an uncovered time and throughout when status is ENUMERIC.
        smoothed: each state conditioned on both solved frames around it instead, meeting the next frame rather than
        jumping there (pvio_b200_batch_window_smoothed_trajectory); the same dicts, and frame -2 (a zero state, a NaN
        covariance) for the times of a factor whose increment covariance is not positive definite, as a one-sample
        factor's is not."""
        n = len(slots)
        if len(times) != n:
            raise ValueError("one time list per slot")
        recs, out = (_lib.CWindowTrajectory * max(n, 1))(), []
        for r, s, t in zip(recs, slots, times):
            t = np.ascontiguousarray(t, dtype=np.float64).reshape(-1)
            k = len(t)
            o = dict(times=t, states=np.zeros((k, 16)), frame=np.zeros(k, dtype=np.int32))
            if covariance:
                o["state_cov"] = np.zeros((k, 15, 15))
            out.append(o)
            r.slot, r.n_times = int(s), k
            _lib.set_ptrs(r, times=t if k else None, states=o["states"] if k else None, frame=o["frame"] if k else None,
                          state_cov=o.get("state_cov") if k else None)
        call = self.lib.pvio_b200_batch_window_smoothed_trajectory if smoothed else self.lib.pvio_b200_batch_window_trajectory
        self.ba._ck(call(self.h, n, recs))
        for r, o in zip(recs, out):
            del o["times"]
            o["status"] = int(r.status)
        return out

    def save(self, slots, tracker_slots=None):
        """Save each sequence to host memory: per record a window slot (-1: none) and, from tracker_slots (None: none),
        a tracker slot of batch_feature_track (-1: none).  Returns one blob (bytes) per record, which restore() seats in
        any slot of any handle."""
        recs, n = self._snapshots(slots, tracker_slots)
        self.ba._ck(self.lib.pvio_b200_batch_window_save(self.h, n, recs))          # data NULL: the sizes
        bufs = [np.zeros(recs[i].size, dtype=np.uint8) for i in range(n)]
        for i, b in enumerate(bufs):
            recs[i].data, recs[i].capacity = _lib.ptr(b), len(b)
        self.ba._ck(self.lib.pvio_b200_batch_window_save(self.h, n, recs))
        return [b.tobytes() for b in bufs]

    def restore(self, slots, blobs, tracker_slots=None):
        """Restore blobs of save(): record i seats blobs[i]'s window in slots[i] and its tracker part in
        tracker_slots[i] (-1 or None: that part is skipped).  The link between them comes back only when both are
        restored; a restored tracker slot needs its lens set again (batch_set_lens) if it had one."""
        recs, n = self._snapshots(slots, tracker_slots)
        arrs = [np.frombuffer(b, dtype=np.uint8) for b in blobs]
        if len(arrs) != n:
            raise ValueError("one blob per record")
        for i, a in enumerate(arrs):
            recs[i].data, recs[i].capacity = _lib.ptr(a), len(a)
        self.ba._ck(self.lib.pvio_b200_batch_window_restore(self.h, n, recs))

    @staticmethod
    def _snapshots(slots, tracker_slots):
        """the pvio_b200_window_snapshot records of a save / restore call, and their count"""
        slots = [-1 if s is None else int(s) for s in slots]
        ts = [-1] * len(slots) if tracker_slots is None else [-1 if t is None else int(t) for t in tracker_slots]
        if len(ts) != len(slots):
            raise ValueError("one tracker slot per record")
        recs = (_lib.CWindowSnapshot * max(len(slots), 1))()
        for r, s, t in zip(recs, slots, ts):
            r.slot, r.tracker_slot = s, t
        return recs, len(slots)

    def download(self, slots, track_stride):
        """Per slot a dict: frames [N, 16], and per live track in id order: id, inv_depth, anchor, n_obs, valid, quality."""
        s = np.ascontiguousarray(slots, dtype=np.int32)
        n, fs = len(s), 16 * self.ba.max_frames
        nf = np.zeros(max(n, 1), dtype=np.int32); nt = np.zeros(max(n, 1), dtype=np.int32)
        fr = np.zeros((max(n, 1), fs))
        T = max(int(track_stride), 1)
        ids = np.zeros((max(n, 1), T), dtype=np.int32); rho = np.zeros((max(n, 1), T)); an = np.zeros_like(ids)
        cnt = np.zeros_like(ids); val = np.zeros((max(n, 1), T), dtype=np.uint8); q = np.zeros((max(n, 1), T))
        p = _lib.ptr
        self.ba._ck(self.lib.pvio_b200_batch_window_download(self.h, n, p(s), p(nf), p(fr), fs, p(nt), T, p(ids), p(rho),
                                                             p(an), p(cnt), p(val), p(q)))
        out = []
        for i in range(n):
            N, k = int(nf[i]), int(nt[i])
            out.append(dict(frames=fr[i, :16 * N].reshape(N, 16).copy(), ids=ids[i, :k].copy(), inv_depth=rho[i, :k].copy(),
                            anchor=an[i, :k].copy(), n_obs=cnt[i, :k].copy(), valid=val[i, :k].copy(), quality=q[i, :k].copy()))
        return out
