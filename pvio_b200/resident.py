"""Host mirror of the resident sliding window (include/pvio_b200.h, csrc/batch_window.cu): the window persists in the handle
between keyframes; the caller reports appended frames, new tracks / observations and drops the oldest frame, which
marginalises it into a prior that stays on the device (map/map.cpp:76-88, core/sliding_window_tracker.cpp:79-125)."""
import ctypes as C

import numpy as np

from . import _lib


class ResidentWindow:
    def __init__(self, ba, win):
        """ba: a BundleAdjustor (owns the device handle); win: any Window carrying the constants (extrinsics, noise model,
        use_inertial) -- its arrays are not used."""
        self.ba, self.lib, self.h = ba, ba.lib, ba.h
        ba._ck(self.lib.pvio_b200_window_reset(self.h, C.byref(_lib.window_constants(win))))

    def append_frame(self, state16, fixed=False, imu_record=None):
        s = np.ascontiguousarray(state16, dtype=np.float64)
        rec = None if imu_record is None else np.ascontiguousarray(imu_record, dtype=np.float64)
        self.ba._ck(self.lib.pvio_b200_window_append_frame(self.h, _lib.ptr(s), 1 if fixed else 0, _lib.ptr(rec)))

    def add_tracks(self, frames, z, inv_depth):
        n = len(frames)
        f = np.ascontiguousarray(frames, dtype=np.int32); zz = np.ascontiguousarray(z, dtype=np.float64).reshape(-1, 2)
        r = np.ascontiguousarray(inv_depth, dtype=np.float64); ids = np.zeros(max(n, 1), dtype=np.int32)
        self.ba._ck(self.lib.pvio_b200_window_add_tracks(self.h, n, _lib.ptr(f), _lib.ptr(zz), _lib.ptr(r), _lib.ptr(ids)))
        return ids[:n]

    def add_observations(self, tracks, frames, z):
        n = len(tracks)
        t = np.ascontiguousarray(tracks, dtype=np.int32); f = np.ascontiguousarray(frames, dtype=np.int32)
        zz = np.ascontiguousarray(z, dtype=np.float64).reshape(-1, 2)
        self.ba._ck(self.lib.pvio_b200_window_add_observations(self.h, n, _lib.ptr(t), _lib.ptr(f), _lib.ptr(zz)))

    def remove_track(self, track):
        self.ba._ck(self.lib.pvio_b200_window_remove_track(self.h, int(track)))

    def set_prior(self, S, e, state0):
        S = np.ascontiguousarray(S, dtype=np.float64); e = np.ascontiguousarray(e, dtype=np.float64)
        x0 = np.ascontiguousarray(state0, dtype=np.float64).reshape(-1, 16)
        self.ba._ck(self.lib.pvio_b200_window_set_prior(self.h, len(x0), _lib.ptr(S), _lib.ptr(e), _lib.ptr(x0)))

    def solve(self, max_iterations=10, max_time=1e6, alias_bias=True):
        opt = _lib.COptions(max_iterations, max_time, 1 if alias_bias else 0, 0, 0.0)
        sm = _lib.CSummary()
        self.ba._ck(self.lib.pvio_b200_window_solve(self.h, C.byref(opt), C.byref(sm)))
        return _lib.summary(sm)

    def drop_victim(self):
        self.ba._ck(self.lib.pvio_b200_window_drop_victim(self.h))

    def get(self, tracks=()):
        """(frames [N,16], inverse depths, anchor frames, observation counts) of the queried tracks."""
        n = C.c_int32()
        self.ba._ck(self.lib.pvio_b200_window_get(self.h, C.byref(n), None, 0, None, None, None, None))
        fr = np.zeros((max(n.value, 1), 16))
        t = np.ascontiguousarray(tracks, dtype=np.int32)
        rho = np.zeros(max(len(t), 1)); an = np.zeros(max(len(t), 1), dtype=np.int32); cnt = np.zeros(max(len(t), 1), dtype=np.int32)
        self.ba._ck(self.lib.pvio_b200_window_get(self.h, C.byref(n), _lib.ptr(fr), len(t), _lib.ptr(t) if len(t) else None,
                                                  _lib.ptr(rho), _lib.ptr(an), _lib.ptr(cnt)))
        return fr[:n.value], rho[:len(t)], an[:len(t)], cnt[:len(t)]
