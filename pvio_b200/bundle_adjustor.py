"""Host-side mirror of PVIO's BundleAdjustor (estimation/bundle_adjustor.h:29-42) over the
C-ABI: same entry points (solve, marginalize_frame, compute_reprojection_error), operating
on the flat Window/State containers the shim gathers from Map.  All arithmetic happens in
libpvio_b200.so on the GPU; this module only marshals arrays (no CPU fallback)."""
import ctypes as C

import numpy as np

from . import _lib
from .window import State


class PvioB200Error(RuntimeError):
    pass


class BundleAdjustor:
    """One handle = one GPU stream + device buffers, like BundleAdjustorSolver (bundle_adjustor.cpp:52-61)."""

    def __init__(self, device=0, max_windows=1, max_frames=16, max_landmarks=1024, max_obs=8192):
        self.lib = _lib.load()
        self.h = C.c_void_p()
        rc = self.lib.pvio_b200_create(device, max_windows, max_frames, max_landmarks, max_obs, C.byref(self.h))
        if rc != 0:
            msg = self.lib.pvio_b200_last_error(self.h).decode() if self.h else ""
            raise PvioB200Error(f"pvio_b200_create failed ({rc}) {msg}: a CUDA device is required, there is no CPU fallback")
        self.max_windows = max_windows
        self.max_frames = max_frames
        self.max_landmarks = max_landmarks
        self._keep = {}
        self._slot_frames = {}          # frame count of the window packed into each slot by batch_set / batch_replicate

    def close(self):
        if self.h:
            self.lib.pvio_b200_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc != 0:
            raise PvioB200Error(f"pvio_b200 error {rc}: {self.lib.pvio_b200_last_error(self.h).decode()}")

    @property
    def kernel_launches(self):
        return int(self.lib.pvio_b200_kernel_launches(self.h))

    # ---- reference-facing calls ------------------------------------------------------
    def solve(self, win, st, max_iterations=10, max_time=1e6, alias_bias=True, postpass=True, initial_radius=0.0):
        """BundleAdjustor::solve (bundle_adjustor.cpp:308-319).  Returns (State, summary dict)."""
        pa = _lib.PackedArgs(win, st)
        opt = _lib.COptions(max_iterations, max_time, 1 if alias_bias else 0, 1 if postpass else 0, initial_radius)
        sm = _lib.CSummary()
        valid = np.zeros(max(win.M, 1), dtype=np.uint8)
        quality = np.zeros(max(win.M, 1))
        self._ck(self.lib.pvio_b200_ba_solve(self.h, C.byref(pa.cw), C.byref(pa.cs), C.byref(opt), C.byref(sm),
                                             _lib.ptr(valid), _lib.ptr(quality)))
        fr = pa.keep["frames"]
        out = State(fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy(), fr[:, 10:13].copy(),
                    fr[:, 13:16].copy(), pa.keep["rho"].copy())
        summ = _lib.summary(sm)
        summ["valid"] = valid[:win.M].astype(bool)
        summ["quality"] = quality[:win.M]
        return out, summ

    def gn_step(self, win, st, mu=1e-8, want_system=False):
        """One regularised Gauss-Newton iteration (the parity / benchmark unit)."""
        pa = _lib.PackedArgs(win, st)
        n = 15 * win.N + win.M
        dx = np.zeros(n)
        cost, new_cost = C.c_double(), C.c_double()
        D = 15 * win.N
        H = np.zeros((D, D)) if want_system else None
        g = np.zeros(D) if want_system else None
        self._ck(self.lib.pvio_b200_ba_gn_step(
            self.h, C.byref(pa.cw), C.byref(pa.cs), mu, _lib.ptr(dx), C.byref(cost), C.byref(new_cost), _lib.ptr(H),
            _lib.ptr(g)))
        out = dict(dx=dx, cost=cost.value, new_cost=new_cost.value)
        if want_system:
            out.update(Hred=H, gred=g)
        return out

    def marginalize_frame(self, win, st, index=0, want_info=False):
        """BundleAdjustor::marginalize_frame (bundle_adjustor.cpp:348-599): returns (S, e[, H, b])."""
        pa = _lib.PackedArgs(win, st)
        d = 15 * (win.N - 1)
        S, e = np.zeros((d, d)), np.zeros(d)
        H = np.zeros((d, d)) if want_info else None
        b = np.zeros(d) if want_info else None
        self._ck(self.lib.pvio_b200_ba_marginalize(
            self.h, C.byref(pa.cw), C.byref(pa.cs), index, _lib.ptr(S), _lib.ptr(e), _lib.ptr(H), _lib.ptr(b)))
        return (S, e, H, b) if want_info else (S, e)

    def compute_reprojection_error(self, win, st):
        """BundleAdjustor::compute_reprojection_error (bundle_adjustor.cpp:321-336)."""
        pa = _lib.PackedArgs(win, st)
        err = C.c_double()
        self._ck(self.lib.pvio_b200_reprojection_error(self.h, C.byref(pa.cw), C.byref(pa.cs), C.byref(err)))
        return err.value

    # ---- batched windows -------------------------------------------------------------
    def batch_set(self, slot, win, st, resident_prior=False):
        """Pack `win` into slot `slot`.  resident_prior: the window's prior is the one batch_marginalize left in this slot
        on the device (n_prior and prior_frames are passed, the prior's S, e and linearisation point are not)."""
        pa = _lib.PackedArgs(win, st)
        if resident_prior:
            pa.cw.prior_S = pa.cw.prior_e = pa.cw.prior_state0 = None
        self._ck(self.lib.pvio_b200_batch_set_window(self.h, slot, C.byref(pa.cw), C.byref(pa.cs)))
        self._slot_frames[slot] = win.N

    def batch_replicate(self, n):
        self._ck(self.lib.pvio_b200_batch_replicate(self.h, n))
        for i in range(1, n):
            self._slot_frames[i] = self._slot_frames.get(0)

    def batch_marginalize(self, n, want=False):
        """BundleAdjustor::marginalize_frame(0) of each of the first n uploaded windows at its device state; the new priors
        stay in the slots' device arrays (see batch_set(resident_prior=True)).  want: also return [(S_i, e_i)], shaped by
        the frame count of the window batch_set packed into slot i."""
        if not want:
            self._ck(self.lib.pvio_b200_batch_marginalize(self.h, n, None, 0, None, 0))
            return None
        dmax = 15 * (self.max_frames - 1)
        S, e = np.zeros((n, dmax * dmax)), np.zeros((n, dmax))
        self._ck(self.lib.pvio_b200_batch_marginalize(self.h, n, _lib.ptr(S), dmax * dmax, _lib.ptr(e), dmax))
        out = []
        for i in range(n):
            d = 15 * (self._slot_frames[i] - 1)
            out.append((S[i, :d * d].reshape(d, d).copy(), e[i, :d].copy()))
        return out

    def batch_upload(self, n):
        self._ck(self.lib.pvio_b200_batch_upload(self.h, n))

    def batch_gn_step(self, n, mu=1e-8, apply=False):
        self._ck(self.lib.pvio_b200_batch_gn_step(self.h, n, mu, 1 if apply else 0))

    def batch_download(self, n, stride):
        dx = np.zeros((n, stride))
        costs = np.zeros((n, 2))
        self._ck(self.lib.pvio_b200_batch_download(self.h, n, _lib.ptr(dx), stride, _lib.ptr(costs)))
        return dx, costs

    def batch_gn_step_host(self, n, stride, mu=1e-8, dx=None, costs=None):
        dx = np.zeros((n, stride)) if dx is None else dx
        costs = np.zeros((n, 2)) if costs is None else costs
        _lib.check_rows(dx, n, stride, "dx")
        _lib.check_rows(costs, n, 2, "costs")
        self._ck(self.lib.pvio_b200_batch_gn_step_host(self.h, n, mu, _lib.ptr(dx), stride, _lib.ptr(costs)))
        return dx, costs

    def batch_solve(self, n, max_iterations=10, max_time=0.0, alias_bias=True, initial_radius=0.0):
        """Full trust-region solve of the first n uploaded windows, device-side loop with per-window termination."""
        opt = _lib.COptions(max_iterations, max_time, 1 if alias_bias else 0, 0, initial_radius)
        self._ck(self.lib.pvio_b200_batch_solve(self.h, n, C.byref(opt)))

    def batch_download_state(self, n, N, M):
        """Solved states of the first n windows: (frames [n, N, 16], inv_depth [n, M], list of summary dicts)."""
        frames = np.zeros((n, N * 16))
        rho = np.zeros((n, max(M, 1)))
        sm = (_lib.CSummary * n)()
        self._ck(self.lib.pvio_b200_batch_download_state(self.h, n, _lib.ptr(frames), N * 16, _lib.ptr(rho), max(M, 1),
                                                         sm))
        return frames.reshape(n, N, 16), rho[:, :M], [_lib.summary(x) for x in sm]

    def batch_solve_host(self, n, N, M, max_iterations=10, alias_bias=True, frames=None, rho=None):
        """upload + solve + download through host buffers (the end-to-end call bench.py times)."""
        frames = np.zeros((n, N * 16)) if frames is None else frames
        rho = np.zeros((n, max(M, 1))) if rho is None else rho
        _lib.check_rows(frames, n, N * 16, "frames")
        _lib.check_rows(rho, n, max(M, 1), "rho")
        opt = _lib.COptions(max_iterations, 0.0, 1 if alias_bias else 0, 0, 0.0)
        sm = (_lib.CSummary * n)()
        self._ck(self.lib.pvio_b200_batch_solve_host(self.h, n, C.byref(opt), _lib.ptr(frames), N * 16, _lib.ptr(rho),
                                                     max(M, 1), sm))
        return frames, rho, sm

    def selftest_lie(self, w):
        """Device expmap / logmap / right_jacobian / Plus on rotation vectors w [n, 3] -> [n, 32] (see the header)."""
        w = np.ascontiguousarray(w, dtype=np.float64)
        out = np.zeros((len(w), 32))
        self._ck(self.lib.pvio_b200_selftest_lie(self.h, len(w), _lib.ptr(w), _lib.ptr(out)))
        return out

    def selftest_eig(self, problems):
        """The marginaliser's eigen-solver on [(A, b)] in one launch (see the header) -> [(S, e)]."""
        dk = np.array([len(b) for _, b in problems], dtype=np.int32)
        A = np.concatenate([np.ascontiguousarray(a, dtype=np.float64).ravel() for a, _ in problems])
        b = np.concatenate([np.asarray(v, dtype=np.float64) for _, v in problems])
        S, e = np.zeros_like(A), np.zeros_like(b)
        self._ck(self.lib.pvio_b200_selftest_eig(self.h, len(dk), _lib.ptr(dk), _lib.ptr(A), _lib.ptr(b), _lib.ptr(S),
                                                 _lib.ptr(e)))
        out, oa, ob = [], 0, 0
        for d in dk:
            out.append((S[oa:oa + d * d].reshape(d, d), e[ob:ob + d]))
            oa += d * d
            ob += d
        return out

    CHOL_MODES = {"narrow": 0, "wide": 1, "wide-tiled": 2}

    def selftest_chol(self, systems, mode):
        """The reduced-system Cholesky solve on [(A, b)] in one launch (see the header); mode: one of CHOL_MODES.
        -> ([x], ok [n] bool)"""
        D = np.array([len(b) for _, b in systems], dtype=np.int32)
        A = np.concatenate([np.ascontiguousarray(a, dtype=np.float64).ravel() for a, _ in systems])
        b = np.concatenate([np.asarray(v, dtype=np.float64) for _, v in systems])
        x, ok = np.zeros_like(b), np.zeros(len(D), dtype=np.int32)
        self._ck(self.lib.pvio_b200_selftest_chol(self.h, len(D), self.CHOL_MODES[mode], _lib.ptr(D), _lib.ptr(A),
                                                  _lib.ptr(b), _lib.ptr(x), _lib.ptr(ok)))
        return np.split(x, np.cumsum(D)[:-1]), ok.astype(bool)

    def sync(self):
        self._ck(self.lib.pvio_b200_sync(self.h))

    def timer_start(self):
        self._ck(self.lib.pvio_b200_timer_start(self.h))

    def timer_stop(self):
        ms = C.c_float()
        self._ck(self.lib.pvio_b200_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def last_kernel_ms(self, which=0):
        ms = C.c_float()
        self._ck(self.lib.pvio_b200_last_kernel_ms(self.h, which, C.byref(ms)))
        return ms.value
