"""Host-side mirror of PreIntegrator::integrate (pvio/src/pvio/estimation/preintegrator.cpp:85-98) over
the C ABI: batches of independent IMU factors, one warp each on the device (csrc/imu.cu)."""
import numpy as np

from . import _lib


def preintegrate(ba, factors, noise_cov):
    """ba: a BundleAdjustor (device handle).  factors: list of (samples [K][7], t_end, bg[3], ba[3]).
    noise_cov: (cov_w, cov_a, cov_bg, cov_ba) 3x3 each.  Returns records [n][288] (PVIO_B200_IMU_* layout)."""
    n = len(factors)
    begin = np.zeros(n + 1, dtype=np.int32)
    for i, f in enumerate(factors):
        begin[i + 1] = begin[i] + len(f[0])
    samples = np.ascontiguousarray(np.concatenate([np.asarray(f[0], dtype=np.float64).reshape(-1, 7) for f in factors]))
    t_end = np.array([f[1] for f in factors], dtype=np.float64)
    bias = np.ascontiguousarray(np.array([np.concatenate([f[2], f[3]]) for f in factors], dtype=np.float64))
    noise = np.ascontiguousarray(np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in noise_cov]))
    rec = np.zeros((n, _lib.IMU_STRIDE))
    ba._ck(ba.lib.pvio_b200_preintegrate(ba.h, n, _lib.ptr(begin), _lib.ptr(samples), _lib.ptr(t_end), _lib.ptr(bias),
                                         _lib.ptr(noise), _lib.ptr(rec)))
    return rec
