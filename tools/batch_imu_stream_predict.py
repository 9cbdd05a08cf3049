"""Wall times of pvio_b200_batch_imu_stream_set_covariance and pvio_b200_batch_imu_stream_predict for n stream slots,
and the device time of their kernels.  Each slot holds a latest state with about 20 kept samples after it (200 Hz
readings, gyroscope and accelerometer on the same stamps, no camera stamp) and a DIRECT seed; predict asks for 1 or 10
times per record, spread over the kept samples, with poses, states and both covariances.  Wall times are medians over
--reps calls through the Python binding, each ending in the call's own synchronisation; a separate torch.profiler pass
gives the mean device time of the seed and predict kernels (CUDA events of the profiler's trace).  Prints one line per
n and times-per-record with the GPU's name and power limit, read in the same run.

    python tools/batch_imu_stream_predict.py [--n 1 132 528 4096] [--reps 20]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from batch_imu_stream import gpu_info  # noqa: E402

from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.imu_stream import ImuStream, StreamRecord  # noqa: E402

NOISE = np.stack([np.eye(3) * 1e-4, np.eye(3) * 3e-3, np.eye(3) * 1e-7, np.eye(3) * 2e-5]).reshape(4, 9)


def setup(st, slots, rng):
    """a state at t = 0, then 21 readings at 200 Hz: 20 samples kept after the state"""
    st.reset(slots)
    q = np.r_[[0.0, 0.0, 0.0, 1.0], rng.normal(size=12) * 0.1]
    st.push([StreamRecord(s).set_state(0.0, q) for s in slots])
    ev = []
    for k in range(21):
        t = 0.005 * k
        ev += [(0, t, *rng.normal(size=3) * 0.3), (1, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3) * 0.3))]
    outs = st.push([StreamRecord(s, ev) for s in slots])
    if any(o["n_consumed"] != len(ev) for o in outs):
        raise RuntimeError("the readings were not consumed whole")
    a = rng.normal(size=(15, 15)) * 1e-2
    return a @ a.T + np.eye(15) * 1e-4


def median_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts))


def kernel_ms(fn, reps):
    """mean device time per call of the stream kernels fn launches, from a torch.profiler trace"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("imu_stream_seed_kernel", "imu_stream_predict_kernel"):
            if k in e.key:
                out[k] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0)) / 1e3 / reps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 132, 528, 4096])
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    print(gpu_info())
    rng = np.random.default_rng(0)
    ba = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    st = ImuStream(ba)
    for n in args.n:
        slots = list(range(n))
        P = setup(st, slots, rng)

        def seed():
            st.set_covariance(slots, [0.0] * n, [P] * n, NOISE)
        seed()
        set_ms = median_ms(seed, args.reps)
        set_k = kernel_ms(seed, args.reps).get("imu_stream_seed_kernel", float("nan"))
        for k in (1, 10):
            times = [np.linspace(0.01, 0.1, k) if k > 1 else np.array([0.1])] * n

            def pred():
                st.predict(slots, times, states=True, covariances=True)
            pred()
            p_ms = median_ms(pred, args.reps)
            p_k = kernel_ms(pred, args.reps).get("imu_stream_predict_kernel", float("nan"))
            print(f"n={n:5d} times/record={k:2d}: set_covariance {set_ms:.3f} ms (kernel {set_k:.4f} ms), "
                  f"predict {p_ms:.3f} ms (kernel {p_k:.4f} ms)", flush=True)
    ba.close()


if __name__ == "__main__":
    main()
