"""Wall time of pvio_b200_batch_imu_stream for n sequences, one camera period per call: 10 gyroscope and 10
accelerometer readings (200 Hz, equal stamps) and one camera stamp that arrives ahead of them, so each call's last
reading releases one frame per sequence and the next call feeds back a latest state, as a lockstep caller does at
20 Hz.  Each call is timed with the host clock from the call to
its return, which ends in the call's own synchronisation; the C entry point is called directly with its records built
once, so the time is the call's: host checks, staging, one upload, one kernel, one download.  Medians over --reps
calls after --warmup calls (which also grow the queues).  Prints one line per n with the GPU's name and power limit, read in the same run.

    python tools/batch_imu_stream.py [--n 1 8 132 528 4096] [--reps 200] [--warmup 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pvio_b200 import _lib  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.imu_stream import ImuStream  # noqa: E402

PERIOD, RATE = 0.05, 200.0


def period_events(k, rng):
    """camera period k: the stamp of the frame the period closes, then 10 gyroscope + 10 accelerometer readings; the
    last reading is the first after the stamp"""
    ev = [(_lib.IMU_EVENT_CAMERA, k * PERIOD + PERIOD - 0.5 / RATE, 0.0, 0.0, 0.0)]
    for j in range(10):
        t = k * PERIOD + (j + 1) / RATE
        ev.append((_lib.IMU_EVENT_GYROSCOPE, t, *rng.normal(size=3) * 0.3))
        ev.append((_lib.IMU_EVENT_ACCELEROMETER, t, *(np.array([0, 0, 9.8]) + rng.normal(size=3) * 0.2)))
    return np.ascontiguousarray(ev, dtype=np.float64)


class Call:
    """the records of one call over n slots, reused from call to call (events and state rewritten in place)"""

    def __init__(self, n):
        self.n = n
        self.recs = (_lib.CImuStreamRecord * n)()
        self.ev = np.zeros((n, 21, 5))
        self.state = np.zeros((n, 16))
        self.state[:, 3] = 1.0
        self.poses = np.zeros((n, 21, 7))
        self.ft = np.zeros((n, 4))
        self.fr = np.zeros((n, 4), dtype=np.int32)
        self.rows = np.zeros((n, 64, 7))
        for i, r in enumerate(self.recs):
            r.slot, r.n_events, r.max_frames, r.max_rows = i, 21, 4, 64
            _lib.set_ptrs(r, events=self.ev[i], state=self.state[i], poses=self.poses[i], frame_t=self.ft[i],
                          frame_rows=self.fr[i], rows=self.rows[i])

    def fill(self, events, t_state):
        self.ev[:] = events
        for r in self.recs:
            r.state_op = _lib.IMU_STREAM_SET if t_state is not None else _lib.IMU_STREAM_KEEP
            r.state_time = t_state or 0.0


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError):
        return "unknown GPU"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528, 4096])
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    info = gpu_info()
    rng = np.random.default_rng(0)
    ba = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
    st = ImuStream(ba)
    for n in args.n:
        st.reset(list(range(n)))
        call = Call(n)
        times, k, t_frame = [], 0, None
        launches = 0
        for it in range(args.warmup + args.reps):
            call.fill(period_events(k, rng), t_frame)
            l0 = ba.kernel_launches
            t0 = time.perf_counter()
            rc = ba.lib.pvio_b200_batch_imu_stream(ba.h, n, call.recs)
            dt = time.perf_counter() - t0
            ba._ck(rc)
            if any(r.n_consumed != 21 for r in call.recs):
                raise RuntimeError("a period was not consumed whole")
            t_frame = call.ft[0, 0] if call.recs[0].n_frames else None
            k += 1
            if it >= args.warmup:
                times.append(dt)
                launches = ba.kernel_launches - l0
        us = np.median(times) * 1e6
        print(f"n={n:5d}  call {us:8.1f} us  ({us / n:7.3f} us/sequence, {n * 21 / np.median(times) / 1e6:7.2f} M events/s)"
              f"  launches/call {launches}  [{info}]", flush=True)
    ba.close()


if __name__ == "__main__":
    main()
