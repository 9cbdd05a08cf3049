"""Bytes per sequence and wall times of pvio_b200_batch_imu_stream_save / pvio_b200_batch_imu_stream_restore for n stream
slots in two states:
  - steady: a lockstep caller at 200 Hz IMU and 20 Hz camera (tools/batch_imu_stream.py's periods), checkpointed after
    a frame's release with that frame's state seated by a zero-event SET (INTEGRATION 2c);
  - backlog: 500 gyroscope and 500 accelerometer readings with no camera stamp and no state, so about 1000 rows queued
    (500 unreleased samples, 500 kept samples).
The restore seats the blobs back in their own slots (a rollback).  Wall times are medians over --reps calls through the
Python binding, each ending in the call's own synchronisation (save includes its size query); a separate
torch.profiler pass gives the device time of the pack and unpack kernels.  Prints one line per state and n with the
GPU's name and power limit, read in the same run.

    python tools/batch_imu_stream_save.py [--n 1 8 132 528 4096] [--reps 5]"""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from batch_imu_stream import gpu_info, period_events  # noqa: E402

from pvio_b200 import _lib  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.imu_stream import ImuStream, StreamRecord  # noqa: E402


def steady(st, slots, rng):
    """four camera periods in lockstep, then the last frame's state seated with a zero-event SET"""
    state = None
    for k in range(4):
        ev = period_events(k, rng)
        recs = [StreamRecord(s, ev) for s in slots]
        if state is not None:
            for r in recs:
                r.set_state(*state)
        outs = st.push(recs)
        if any(o["n_consumed"] != len(ev) or len(o["frames"]) != 1 for o in outs):
            raise RuntimeError("a period was not consumed whole")
        q = np.r_[[0.0, 0.0, 0.0, 1.0], rng.normal(size=12) * 0.1]
        state = (outs[0]["frames"][0][0], q)
    st.push([StreamRecord(s).set_state(*state) for s in slots])


def backlog(st, slots, rng):
    t = np.arange(500) / 200.0
    ev = np.zeros((1000, 5))
    ev[0::2, 0], ev[1::2, 0] = _lib.IMU_EVENT_GYROSCOPE, _lib.IMU_EVENT_ACCELEROMETER
    ev[0::2, 1] = ev[1::2, 1] = t
    ev[:, 2:] = rng.normal(size=(1000, 3))
    for c in range(0, len(slots), 528):
        outs = st.push([StreamRecord(s, ev) for s in slots[c:c + 528]])
        if any(o["n_consumed"] != len(ev) for o in outs):
            raise RuntimeError("the backlog was not consumed whole")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528, 4096])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    info = gpu_info()
    for name, fill in (("steady", steady), ("backlog", backlog)):
        for n in a.n:
            ba = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=64, max_obs=256)
            try:
                st = ImuStream(ba)
                slots = list(range(n))
                st.reset(slots)
                fill(st, slots, np.random.default_rng(1))
                blobs = st.save(slots)
                st.restore(slots, blobs)                     # warm: staging grown, modules loaded
                ts, tr = [], []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    blobs = st.save(slots)
                    t1 = time.perf_counter()
                    st.restore(slots, blobs)
                    t2 = time.perf_counter()
                    ts.append(t1 - t0)
                    tr.append(t2 - t1)
                if st.save(slots) != blobs:
                    raise RuntimeError("save -> restore -> save changed the blobs")
                kern = {}
                try:
                    import torch
                    from torch.profiler import ProfilerActivity, profile
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        st.restore(slots, st.save(slots))
                        torch.cuda.synchronize()
                    for ev in prof.key_averages():
                        for k in ("imu_stream_pack_kernel", "imu_stream_unpack_kernel"):
                            if k in ev.key:
                                kern[k.split("_")[2]] = ev.device_time_total / max(ev.count, 1) / 1e3
                except Exception as e:                        # the profiler pass is optional; the wall times are not
                    print(f"  (no profiler pass: {e})")
                per = np.mean([len(b) for b in blobs])
                ks = " ".join(f"{k} kernel {v:.3f} ms" for k, v in sorted(kern.items())) or "kernels not profiled"
                print(f"{name:7s} n={n:5d}  {per:8.0f} B per sequence  save {1e3 * np.median(ts):8.3f} ms  "
                      f"restore {1e3 * np.median(tr):8.3f} ms  (wall, median of {a.reps})  {ks}  [{info}]", flush=True)
            finally:
                ba.close()


if __name__ == "__main__":
    main()
