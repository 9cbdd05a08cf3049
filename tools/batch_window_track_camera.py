"""Times one camera frame of n cfg3-shaped sequences through pvio_b200_batch_window_track_camera against the two calls
it replaces, batch_feature_track with a host-given predict_q then batch_window_mirror_frame, on twin window and tracker
slots fed the same frames and samples (the twins take the call's predict_q, so both paths track alike).  Per n: the
median wall time of a frame through each path, and the device kernel time of each path summed over the timed frames
(torch.profiler, CUDA activities), per frame.  The host PreIntegrator::integrate + predict and the delta_key_q
composition that the call takes off the host are C++ in a shim and are not measured here.  Prints one line per n with
the GPU's name and power limit.

    python tools/batch_window_track_camera.py [--n 1 8 132 528] [--frames 12] [--warmup 6]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from pvio_b200.batch_window import BatchWindows, Camera, Edit, Mirror  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.feature_track import batch_feature_track, min_capacity  # noqa: E402
from test_gpu_batch_window_track_camera import render_run, KD, SHAPE  # noqa: E402
from synthetic.sequence import Run  # noqa: E402

H, W = SHAPE
CAP = min_capacity(W, H, KD)


def kernel_ms(fn):
    """device time of the kernels fn() launches, ms"""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.self_device_time_total for e in prof.key_averages() if e.self_device_time_total > 0)
    if us <= 0:
        raise RuntimeError("the profiler recorded no kernel")
    return us * 1e-3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--frames", type=int, default=12)
    ap.add_argument("--warmup", type=int, default=6)
    a = ap.parse_args()
    torch.cuda.init()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    seqs8 = []
    for k in range(8):
        run = Run(F=a.frames + 2, N=6, M=40, seed=700 + k)
        frames, samples, K = render_run(run, 700 + k, ())
        run.w.K_fx, run.w.K_fy = K[0], K[1]
        seqs8.append((run, frames, samples, K))
    for n in a.n:
        ba = BundleAdjustor(max_windows=2 * n, max_frames=a.frames + 2, max_landmarks=2048, max_obs=16384)
        try:
            bw = BatchWindows(ba)
            for i in range(n):                               # slot i / tracker i: the call; n + i: the two-call twin
                run, frames, samples, K = seqs8[i % 8]
                for slot in (i, n + i):
                    z = batch_feature_track(ba, [dict(slot=slot, frame_id=1, image=frames[0], K=K, map_frames=0,
                                                      max_keypoints=CAP)], keypoint_distance=KD)[0]["keypoints"]
                    g = run.guess
                    bw.reset(slot, run.w)
                    e = Edit(slot).frame(np.concatenate([g.q[0], g.p[0], g.v[0], g.bg[0], g.ba[0]]))
                    e.new = [(0, q, 1.0) for q in z]
                    ids = bw.edit([e])[0]
                    bw.set_keypoints(slot, slot, 1, {int(t): k for k, t in enumerate(ids)})
            times, kern = [[], []], [0.0, 0.0]
            for f in range(1, a.frames + 1):
                cams = []
                for i in range(n):
                    run, frames, samples, K = seqs8[i % 8]
                    s, t = samples[f]
                    cams.append(Camera(i, i, f + 1, frames[f], K, f, s, t, run.truth.imu_noise))
                out = []

                def call():
                    out[:] = bw.track_camera(cams, CAP, keypoint_distance=KD)

                def chain():
                    batch_feature_track(ba, [dict(slot=n + i, frame_id=f + 1, image=c.image, K=c.K, map_frames=f,
                                                  max_keypoints=CAP, predict_q=o["predict_q"])
                                             for i, (c, o) in enumerate(zip(cams, out))], keypoint_distance=KD)
                    bw.mirror_frame([Mirror(n + i, n + i, c.samples, c.t_end, c.noise.reshape(4, 3, 3), c.cx, c.cy)
                                     for i, c in enumerate(cams)], CAP)

                for p, fn in enumerate((call, chain)):
                    ba.lib.pvio_b200_sync(ba.h)
                    if f > a.warmup and f == a.frames:
                        kern[p] = kernel_ms(fn)
                        continue
                    t0 = time.perf_counter()
                    fn()
                    ba.lib.pvio_b200_sync(ba.h)
                    if f > a.warmup:
                        times[p].append(time.perf_counter() - t0)
            c, h = 1e3 * np.median(times[0]), 1e3 * np.median(times[1])
            print(f"n={n:4d}  track_camera {c:8.2f} ms/frame (kernels {kern[0]:7.2f} ms)  feature_track + "
                  f"mirror_frame {h:8.2f} ms/frame (kernels {kern[1]:7.2f} ms)  ({len(times[0])} frames each, median "
                  f"wall; kernels of one frame; host PreIntegrator not measured)  [{gpu}]")
        finally:
            ba.close()


if __name__ == "__main__":
    main()
