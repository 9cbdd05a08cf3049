"""Time pvio_b200_batch_window_trajectory and pvio_b200_batch_window_smoothed_trajectory on n = 1 / 8 / 132 / 528
resident cfg3 slots (N = 9, M = 300, prior over 8 frames, every IMU factor with its 50 samples kept, solved), one query
per kept sample (400 per slot): the wall time of each call without and with covariances, and its kernel's and
cov_kernel's device time from torch.profiler in a pass of its own; the card's name and power limit are read in the same
run.  Prints the result as JSON, and writes it
to --json when given.

    python tools/batch_window_trajectory.py [--reps 20] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from pvio_b200.batch_window import BatchWindows, Imu                            # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor                            # noqa: E402
from synthetic import synth                                                     # noqa: E402
from test_gpu_batch_window_covariance import _feed, _tracks                      # noqa: E402

KERNELS = ("bw_trajectory_kernel", "bw_smoothed_trajectory_kernel", "cov_kernel")


def _wall(call, reps):
    call()
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        call()
        t.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(t)), 1e3 * float(np.min(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None, help="also write the result to this file")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    sizes = (1, 8, 132, 528)
    W = max(sizes)
    ba = BundleAdjustor(max_windows=W, max_frames=9, max_landmarks=400, max_obs=3000)
    bw = BatchWindows(ba)
    w, st, truth = synth.make_cfg3(seed=649, N=9, M=300)
    assert w.n_prior == 8, w.n_prior
    _feed(bw, 0, w, st, _tracks(w, planes=False))
    F = truth.imu_factors
    bw.set_imu([Imu(0, k + 1, F[k][0], F[k][1], truth.imu_noise) for k in range(w.N - 1)])
    bw.solve([0], max_iterations=4)
    blob = bw.save([0])[0]
    bw.restore(list(range(1, W)), [blob] * (W - 1))
    ts = np.sort(np.concatenate([F[k][0][:, 0] for k in range(w.N - 1)]))
    res = dict(card=card, window=f"cfg3 N=9 M=300, prior over 8 frames, {len(ts)} queries per slot (one per kept sample)",
               rows=[])
    for smoothed in (False, True):
        for n in sizes:
            sl = list(range(n))
            p = _wall(lambda: bw.trajectory(sl, [ts] * n, smoothed=smoothed), args.reps)
            c = _wall(lambda: bw.trajectory(sl, [ts] * n, covariance=True, smoothed=smoothed), args.reps)
            res["rows"].append(dict(call="smoothed" if smoothed else "forward", n=n, states_ms_median=p[0],
                                    states_ms_min=p[1], cov_ms_median=c[0], cov_ms_min=c[1]))
    import torch
    from torch.profiler import ProfilerActivity, profile
    for row in res["rows"]:
        sl = list(range(row["n"]))
        smoothed = row["call"] == "smoothed"
        own = "bw_smoothed_trajectory_kernel" if smoothed else "bw_trajectory_kernel"
        for cov in (False, True):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    bw.trajectory(sl, [ts] * len(sl), covariance=cov, smoothed=smoothed)
                torch.cuda.synchronize()
            for e in prof.key_averages():
                k = next((k for k in KERNELS if k in e.key), None)
                if k and e.count and (k == own or (cov and k == "cov_kernel")):
                    row[k + ("_us" if cov else "_states_only_us")] = e.device_time_total / e.count
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    ba.close()


if __name__ == "__main__":
    main()
