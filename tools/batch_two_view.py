"""Time of pvio_b200_batch_two_view (init_sfm's two-view step, initializer.cpp:102-161) for n sequences of 150 matches
(20 % outliers, 0.5 px noise, PVIO's defaults: 1000 iterations, seed 648), with the device time of each kernel from a
torch.profiler pass of its own.  For orientation only, a DIFFERENT algorithm on one host thread: OpenCV's
findHomography(RANSAC) + findEssentialMat(RANSAC) per problem (cv2 4-point / 5-point with its own sampler and stopping
rule).  The GPU's name and power limit are read in the same run.

    python tools/batch_two_view.py [--sizes 1,8,132,528] [--reps 5] [--profile-n 132] [--out DIR]

Per size: the host wall time of the whole call (stage, 4 launches, replay, read-back), the median of --reps calls after
2 warm-up calls on the same inputs.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile-n", type=int, default=132)
    ap.add_argument("--cv-n", type=int, default=32)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from bench import gpu_identity
    from synthetic import synth
    from pvio_b200.bundle_adjustor import BundleAdjustor
    from pvio_b200.two_view import batch_two_view

    sizes = [int(s) for s in args.sizes.split(",")]
    base = []
    for i in range(16):
        s = synth.make_two_view(seed=500 + i, n=150, outlier_frac=0.2, kind="plane" if i % 4 == 3 else "general")
        base.append(dict(p1=s["p1"], p2=s["p2"], fx=s["fx"], fy=s["fy"]))
    ba = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "matches": 150, "rows": []}
    for n in sizes:
        probs = [base[i % len(base)] for i in range(n)]
        for _ in range(2):
            batch_two_view(ba, probs)
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            batch_two_view(ba, probs)
            ts.append(time.perf_counter() - t0)
        row = {"n": n, "wall_ms": 1e3 * float(np.median(ts)), "wall_ms_per_problem": 1e3 * float(np.median(ts)) / n}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)

    try:
        import cv2
        t0 = time.perf_counter()
        for d in base[:1] * args.cv_n:
            p1 = np.ascontiguousarray(d["p1"])
            p2 = np.ascontiguousarray(d["p2"])
            thr = 0.7 / d["fx"]
            cv2.findHomography(p1, p2, cv2.RANSAC, 2 * thr, maxIters=1000, confidence=0.999)
            cv2.findEssentialMat(p1, p2, np.eye(3), cv2.RANSAC, 0.999, thr)
        res["opencv_host_ms_per_problem"] = 1e3 * (time.perf_counter() - t0) / args.cv_n
        res["opencv_note"] = "cv2.findHomography + cv2.findEssentialMat, one host thread: a different algorithm"
        print(json.dumps({"opencv_host_ms_per_problem": res["opencv_host_ms_per_problem"]}), flush=True)
    except ImportError:
        res["opencv_host_ms_per_problem"] = None

    from torch.profiler import profile, ProfilerActivity
    probs = [base[i % len(base)] for i in range(args.profile_n)]
    batch_two_view(ba, probs)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        batch_two_view(ba, probs)
        torch.cuda.synchronize()
    kern = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "tv_" in e.name:
            name = e.name.split("tv_")[1].split("(")[0].split("<")[0]
            kern["tv_" + name] = kern.get("tv_" + name, 0.0) + e.device_time_total / 1e3
    res["profile_n"] = args.profile_n
    res["kernel_ms"] = kern
    print(json.dumps({"profile_n": args.profile_n, "kernel_ms": kern}), flush=True)
    ba.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_two_view.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
