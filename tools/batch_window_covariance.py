"""Time pvio_b200_batch_window_covariance on n = 1 / 8 / 132 / 528 resident cfg3 slots (N = 9, M = 300, prior over 8
frames): the call's wall time, and each new kernel's device time from torch.profiler in a pass of its own; the card's
name and power limit are read in the same run.  Prints the result as JSON, and writes it to --json when given.

    python tools/batch_window_covariance.py [--reps 20] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
from pvio_b200.batch_window import BatchWindows                                 # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor                            # noqa: E402
from synthetic import synth                                                     # noqa: E402
from test_gpu_batch_window_covariance import _feed, _tracks                      # noqa: E402


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
    w, st = synth.make_cfg3(seed=649, N=9, M=300)[:2]
    assert w.n_prior == 8, w.n_prior
    _feed(bw, 0, w, st, _tracks(w, planes=False))
    bw.solve([0], max_iterations=4)
    blob = bw.save([0])[0]
    bw.restore(list(range(1, W)), [blob] * (W - 1))
    ids = [int(i) for i in bw.download([0], 400)[0]["ids"]]
    res = dict(card=card, window="cfg3 N=9 M=300, prior over 8 frames", rows=[])
    for n in sizes:
        call = lambda: bw.covariance(list(range(n)), [list(range(9))] * n, [ids] * n)   # noqa: E731
        call()
        t = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            call()
            t.append(time.perf_counter() - t0)
        res["rows"].append(dict(n=n, wall_ms_median=1e3 * float(np.median(t)), wall_ms_min=1e3 * float(np.min(t))))
    import torch
    from torch.profiler import ProfilerActivity, profile
    for row in res["rows"]:
        n = row["n"]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                bw.covariance(list(range(n)), [list(range(9))] * n, [ids] * n)
            torch.cuda.synchronize()
        for e in prof.key_averages():
            if "cov_kernel" in e.key or "cov_lm_kernel" in e.key:
                name = "cov_lm_kernel" if "cov_lm_kernel" in e.key else "cov_kernel"
                row[name + "_us"] = e.device_time_total / e.count if e.count else None
    print(json.dumps(res, indent=1))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)
    ba.close()


if __name__ == "__main__":
    main()
