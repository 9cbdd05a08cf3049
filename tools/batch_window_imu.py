"""IMU re-integration of the resident slots (pvio_b200_batch_window_set_imu) on n cfg3 sequences (N = 9, 200 Hz IMU,
0.25 s keyframes: 50 samples per factor; the factors of every other sequence hold merged lists of 100, as a frame that
replaces an erased non-keyframe does), n = 1, 8, 132, 528:

  - reintegrate_us: device time of the one re-integration launch of a solve (bw_reintegrate_kernel, torch.profiler)
  - solve_ms: the trust-region chain of the same solve (summary.solve_seconds) for scale
  - cycle_ms (with / without samples): wall time of one keyframe cycle of all n slots -- solve, drop, a non-keyframe
    edit that the keyframe replaces, each edit followed by its set_imu when the slots hold samples -- median over --reps
  - h2d_bytes_per_keyframe: the bytes the set_imu calls of one keyframe upload (records, samples, t_end and noise)

Prints the card (name, power limit) and one JSON line per n.
Usage: python tools/batch_window_imu.py [--n 1 8 132 528] [--reps 6]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from synthetic.sequence import BatchPlayer, Run  # noqa: E402

N, M, KINDS, CAP = 9, 300, 4, 360


class MergedPlayer(BatchPlayer):
    """the factors of the odd sequences hold the samples of two factors back to back (about 100)"""

    def imu(self, j, f_win, f_abs, first=None):
        if first is None and j % 2 == 1 and f_abs >= 2:
            first = f_abs - 2
        return super().imu(j, f_win, f_abs, first)


def cycles(runs, samples, reps):
    n = len(runs)
    ba = BundleAdjustor(max_windows=n, max_frames=N, max_landmarks=CAP, max_obs=6000)
    p = MergedPlayer(ba, runs, imu_samples=samples)
    sent = [0]
    if samples:
        set_imu = p.bw.set_imu

        def counted(recs):
            sent[0] += 16 * len(recs) + sum(8 * 7 * len(r.samples) + 8 * 37 for r in recs)
            set_imu(recs)
        p.bw.set_imu = counted
    js, slots = list(range(n)), list(range(n))
    ts, chain, sent_kf = [], [], []
    for rep in range(reps + 1):
        sent[0] = 0
        t = time.perf_counter()
        sm = p.bw.solve(slots, max_iterations=10)
        p.advance(js, nonkey=True)
        if rep > 0:                                        # the first keyframe grows the staging and the sample store
            ts.append(time.perf_counter() - t)
            chain.append(sm[0]["solve_seconds"])
            sent_kf.append(sent[0])
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        p.bw.solve(slots, max_iterations=10)
    us = [e.device_time for e in prof.events() if "bw_reintegrate_kernel" in e.name]
    ba.close()
    return (1e3 * float(np.median(ts)), float(np.median(us)) if us else 0.0, 1e3 * float(np.median(chain)),
            int(np.median(sent_kf)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--reps", type=int, default=6)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    kinds = [Run(F=N + 2 * a.reps + 6, N=N, M=M, seed=811 + i) for i in range(KINDS)]
    for n in a.n:
        runs = [kinds[i % KINDS] for i in range(n)]
        with_ms, kern_us, chain_ms, h2d = cycles(runs, True, a.reps)
        without_ms, _, chain0_ms, _ = cycles(runs, False, a.reps)
        print(json.dumps(dict(n=n, card=card, reintegrate_us=round(kern_us, 1), solve_ms=round(chain_ms, 3),
                              solve_ms_without=round(chain0_ms, 3), cycle_ms_with=round(with_ms, 3),
                              cycle_ms_without=round(without_ms, 3), h2d_bytes_per_keyframe=h2d)))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
