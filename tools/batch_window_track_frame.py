"""Times one camera frame of n cfg3 sequences in resident slots (n = 1, 8, 132, 528) on two paths:
  (a) pvio_b200_batch_window_track_frame: integrate, predict, PnP, triangulation and keyframe check in one call;
  (b) the host path it replaces: download, pvio_b200_preintegrate (with the merged lists for the non-keyframe half),
      tracker_oracle.predict on the host, localize, and tracker_oracle.keyframe_check on the host.
Wall time of the calls (host clock around calls that end in a synchronise), then in a separate pass the device time of
each new kernel from torch.profiler.  Prints the card's name and power limit from the same run.
Usage: python tools/batch_window_track_frame.py [--sizes 1,8,132,528] [--reps 20]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from oracle import tracker_oracle  # noqa: E402
from pvio_b200.batch_window import Localize  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from synthetic.sequence import BatchPlayer, Run  # noqa: E402
from test_gpu_batch_window_track_frame import _host_records, _oracle_check, _track  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528")
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip())
    run = Run(F=20, N=9, M=260, seed=790)
    for n in [int(x) for x in a.sizes.split(",")]:
        ba = BundleAdjustor(max_windows=n, max_frames=9, max_landmarks=400, max_obs=3000)
        p = BatchPlayer(ba, [run] * n)
        js = list(range(n))
        f, newest = run.N, run.N - 1
        recs = [_track(p, j, f, newest, kf=(j % 2 == 0))[0] for j in js]
        p.bw.track_frame(recs)
        t0 = time.perf_counter()
        for _ in range(a.reps):
            p.bw.track_frame(recs)
        dev = (time.perf_counter() - t0) / a.reps
        t0 = time.perf_counter()
        for _ in range(a.reps):
            ds = p.bw.download(p.slots, 400)
            locs = []
            for T, d in zip(recs, ds):
                rec1, _ = _host_records(ba, T, d["frames"][-1])
                L = Localize(T.slot, tracker_oracle.predict(d["frames"][-1], rec1), rec1)
                L.obs, L.new = T.obs, T.new
                locs.append(L)
                _oracle_check(run, p.model.m[T.slot], T, rec1, newest if T.newest_is_keyframe else newest - 1, newest, 0)
            p.bw.localize(locs)
        host = (time.perf_counter() - t0) / a.reps
        line = f"n={n}: track_frame {dev * 1e3:.3f} ms, host path {host * 1e3:.3f} ms"
        try:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(5):
                    p.bw.track_frame(recs)
            ks = {}
            for e in prof.events():
                if "bw_track" in e.name or "bw_localize" in e.name or "pnp_kernel" in e.name:
                    k = e.name.split("(")[0].split("<")[0].replace("void pvio::", "").replace("pvio::", "")
                    ks[k] = ks.get(k, 0.0) + e.device_time / 5
            line += "; device us per call: " + ", ".join(f"{k} {v:.1f}" for k, v in sorted(ks.items()))
        except Exception as e:  # the wall times above stand on their own
            line += f"; profiler unavailable: {e}"
        print(line, flush=True)
        ba.close()


if __name__ == "__main__":
    main()
