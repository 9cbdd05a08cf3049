"""Times pvio_b200_batch_feature_track against the host-driven chain it replaces (guesses in numpy,
batch_track_keypoints, the thinning on the host, batch_detect_keypoints, the append) at n sequences, and lists the
call's device time per kernel from a torch.profiler pass of its own.  Prints one JSON line; with --out also writes it.
Usage: python tools/batch_feature_track.py [--n 1 8 132 528] [--frames 6] [--out feature_track.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))      # the sequence generator and the host chain of the GPU test

from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.feature_track import batch_feature_track  # noqa: E402
from pvio_b200.undistort import set_lens  # noqa: E402
from test_gpu_batch_feature_track import CLIP, EUROC, KD, LENS_SLOT, Chain, _request, _seqs  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def run(n, n_frames, seqs):
    dev, ref = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64), \
        BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    try:
        for b in (dev, ref):
            set_lens(b, [dict(EUROC, slot=s) for s in range(LENS_SLOT, n, 8)])
        chains = [Chain(ref, s, seqs[s % 8]["K"]) for s in range(n)]
        t_call, t_chain, launches = [], [], 0
        for k in range(n_frames):
            reqs = [_request(seqs[s % 8], k, slot=s) for s in range(n)]
            dev.sync()
            l0 = dev.kernel_launches
            t0 = time.perf_counter()
            batch_feature_track(dev, reqs, keypoint_distance=KD, clahe_clip=CLIP)
            t1 = time.perf_counter()
            launches = dev.kernel_launches - l0
            for s in range(n):
                chains[s].step(reqs[s]["image"], k + 1, reqs[s]["map_frames"], reqs[s]["predict_q"])
            ref.sync()
            t2 = time.perf_counter()
            if k >= 2:                           # frames 0, 1: warm-up (first allocations, a new sequence)
                t_call.append(t1 - t0)
                t_chain.append(t2 - t1)
        # device time per kernel of one more call, profiled on its own
        import torch
        from torch.profiler import ProfilerActivity, profile
        reqs = [_request(seqs[s % 8], n_frames, slot=s) for s in range(n)]
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            batch_feature_track(dev, reqs, keypoint_distance=KD, clahe_clip=CLIP)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.key_averages():
            if e.device_type.name == "CUDA" and e.device_time_total > 0:
                kern[e.key[:60]] = round(e.device_time_total / 1000.0, 4)
        return {"n": n, "call_ms": round(1e3 * min(t_call), 3), "chain_ms": round(1e3 * min(t_chain), 3),
                "launches": launches, "kernel_ms": kern}
    finally:
        dev.close()
        ref.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--out")
    a = ap.parse_args()
    seqs = _seqs()
    rows = [run(n, a.frames, seqs) for n in a.n]
    res = {"card": card(), "rows": rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
