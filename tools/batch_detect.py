"""Time of pvio_b200_batch_detect_keypoints (OpenCvImage::detect_keypoints, opencv_image.cpp:54-86, for n frames in one
call) in the steady state of a tracker: every frame is cached in its slot by a preceding batch_track_keypoints (raw
frames, CLAHE 6.0 on 8 x 8 tiles on the device) and has 120-300 existing keypoints; keypoint_distance 25.  Shapes
alternate between 752 x 480 and 512 x 512; frames and points are tiled from 8 seeds.  Beside it, the same frames as a
loop of single pvio_b200_detect_keypoints calls, one handle per sequence whose frame is cached by track_keypoints.  A
torch.profiler pass of its own per size gives the device time of every kernel and copy of one batched call.  The GPU's
name and power limit are read in the same run.

    python tools/batch_detect.py [--sizes 1,8,132,528] [--reps 20] [--loop-max 132] [--out DIR]

Wall times are host clocks around the C call alone (every call ends in a synchronise).  Medians of --reps calls after
3 warm-up calls.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CLAHE = (6.0, 8, 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--loop-max", type=int, default=132)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from bench import gpu_identity
    from synthetic import synth
    from pvio_b200 import _lib, klt
    from pvio_b200.detect import pack_requests
    from pvio_b200.bundle_adjustor import BundleAdjustor

    if not torch.cuda.is_available():
        raise SystemExit("batch_detect: no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    kinds = []
    for s in range(8):
        size = (752, 480) if s % 2 == 0 else (512, 512)
        A, B, pts, _ = synth.make_klt_pair(seed=1700 + s, size=size, n_points=100)
        r = np.random.default_rng(1700 + s)
        m = int(r.integers(120, 301))
        ex = np.stack([r.uniform(20, size[0] - 20, m), r.uniform(20, size[1] - 20, m)], 1)
        kinds.append({"frames": (A, B), "pts": pts, "existing": ex, "shape": (size[1], size[0])})
    res = {"gpu": gpu_identity(torch.cuda.current_device()),
           "frames": "cached by batch_track_keypoints (raw frames, CLAHE 6.0 on the device), 120-300 existing keypoints, "
                     "keypoint_distance 25, 752x480 / 512x512 alternating, make_klt_pair seeds 1700..1707 tiled",
           "reps": args.reps, "sizes": []}
    lib = None

    def batch_setup(ba, n):
        """n slots holding frames 1 and 2 of their sequence; the requests detect on frame 2"""
        pairs = [{"slot": i, "prev_id": 1, "next_id": 2, "prev": kinds[i % 8]["frames"][0], "next": kinds[i % 8]["frames"][1],
                  "pts": kinds[i % 8]["pts"]} for i in range(n)]
        klt.batch_track_keypoints(ba, pairs, clahe_clip=CLAHE[0])
        reqs = [{"slot": i, "frame_id": 2, "shape": kinds[i % 8]["shape"], "keypoints": kinds[i % 8]["existing"],
                 "keypoint_distance": 25.0} for i in range(n)]
        return pack_requests(reqs)

    def call(ba, n, cr):
        ba._ck(lib.pvio_b200_batch_detect_keypoints(ba.h, n, cr, *CLAHE))

    def timed_batch(ba, n, reps):
        cr, outs, keep = batch_setup(ba, n)
        wall = []
        for r in range(3 + reps):
            t0 = time.perf_counter()
            call(ba, n, cr)
            t1 = time.perf_counter()
            if r >= 3:
                wall.append((t1 - t0) * 1e3)
        return float(np.median(wall))

    def timed_loop(n, reps):
        """one handle per sequence, its frame 2 cached by track_keypoints; single pvio_b200_detect_keypoints calls"""
        fn = lib.pvio_b200_detect_keypoints
        hs = [BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64) for _ in range(n)]
        try:
            bufs = []
            for i in range(n):
                kd = kinds[i % 8]
                klt.track_keypoints(hs[i], kd["frames"][0], kd["frames"][1], kd["pts"], prev_id=1, next_id=2,
                                    clahe_clip=CLAHE[0])
                ex = np.ascontiguousarray(kd["existing"])
                out = np.zeros((2048, 2))
                bufs.append((ex, out, C.c_int(), kd["shape"]))
            wall = []
            for r in range(1 + reps):
                t = 0.0
                for i in range(n):
                    ex, out, cnt, (h, w) = bufs[i]
                    t0 = time.perf_counter()
                    hs[i]._ck(fn(hs[i].h, 2, None, w, h, w, *CLAHE, _lib.ptr(ex), len(ex), 25.0, 2048,
                                 _lib.ptr(out), C.byref(cnt), None, None))
                    t += time.perf_counter() - t0
                if r >= 1:
                    wall.append(t * 1e3)
            return float(np.median(wall))
        finally:
            for b in hs:
                b.close()

    ba = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    lib = ba.lib
    for n in sizes:
        wall = timed_batch(ba, n, args.reps)
        row = {"n": n, "wall_ms": wall, "wall_ms_per_frame": wall / n}
        if n <= args.loop_max:
            lw = timed_loop(n, max(3, args.reps // 4))
            row.update({"loop_wall_ms": lw, "loop_wall_ms_per_frame": lw / n})
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)

    # torch.profiler: one pass of its own per size, 5 steady-state calls
    from torch.profiler import profile, ProfilerActivity
    res["profile"] = []
    for n in sizes:
        cr, outs, keep = batch_setup(ba, n)
        call(ba, n, cr)
        torch.cuda.synchronize()
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                call(ba, n, cr)
            torch.cuda.synchronize()
        rows = []
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                rows.append({"name": e.key, "calls_per_batch": e.count / reps, "ms_per_batch": us / 1e3 / reps})
        rows.sort(key=lambda r: -r["ms_per_batch"])
        res["profile"].append({"n": n, "rows": rows})
    ba.close()

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; {res['frames']}; median of {args.reps} calls",
             "", "| frames | batch call wall (ms) | per frame (ms) | single-call loop wall (ms) | per frame (ms) |",
             "|---|---|---|---|---|"]
    for r in res["sizes"]:
        loop = f"{r['loop_wall_ms']:.2f} | {r['loop_wall_ms_per_frame']:.3f}" if "loop_wall_ms" in r else "- | -"
        lines.append(f"| {r['n']} | {r['wall_ms']:.3f} | {r['wall_ms_per_frame']:.4f} | {loop} |")
    for p in res["profile"]:
        lines += ["", f"device activity of one batch_detect_keypoints({p['n']}):", "", "| kernel / copy | calls | ms |",
                  "|---|---|---|"]
        for r in p["rows"]:
            lines.append(f"| `{r['name'][:90]}` | {r['calls_per_batch']:g} | {r['ms_per_batch']:.3f} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_detect.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "batch_detect.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
