"""Time of undistorting raw camera frames inside pvio_b200_batch_track_keypoints (a lens per slot, remapped on the
device) against undistorting them on the host first, as PVIO's EuRoC reader does (cv::undistort with the EuRoC lens,
euroc_dataset_reader.cpp:70-74), for n sequences in the steady state of a tracker: every pair's previous frame is cached
in its slot, its next 752 x 480 frame arrives raw, CLAHE 6.0 on 8 x 8 tiles on the device, 500 points.

  A        raw frames, slot lenses: one batch_track_keypoints call
  B_all    cv2.undistort of every frame on the host (OpenCV's default thread count), then the same call without lenses
  B_one    the same with cv2.setNumThreads(1)

A torch.profiler pass of its own per size gives the device time of undistort_kernel in one call of A.  Both paths are
checked to give the same results.  The GPU's name and power limit are read in the same run.

    python tools/batch_undistort.py [--sizes 1,8,132,528] [--reps 10] [--out DIR]

Wall times are host clocks around the work of one call (every call ends in a synchronise); medians of --reps calls
after 3 warm-up calls.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARGS = (3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99)     # PVIO's constants: max_level .. ransac_confidence
EUROC_K = (458.654, 457.296, 367.215, 248.375)
EUROC_D = (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import cv2
    import numpy as np
    import torch
    from bench import gpu_identity
    from synthetic import synth
    from pvio_b200 import _lib, klt
    from pvio_b200.bundle_adjustor import BundleAdjustor
    from pvio_b200.undistort import RADTAN, set_lens

    if not torch.cuda.is_available():
        raise SystemExit("batch_undistort: no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    Kf = np.array([[EUROC_K[0], 0, EUROC_K[2]], [0, EUROC_K[1], EUROC_K[3]], [0, 0, 1]], np.float32)
    Df = np.array(EUROC_D, np.float32)
    kinds = []
    for s in range(8):
        A, B, _, _ = synth.make_klt_pair(seed=1960 + s, size=(752, 480))
        r = np.random.default_rng(1960 + s)
        pts = np.stack([r.uniform(25, 727, 500), r.uniform(25, 455, 500)], 1).astype(np.float32)
        kinds.append({"frames": (np.ascontiguousarray(A), np.ascontiguousarray(B)), "pts": pts})
    threads0 = cv2.getNumThreads()
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "cv2": cv2.__version__, "cv2_threads": threads0,
           "cpu_count": os.cpu_count(),
           "pairs": "EuRoC lens, 752x480 raw next frame, 500 points, CLAHE 6.0 8x8, previous frame cached; "
                    "make_klt_pair seeds 1960..1967 tiled",
           "reps": args.reps, "sizes": []}

    def setup(ba, n, lens):
        """n slots holding frame 1 of their sequence (undistorted on the host unless the slot has a lens); returns
        step(k), which readies call k and returns the host time it spent undistorting"""
        if lens:
            set_lens(ba, [{"slot": i, "model": RADTAN, "width": 752, "height": 480, "K": EUROC_K, "coeffs": EUROC_D}
                          for i in range(n)])
        und = (lambda f: f) if lens else (lambda f: cv2.undistort(f, Kf, Df))
        pairs = [{"slot": i, "prev_id": 1, "next_id": 2, "prev": und(kinds[i % 8]["frames"][0]),
                  "next": und(kinds[i % 8]["frames"][1]), "pts": kinds[i % 8]["pts"]} for i in range(n)]
        klt.batch_track_keypoints(ba, pairs, *ARGS[:3], clahe_clip=6.0)
        cp, outs, keep = klt.pack_pairs(pairs)
        dst = [np.zeros((480, 752), np.uint8) for _ in range(n)] if not lens else None
        raw_ptr = [[_lib.ptr(f) for f in k["frames"]] for k in kinds]
        dst_ptr = [_lib.ptr(d) for d in dst] if dst else None

        def step(k):                        # call k: frame k (cached) -> frame k + 1 (new, raw)
            for i in range(n):
                c = cp[i]
                c.prev_id, c.next_id, c.prev = k, k + 1, None
                np.copyto(outs[i][0], kinds[i % 8]["pts"])
            t0 = time.perf_counter()
            for i in range(n):
                if lens:
                    cp[i].next = raw_ptr[i % 8][k % 2]
                else:
                    cv2.undistort(kinds[i % 8]["frames"][k % 2], Kf, Df, dst[i])
                    cp[i].next = dst_ptr[i]
            return time.perf_counter() - t0
        return cp, step, outs, (keep, raw_ptr, dst, dst_ptr)

    def timed(n, lens, threads, reps):
        cv2.setNumThreads(threads)
        ba = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
        try:
            cp, step, outs, keep = setup(ba, n, lens)
            wall, host, k = [], [], 2
            for r in range(3 + reps):
                t_host = step(k)
                t0 = time.perf_counter()
                ba._ck(ba.lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
                t1 = time.perf_counter()
                k += 1
                if r >= 3:
                    wall.append((t1 - t0 + t_host) * 1e3)
                    host.append(t_host * 1e3)
            last = [(o[0].copy(), o[1].copy(), o[3].copy()) for o in outs]
            return float(np.median(wall)), float(np.median(host)), last
        finally:
            ba.close()
            cv2.setNumThreads(threads0)

    for n in sizes:
        a, _, ra = timed(n, True, threads0, args.reps)
        b_all, h_all, rb = timed(n, False, threads0, args.reps)
        b_one, h_one, _ = timed(n, False, 1, max(3, args.reps // 2))
        same = all(np.array_equal(x, y) for p, q in zip(ra, rb) for x, y in zip(p, q))
        row = {"n": n, "A_wall_ms": a, "B_all_wall_ms": b_all, "B_all_host_undistort_ms": h_all,
               "B_one_wall_ms": b_one, "B_one_host_undistort_ms": h_one, "results_equal": same}
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)

    from torch.profiler import profile, ProfilerActivity
    res["profile"] = []
    for n in sizes:                         # a handle of its own per size
        ba = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
        try:
            cp, step, outs, keep = setup(ba, n, True)
            step(2)
            ba._ck(ba.lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
            k, reps = 3, 5
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(reps):
                    step(k)
                    ba._ck(ba.lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
                    k += 1
                torch.cuda.synchronize()
        finally:
            ba.close()
        und_ms, total_ms = 0.0, 0.0
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            total_ms += us / 1e3 / reps
            if "undistort_kernel" in e.key:
                und_ms += us / 1e3 / reps
        px = n * 752 * 480                  # map 6 B, taps ~1 B, write 1 B per pixel
        row = {"n": n, "undistort_kernel_ms": und_ms, "device_ms_per_call": total_ms, "bytes_per_call": 8 * px,
               "undistort_kernel_GBps": 8 * px / (und_ms * 1e-3) / 1e9 if und_ms else None}
        res["profile"].append(row)
        print(json.dumps(row), flush=True)

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; cv2 {res['cv2']} with {threads0} threads "
             f"on {res['cpu_count']} CPUs; {res['pairs']}; median of {args.reps} calls", "",
             "| sequences | A: raw + slot lenses (ms) | B: cv2.undistort all threads + call (ms) | of it host undistort (ms) "
             "| B: cv2.undistort 1 thread + call (ms) | of it host undistort (ms) | same results |",
             "|---|---|---|---|---|---|---|"]
    for r in res["sizes"]:
        lines.append(f"| {r['n']} | {r['A_wall_ms']:.2f} | {r['B_all_wall_ms']:.2f} | {r['B_all_host_undistort_ms']:.2f} | "
                     f"{r['B_one_wall_ms']:.2f} | {r['B_one_host_undistort_ms']:.2f} | {r['results_equal']} |")
    lines += ["", "| sequences | undistort_kernel (ms) | device time of the call (ms) | bytes moved (8 B/px) | GB/s |",
              "|---|---|---|---|---|"]
    for r in res["profile"]:
        gbps = f"{r['undistort_kernel_GBps']:.0f}" if r["undistort_kernel_GBps"] else "-"
        lines.append(f"| {r['n']} | {r['undistort_kernel_ms']:.4f} | {r['device_ms_per_call']:.3f} | {r['bytes_per_call']} | {gbps} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_undistort.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "batch_undistort.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
