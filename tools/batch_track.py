"""Time of pvio_b200_batch_track_keypoints (OpenCvImage::track_keypoints, opencv_image.cpp:88-136, for n sequences in
one call) in the steady state of a tracker: every pair's previous frame is cached in its slot, its next frame arrives
raw (CLAHE 6.0 on 8 x 8 tiles on the device) with 500 points whose initial guesses carry outliers.  Shapes alternate
between 752 x 480 and 512 x 512; frames and points are tiled from 8 seeds.  Beside it, the same pairs as a loop of single
pvio_b200_track_keypoints calls, one handle per sequence so that each keeps its own frames cached.  A torch.profiler pass
of its own per size gives the device time of every kernel and copy of one batched call.  The GPU's name and power limit
are read in the same run.

    python tools/batch_track.py [--sizes 1,8,132,528] [--reps 20] [--loop-max 132] [--out DIR]

Wall times are host clocks around the C call alone (every call ends in a synchronise); the pair records are updated
outside the timed region.  Medians of --reps calls after 3 warm-up calls.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ARGS = (3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99)     # PVIO's constants: max_level .. ransac_confidence


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
    from pvio_b200.bundle_adjustor import BundleAdjustor

    if not torch.cuda.is_available():
        raise SystemExit("batch_track: no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    kinds = []
    for s in range(8):
        size = (752, 480) if s % 2 == 0 else (512, 512)
        A, B, _, _ = synth.make_klt_pair(seed=960 + s, size=size)
        r = np.random.default_rng(960 + s)
        pts = np.stack([r.uniform(25, size[0] - 25, 500), r.uniform(25, size[1] - 25, 500)], 1).astype(np.float32)
        init = pts.copy()
        a = r.choice(500, 50, replace=False)
        init[a] += r.uniform(-6, 6, (50, 2)).astype(np.float32)
        b = r.choice(500, 25, replace=False)
        init[b] += r.uniform(-40, 40, (25, 2)).astype(np.float32)
        kinds.append({"frames": (A, B), "pts": pts, "init": init, "shape": (size[1], size[0])})
    res = {"gpu": gpu_identity(torch.cuda.current_device()),
           "pairs": "500 points (a tenth of the guesses 6 px off, a twentieth 40 px off), raw next frame with CLAHE, "
                    "752x480 / 512x512 alternating, make_klt_pair seeds 960..967 tiled; previous frame cached",
           "reps": args.reps, "sizes": []}
    lib = None

    def batch_setup(ba, n):
        """n slots holding frame 1 of their sequence; returns a step(k) that readies call k (prev id k cached)"""
        pairs = [{"slot": i, "prev_id": 1, "next_id": 2, "prev": kinds[i % 8]["frames"][0],
                  "next": kinds[i % 8]["frames"][1], "pts": kinds[i % 8]["pts"], "init": kinds[i % 8]["init"]}
                 for i in range(n)]
        klt.batch_track_keypoints(ba, pairs, *ARGS[:3], clahe_clip=6.0)
        cp, outs, keep = klt.pack_pairs(pairs)
        frame_ptr = [[_lib.ptr(np.ascontiguousarray(f)) for f in k["frames"]] for k in kinds]

        def step(k):                        # call k: frame k (cached) -> frame k + 1 (new, raw)
            for i in range(n):
                c = cp[i]
                c.prev_id, c.next_id, c.prev = k, k + 1, None
                c.next = frame_ptr[i % 8][k % 2]
                np.copyto(outs[i][0], kinds[i % 8]["init"])
        return cp, step, (keep, frame_ptr, outs)

    def timed_batch(ba, n, reps):
        cp, step, keep = batch_setup(ba, n)
        wall, k = [], 2
        for r in range(3 + reps):
            step(k)
            t0 = time.perf_counter()
            ba._ck(lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
            t1 = time.perf_counter()
            k += 1
            if r >= 3:
                wall.append((t1 - t0) * 1e3)
        return float(np.median(wall))

    def timed_loop(n, reps):
        """one handle per sequence, single pvio_b200_track_keypoints calls over the same steady-state pairs"""
        fn = lib.pvio_b200_track_keypoints
        hs = [BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64) for _ in range(n)]
        try:
            bufs = []
            for i in range(n):
                kd = kinds[i % 8]
                frames = [np.ascontiguousarray(f) for f in kd["frames"]]
                nxt = kd["init"].copy()
                st = np.zeros(500, np.uint8)
                bufs.append((frames, [_lib.ptr(f) for f in frames], _lib.ptr(kd["pts"]), nxt,
                             _lib.ptr(nxt), st, _lib.ptr(st), kd["shape"]))
            for i in range(n):                  # frame 1 -> 2 with both frames given: frame 2 is cached
                frames, fp, pp, nxt, np_, st, sp, (h, w) = bufs[i]
                hs[i]._ck(fn(hs[i].h, 1, fp[0], 2, fp[1], w, h, w, pp, np_, sp, 500, *ARGS))
            wall, k = [], 2
            for r in range(1 + reps):
                t = 0.0
                for i in range(n):
                    frames, fp, pp, nxt, np_, st, sp, (h, w) = bufs[i]
                    np.copyto(nxt, kinds[i % 8]["init"])
                    t0 = time.perf_counter()
                    hs[i]._ck(fn(hs[i].h, k, None, k + 1, fp[k % 2], w, h, w, pp, np_, sp, 500, *ARGS))
                    t += time.perf_counter() - t0
                k += 1
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
        row = {"n": n, "wall_ms": wall, "wall_ms_per_pair": wall / n}
        if n <= args.loop_max:
            lw = timed_loop(n, max(3, args.reps // 4))
            row.update({"loop_wall_ms": lw, "loop_wall_ms_per_pair": lw / n})
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)

    # torch.profiler: one pass of its own per size, 5 steady-state calls
    from torch.profiler import profile, ProfilerActivity
    res["profile"] = []
    for n in sizes:
        cp, step, keep = batch_setup(ba, n)
        step(2)
        ba._ck(lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
        k = 3
        torch.cuda.synchronize()
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                step(k)
                ba._ck(lib.pvio_b200_batch_track_keypoints(ba.h, n, cp, *ARGS))
                k += 1
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
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; {res['pairs']}; median of {args.reps} calls",
             "", "| pairs | batch call wall (ms) | per pair (ms) | single-call loop wall (ms) | per pair (ms) |",
             "|---|---|---|---|---|"]
    for r in res["sizes"]:
        loop = f"{r['loop_wall_ms']:.2f} | {r['loop_wall_ms_per_pair']:.3f}" if "loop_wall_ms" in r else "- | -"
        lines.append(f"| {r['n']} | {r['wall_ms']:.3f} | {r['wall_ms_per_pair']:.4f} | {loop} |")
    for p in res["profile"]:
        lines += ["", f"device activity of one batch_track_keypoints({p['n']}):", "", "| kernel / copy | calls | ms |",
                  "|---|---|---|"]
        for r in p["rows"]:
            lines.append(f"| `{r['name'][:90]}` | {r['calls_per_batch']:g} | {r['ms_per_batch']:.3f} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_track.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "batch_track.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
