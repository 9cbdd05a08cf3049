"""Time of pvio_b200_batch_pnp_solve (visual_inertial_pnp, pnp.cpp:32-100, for n independent problems in one launch)
on 150-point inertial problems, tiled from 8 seeded problems of both calibrations (EUROC and TUMVI), beside the same
problems solved one pvio_b200_pnp_solve call at a time on the same handle.  A torch.profiler pass at one size (a pass of
its own) shows the single kernel of a batch.  The GPU's name and power limit are read in the same run.

    python tools/batch_pnp.py [--sizes 1,8,132,1024,4096] [--reps 20] [--profile-n 1024] [--out DIR]

Per size: the device time of the batched launch (the handle's CUDA events around it, as the summary's solve_seconds
gives it) and the host wall time of the whole call (pack, upload, kernel, read-back, synchronise), each the median of
--reps calls after 3 warm-up calls.  The problem descriptors are built once, outside the timed region, and every call
starts from the same initial frames, so every call does the same work.  The loop of single calls reports the sum of its
calls' kernel times and its wall time.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,1024,4096")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--loop-max", type=int, default=132)
    ap.add_argument("--profile-n", type=int, default=1024)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from bench import gpu_identity
    from synthetic import synth
    from pvio_b200 import _lib, pnp
    from pvio_b200.bundle_adjustor import BundleAdjustor

    if not torch.cuda.is_available():
        raise SystemExit("batch_pnp: no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    kinds = [synth.make_pnp(seed=651 + i, n_points=150, cal=synth.TUMVI if i % 2 else synth.EUROC) for i in range(8)]
    ba = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    lib = ba.lib
    res = {"gpu": gpu_identity(torch.cuda.current_device()),
           "problems": "150 points + IMU prior, make_pnp seeds 651..658 (EUROC / TUMVI alternating) tiled",
           "reps": args.reps, "sizes": []}
    opt = _lib.COptions(10, 1e6, 1, 0, 0.0)

    def packed(n):
        pbs, keep = (_lib.CPnpProblem * n)(), []
        for i in range(n):
            d = kinds[i % 8]
            pnp._fill_problem(pbs[i], keep, d['last'], d['imu'], d['pts'], d['zs'], d['cam_q'], d['cam_p'],
                              d['imu_q'], d['imu_p'], d['W'], True, 1.0)
        init = np.stack([kinds[i % 8]['frame'] for i in range(n)])
        return pbs, keep, init

    def timed(call, init, frames, reps, warm=3):
        wall, kern = [], []
        for r in range(warm + reps):
            frames[:] = init
            t0 = time.perf_counter()
            k = call()                   # every call ends in a synchronise
            t1 = time.perf_counter()
            if r >= warm:
                wall.append((t1 - t0) * 1e3)
                kern.append(k)
        return float(np.median(kern)), float(np.median(wall))

    for n in sizes:
        pbs, keep, init = packed(n)
        frames = init.copy()
        sms = (_lib.CSummary * n)()

        def batch():
            ba._ck(lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), 16, C.byref(opt), sms))
            return sms[0].solve_seconds * 1e3
        kern, wall = timed(batch, init, frames, args.reps)
        its = [sms[i].iterations for i in range(n)]
        row = {"n": n, "kernel_ms": kern, "wall_ms": wall, "kernel_ms_per_problem": kern / n,
               "iterations": [int(min(its)), int(max(its))]}
        if n <= args.loop_max:           # the same problems, one pnp_solve call each (host round trip per call)
            sm1 = _lib.CSummary()

            def loop():
                k = 0.0
                for i in range(n):
                    ba._ck(lib.pvio_b200_pnp_solve(ba.h, C.byref(pbs[i]), _lib.ptr(frames[i]),
                                                   C.byref(opt), C.byref(sm1)))
                    k += sm1.solve_seconds * 1e3
                return k
            lkern, lwall = timed(loop, init, frames, max(3, args.reps // 4), warm=1)
            row.update({"loop_kernel_ms": lkern, "loop_wall_ms": lwall})
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)

    prof_rows = []
    if args.profile_n > 0:
        from torch.profiler import profile, ProfilerActivity
        n = args.profile_n
        pbs, keep, init = packed(n)
        frames = init.copy()
        lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), 16, C.byref(opt), None)
        torch.cuda.synchronize()
        reps = 5
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                frames[:] = init
                ba._ck(lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), 16, C.byref(opt),
                                                     None))
            torch.cuda.synchronize()
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                prof_rows.append({"name": e.key, "calls_per_batch": e.count / reps, "ms_per_batch": us / 1e3 / reps})
        prof_rows.sort(key=lambda r: -r["ms_per_batch"])
        res["profile"] = {"n": n, "rows": prof_rows}
    ba.close()

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; {res['problems']}; median of {args.reps} calls",
             "", "| problems | batch kernel (ms) | per problem (ms) | batch call wall (ms) | "
                 "pnp_solve loop: kernels (ms) | loop wall (ms) |", "|---|---|---|---|---|---|"]
    for r in res["sizes"]:
        loop = f"{r['loop_kernel_ms']:.2f} | {r['loop_wall_ms']:.2f}" if "loop_kernel_ms" in r else "- | -"
        lines.append(f"| {r['n']} | {r['kernel_ms']:.3f} | {r['kernel_ms_per_problem']:.4f} | {r['wall_ms']:.3f} | "
                     f"{loop} |")
    if prof_rows:
        lines += ["", f"device activity of one batch_pnp_solve({res['profile']['n']}):", "",
                  "| kernel / copy | calls | ms |", "|---|---|---|"]
        for r in prof_rows:
            lines.append(f"| `{r['name'][:80]}` | {r['calls_per_batch']:g} | {r['ms_per_batch']:.3f} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_pnp.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "batch_pnp.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
