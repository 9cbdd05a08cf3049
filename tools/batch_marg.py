"""Device time of pvio_b200_batch_marginalize (BundleAdjustor::marginalize_frame(0) of a whole batch, the new priors kept
in the slots) on cfg3 windows (N = 9, M = 300; the batch tiles the 8 windows of seeds 648 + i), beside the same windows
marginalised one pvio_b200_ba_marginalize call at a time on the same handle, the CPU port over all usable cores, and one
keyframe cycle of BASELINE config 5 (upload + batch_solve + batch_marginalize of 8 cfg3 windows).  A per-kernel breakdown
of one batch (torch.profiler, a pass of its own) closes the run.  The GPU's name and power limit are read in the same run.

    python tools/batch_marg.py [--sizes 1,8,132,528,1024] [--reps 20] [--profile-n 132] [--out DIR]

The timed calls repeat the marginalisation of one upload.  Each call does the same work: the dense system depends on the
window's old prior only through Lambda = S^T S, formed at upload, and the eigen-solver sees only that system.
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
    ap.add_argument("--sizes", default="1,8,132,528,1024")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--loop-max", type=int, default=132)
    ap.add_argument("--profile-n", type=int, default=132)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from bench import gpu_identity
    from oracle import c_oracle
    from synthetic import synth
    from pvio_b200.bundle_adjustor import BundleAdjustor

    if not torch.cuda.is_available():
        raise SystemExit("batch_marg: no CUDA device")
    sizes = [int(s) for s in args.sizes.split(",")]
    kinds = [synth.make_cfg3(seed=648 + i)[:2] for i in range(8)]
    Wmax = max(sizes)
    ba = BundleAdjustor(max_windows=Wmax, max_frames=9, max_landmarks=320, max_obs=2560)
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "windows": "cfg3 N=9 M=300, seeds 648..655 tiled",
           "reps": args.reps, "sizes": []}

    def med_ms(fn, reps, warm=3):
        for _ in range(warm):
            fn()
        ts = []
        for _ in range(reps):
            ba.timer_start()
            fn()
            ts.append(ba.timer_stop())
        return float(np.median(ts)), float(np.min(ts)), float(np.max(ts))

    for n in sizes:
        for i in range(n):
            ba.batch_set(i, *kinds[i % 8])
        ba.batch_upload(n)
        med, lo, hi = med_ms(lambda: ba.batch_marginalize(n), args.reps)
        row = {"n": n, "batch_ms": med, "batch_ms_min": lo, "batch_ms_max": hi, "batch_ms_per_window": med / n}
        if n <= args.loop_max:           # the same windows, one ba_marginalize call each (host round trip per call)
            def loop():
                for i in range(n):
                    ba.marginalize_frame(*kinds[i % 8], index=0)
            row["loop_ms"] = med_ms(loop, max(3, args.reps // 4), warm=1)[0]
        t0 = time.perf_counter()         # the CPU port, n independent windows over all usable cores
        used, _ = c_oracle.batch("marginalize", *kinds[0], n_windows=n, n_threads=0)
        row["cpu_port_ms"] = (time.perf_counter() - t0) * 1e3
        row["cpu_threads"] = int(used)
        res["sizes"].append(row)
        print(json.dumps(row), flush=True)

    # keyframe cycle of BASELINE config 5: 8 cfg3 windows, upload + full solve + marginalisation (re-packed with their host
    # priors before each cycle, outside the timed region)
    def pack8():
        for i in range(8):
            ba.batch_set(i, *kinds[i])
    cyc, solve_only = [], []
    for r in range(args.reps + 3):
        pack8()
        ba.timer_start()
        ba.batch_upload(8)
        ba.batch_solve(8, max_iterations=10)
        t_solve = ba.timer_stop()
        ba.timer_start()
        ba.batch_marginalize(8)
        t_marg = ba.timer_stop()
        if r >= 3:
            solve_only.append(t_solve)
            cyc.append(t_solve + t_marg)
    res["cfg5_cycle"] = {"upload_solve_ms": float(np.median(solve_only)), "cycle_ms": float(np.median(cyc)),
                         "marginalize_ms": float(np.median(np.array(cyc) - np.array(solve_only)))}
    print(json.dumps(res["cfg5_cycle"]), flush=True)

    # per-kernel breakdown of one batch of profile_n windows
    prof_rows = []
    if args.profile_n > 0:
        from torch.profiler import profile, ProfilerActivity
        n = args.profile_n
        for i in range(n):
            ba.batch_set(i, *kinds[i % 8])
        ba.batch_upload(n)
        ba.batch_marginalize(n)
        ba.sync()
        torch.cuda.synchronize()
        reps = 10
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(reps):
                ba.batch_marginalize(n)
            ba.sync()
            torch.cuda.synchronize()
        for e in prof.key_averages():
            us = getattr(e, "device_time_total", None)
            if us is None:
                us = e.cuda_time_total
            if us > 0:
                prof_rows.append({"kernel": e.key, "calls_per_batch": e.count / reps, "ms_per_batch": us / 1e3 / reps})
        prof_rows.sort(key=lambda r: -r["ms_per_batch"])
        res["profile"] = {"n": n, "kernels": prof_rows}
    ba.close()

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; {res['windows']}; median of {args.reps} calls",
             "", "| windows | batch_marginalize (ms) | per window (ms) | ba_marginalize loop (ms) | CPU port (ms, threads) |",
             "|---|---|---|---|---|"]
    for r in res["sizes"]:
        loop = f"{r['loop_ms']:.2f}" if "loop_ms" in r else "-"
        lines.append(f"| {r['n']} | {r['batch_ms']:.3f} | {r['batch_ms_per_window']:.4f} | {loop} | "
                     f"{r['cpu_port_ms']:.1f} ({r['cpu_threads']}) |")
    c = res["cfg5_cycle"]
    lines += ["", f"config 5 keyframe cycle (8 windows): upload + batch_solve {c['upload_solve_ms']:.3f} ms, "
                  f"+ batch_marginalize {c['marginalize_ms']:.3f} ms = {c['cycle_ms']:.3f} ms"]
    if prof_rows:
        lines += ["", f"kernels of one batch_marginalize({res['profile']['n']}):", "",
                  "| kernel | calls | ms |", "|---|---|---|"]
        for r in prof_rows:
            lines.append(f"| `{r['kernel'][:80]}` | {r['calls_per_batch']:g} | {r['ms_per_batch']:.3f} |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_marg.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "batch_marg.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
