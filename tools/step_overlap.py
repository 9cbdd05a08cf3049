"""How the batched GN step (batch_gn_step) fills the GPU with and without its sub-batch split.

    python tools/step_overlap.py [--windows 4096] [--hetero] [--steps 3] [--parts 1,0]
    python tools/step_overlap.py --time [--windows 1024,2048,4096] [--parts 1,2,3,4] [--hetero]

Default mode: one torch.profiler pass per sub-batch count over a few steps.  It prints each kernel's start and end per
stream (relative to the step's first kernel), then per step the span, the time with no kernel of the step running on
any stream, and each idle gap between one kernel's end and the next kernel's start.  --time: CUDA-event step times
(no profiler) for every (windows, sub-batch count), repeated and interleaved, and the stage times of last_kernel_ms.
--parts: 0 lets the library choose (what bench.py runs), > 0 forces that many sub-batches.  cfg2 windows, or bench.py's
five-kind heterogeneous batch with --hetero."""
import argparse
import json
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C  # noqa: E402

import numpy as np  # noqa: E402

from pvio_b200 import _lib as L  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from synthetic import synth  # noqa: E402


def hetero_kinds():
    """bench.py's heterogeneous batch: 5 window kinds (sizes, anchors, visibility, fixed sets differ)"""
    kinds = [synth.make_cfg2(N=10, M=500, seed=41)[:2], synth.make_cfg2(N=10, M=420, staggered=True, seed=42)[:2],
             synth.make_cfg2(N=8, M=300, seed=43)[:2], synth.make_cfg2(N=9, M=350, staggered=True, seed=44)[:2],
             synth.make_cfg2(N=10, M=500, seed=45)[:2]]
    kinds[2][0].frame_fixed[:] = 0; kinds[2][0].frame_fixed[0] = 1; kinds[2][0].frame_fixed[5] = 1
    return kinds


def make(W, hetero):
    ba = BundleAdjustor(max_windows=W, max_frames=10, max_landmarks=512, max_obs=4608)
    if hetero:
        pas = [L.PackedArgs(w, s) for w, s in hetero_kinds()]
        for i in range(W):
            p = pas[i % len(pas)]
            ba.lib.pvio_b200_batch_set_window(ba.h, i, C.byref(p.cw), C.byref(p.cs))
    else:
        w, st, _ = synth.make_cfg2()
        ba.batch_set(0, w, st)
        ba.batch_replicate(W)
    ba.batch_upload(W)
    return ba


def set_parts(ba, spec):
    assert ba.lib.pvio_b200_internal_set_step_split(ba.h, int(spec)) == 0


def short(name):
    for k in ("lin_obs_kernel", "schur_kernel", "solve_kernel_visual", "solve_kernel", "update_obs_kernel",
              "aux_cost_kernel", "lm_finish_kernel", "zero_system_kernel"):
        if k in name:
            return k
    return name[:40]


def profile(args):
    from torch.profiler import ProfilerActivity, profile as tprof
    out = {}
    for spec in args.parts.split(","):
        ba = make(args.windows[0], args.hetero)
        set_parts(ba, spec)
        for _ in range(3):
            ba.batch_gn_step(args.windows[0], 1e-8, apply=False)
        ba.sync()
        marks = []
        with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for _ in range(args.steps):
                marks.append(ba.kernel_launches)
                ba.batch_gn_step(args.windows[0], 1e-8, apply=False)
            ba.sync()
        per_step = (ba.kernel_launches - marks[0]) // args.steps
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "trace.json")
            prof.export_chrome_trace(path)
            ev = json.load(open(path))["traceEvents"]
        ks = sorted((e for e in ev if e.get("cat") == "kernel"), key=lambda e: e["ts"])
        print(f"\n=== windows {args.windows[0]}{' heterogeneous' if args.hetero else ''}, parts {spec}: "
              f"{per_step} kernels per step")
        if len(ks) < per_step * args.steps:       # the profiler dropped kernel records: no per-step split is possible
            print(f"   the trace holds {len(ks)} kernel records, {per_step * args.steps} were launched; run again")
            ba.close()
            continue
        ks = ks[-per_step * args.steps:]
        res = []
        for s in range(args.steps):
            step = ks[s * per_step:(s + 1) * per_step]
            t0 = step[0]["ts"]
            end = max(e["ts"] + e["dur"] for e in step)
            print(f"-- step {s}: stream  kernel  grid  start_us  end_us")
            for e in step:
                a = e.get("args", {})
                print(f"   {a.get('stream', e.get('tid'))!s:>6}  {short(e['name']):<20} {str(a.get('grid', '')):<16} "
                      f"{e['ts'] - t0:9.1f} {e['ts'] + e['dur'] - t0:9.1f}")
            # idle time: where no kernel of the step runs on any stream
            busy_end, idle, gaps = t0, 0.0, []
            for e in step:
                if e["ts"] > busy_end:
                    gaps.append((busy_end - t0, e["ts"] - busy_end, short(e["name"])))
                    idle += e["ts"] - busy_end
                busy_end = max(busy_end, e["ts"] + e["dur"])
            print(f"   span {end - t0:.1f} us, idle {idle:.1f} us; gaps (at, us, before): " +
                  ", ".join(f"({g[0]:.0f}, {g[1]:.1f}, {g[2]})" for g in gaps))
            res.append({"span_us": end - t0, "idle_us": idle})
        out[spec] = {"span_us": float(np.median([r["span_us"] for r in res])),
                     "idle_us": float(np.median([r["idle_us"] for r in res]))}
        ba.close()
    print("\nmedian per step:", json.dumps(out))


def timing(args):
    import torch
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
    res = {}
    for W in args.windows:
        ba = make(W, args.hetero)
        for _ in range(3):
            ba.batch_gn_step(W, 1e-8, apply=False)
        for rep in range(args.reps):
            for spec in args.parts.split(","):
                set_parts(ba, spec)
                for _ in range(2):
                    ba.batch_gn_step(W, 1e-8, apply=False)
                ba.sync()
                ba.last_kernel_ms(-1)
                ba.timer_start()
                for _ in range(args.steps):
                    ba.batch_gn_step(W, 1e-8, apply=False)
                ms = ba.timer_stop() / args.steps
                st = [ba.last_kernel_ms(i) for i in (1, 2, 3)]
                res.setdefault((W, spec), []).append((ms, *st))
        ba.close()
    for (W, spec), v in res.items():
        v = np.array(v)
        print(json.dumps({"windows": W, "parts": spec, "ms_per_step": [round(x, 4) for x in v[:, 0]],
                          "median_ms": round(float(np.median(v[:, 0])), 4),
                          "stage_lin_schur_ms": round(float(np.median(v[:, 1])), 4),
                          "lin_ms": round(float(np.median(v[:, 2])), 4), "schur_ms": round(float(np.median(v[:, 3])), 4)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", default="4096")
    ap.add_argument("--hetero", action="store_true")
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--parts", default=None)
    ap.add_argument("--time", action="store_true")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    args.windows = [int(x) for x in args.windows.split(",")]
    if args.time:
        args.steps = args.steps or 20
        args.parts = args.parts or "1,2,3,4"
        timing(args)
    else:
        args.steps = args.steps or 3
        args.parts = args.parts or "1,0"
        profile(args)


if __name__ == "__main__":
    main()
