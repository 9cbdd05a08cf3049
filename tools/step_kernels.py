"""Per-kernel CUDA time of the batched Gauss-Newton step that bench.py measures (cfg2, W = 4096 windows,
batch_gn_step(W, 1e-8, apply=False)), from torch.profiler with CUDA activities in a run of its own, with the name and
power limit of the GPU it ran on.  The update sweep's achieved rate is its compulsory traffic (update_bytes) over its
kernel time.

    python tools/step_kernels.py [--windows W] [--steps S] [--warmup K] [--out DIR]

--out DIR writes DIR/step_kernels.json and DIR/step_kernels.md beside the table printed on stdout.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def update_bytes(M, K):
    """Compulsory bytes of update_obs_kernel<float, ., ., 0> for one window: the fp32 h record (24 B) and the frame-major
    observation (16 B) of every residual block; LmRec, rho, LmAux, lm_scale (64 B) read and rho_cand, dx_lm (16 B)
    written per landmark."""
    return K * (24 + 16) + M * (16 + 8 + 32 + 8) + M * (8 + 8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch
    from torch.profiler import profile, ProfilerActivity
    from bench import gpu_identity
    from synthetic import synth
    from pvio_b200.bundle_adjustor import BundleAdjustor

    if not torch.cuda.is_available():
        raise SystemExit("step_kernels: no CUDA device")
    W = args.windows
    win, st, _ = synth.make_cfg2()
    ba = BundleAdjustor(max_windows=W, max_frames=win.N, max_landmarks=512, max_obs=4608)
    ba.batch_set(0, win, st)
    ba.batch_replicate(W)
    ba.batch_upload(W)
    for _ in range(args.warmup):
        ba.batch_gn_step(W, 1e-8, apply=False)
    ba.sync()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            ba.batch_gn_step(W, 1e-8, apply=False)
        ba.sync()
        torch.cuda.synchronize()
    ba.close()

    rows = []
    for e in prof.key_averages():
        us = getattr(e, "device_time_total", None)
        if us is None:
            us = e.cuda_time_total
        if us > 0:
            rows.append({"kernel": e.key, "calls": e.count, "ms_per_step": us / 1e3 / args.steps})
    rows.sort(key=lambda r: -r["ms_per_step"])
    total = sum(r["ms_per_step"] for r in rows)
    upd = [r for r in rows if "update_obs_kernel" in r["kernel"]]
    ub = update_bytes(win.M, win.K)
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "windows": W, "steps": args.steps,
           "kernel_ms_per_step": total, "kernels": rows,
           "update_bytes_per_window": ub,
           "update_gbs": ub * W / (upd[0]["ms_per_step"] * 1e-3) / 1e9 if upd else None}

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; cfg2, {W} windows, {args.steps} steps",
             "", "| kernel | calls / step | ms / step | share |", "|---|---|---|---|"]
    for r in rows:
        lines.append(f"| `{r['kernel'][:90]}` | {r['calls'] / args.steps:g} | {r['ms_per_step']:.3f} | "
                     f"{100 * r['ms_per_step'] / total:.1f} % |")
    lines.append(f"| total kernel time | | {total:.3f} | |")
    if upd:
        lines += ["", f"update_obs_kernel: {upd[0]['ms_per_step']:.3f} ms / step, {ub / 1e3:.0f} KB / window compulsory -> "
                      f"{res['update_gbs']:.0f} GB/s ({100 * res['update_gbs'] / 3350:.0f} % of the 3.35 TB/s data-sheet HBM rate)"]
    text = "\n".join(lines)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "step_kernels.json"), "w") as f:
            json.dump(res, f, indent=1)
        with open(os.path.join(args.out, "step_kernels.md"), "w") as f:
            f.write(text + "\n")
    return 0


if __name__ == "__main__":
    sys.exit(main())
