"""Per-kernel CUDA time of the batched Gauss-Newton step that bench.py measures (cfg2, W = 4096 windows,
batch_gn_step(W, 1e-8, apply=False)), from torch.profiler with CUDA activities in a run of its own, with the name and
power limit of the GPU it ran on.  Beside each kernel's time it prints a compulsory-byte model of the kernel (the
*_bytes functions below, per window, from the shapes) and the rate that model implies, against the data sheet's HBM rate.

    python tools/step_kernels.py [--windows W] [--steps S] [--warmup K] [--out DIR] [--table-bytes B] [--jr-records]

--table-bytes / --jr-records describe the build being profiled: bytes per entry of the frame-major table (10: keypoint +
16-bit landmark index; 16: the earlier padded record) and whether the linearise sweep's (j.j, j.r) pairs make a round
trip through HBM (the earlier layout, and today's layout when several CTAs share a window).

--out DIR writes DIR/step_kernels.json and DIR/step_kernels.md beside the table printed on stdout.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


# cfg2 as bench.py allocates it: every landmark anchored in frame 0 and seen by every other frame, frames 0 and 1 fixed
def table_slots(N, M):
    """Entries of the frame-major table a sweep walks: N - 1 segments (t, 0) of M blocks, each on whole rows of 32."""
    return (N - 1) * ((M + 31) // 32) * 32


def lin_bytes(N, M, K, slots, Ncap, Mcap, table_bytes=10, jr=False, nfree=None):
    """lin_obs_kernel<true, float, ...> (either instantiation) + its lm_finish epilogue, one window: the table (table_bytes per slot), LmRec (16 B)
    and rho (8 B) per landmark read; the fp32 h record (24 B) of every (landmark, free target) written; w_l (8), mask (4),
    LmAux (32) and lm_scale (8) per landmark written; the direct and reduced system blocks written (fp64).  jr: the
    (j.j, j.r) pair (8 B) of every (landmark, target) written and read back."""
    nfree = N - 2 if nfree is None else nfree
    npc = Ncap * (Ncap + 1) // 2
    b = slots * table_bytes + M * (16 + 8) + nfree * M * 24 + M * (8 + 4 + 32 + 8)
    b += 8 * (npc * 36 + Ncap * 36 + 2 * Ncap * 6 + 1)
    if jr:
        b += 2 * (N - 1) * M * 8
    return b


def schur_bytes(N, M, K, slots, Ncap, Mcap, nfree=None):
    """schur_kernel<float, 128, 4>, one window: the h records of the free frames (24 B each) over the padded landmark
    range, w_l (8) and mask (4) per landmark, the reduced system read and written (fp64)."""
    nfree = N - 2 if nfree is None else nfree
    Mp = (M + 63) // 64 * 64
    npc = Ncap * (Ncap + 1) // 2
    return nfree * Mp * 24 + Mp * (8 + 4) + 2 * 8 * (npc * 36 + Ncap * 6)


def update_bytes(M, K, table_bytes=10):
    """Compulsory bytes of update_obs_kernel<float, ., ., 0> for one window: the fp32 h record (24 B) and the frame-major
    table entry (table_bytes: 8 B keypoint + 2 B landmark index) of every residual block; LmRec, rho, LmAux, lm_scale
    (64 B) read and rho_cand, dx_lm (16 B) written per landmark."""
    return K * (24 + table_bytes) + M * (16 + 8 + 32 + 8) + M * (8 + 8)


def solve_bytes(N, M, K, slots, Ncap, Mcap):
    """solve_kernel_visual + aux_cost_kernel, one window: the reduced system and gradient read (fp64), the pose step and
    its scaled direction written."""
    npc = Ncap * (Ncap + 1) // 2
    return 8 * (npc * 36 + Ncap * 36 + 2 * Ncap * 6) + 8 * 2 * Ncap * 15


def kernel_bytes(name, N, M, K, Ncap, Mcap, table_bytes, jr):
    slots = table_slots(N, M)
    if "lin_obs_kernel" in name:
        return lin_bytes(N, M, K, slots, Ncap, Mcap, table_bytes, jr)
    if "schur_kernel" in name:
        return schur_bytes(N, M, K, slots, Ncap, Mcap)
    if "update_obs_kernel" in name:
        return update_bytes(M, K, table_bytes)
    if "solve_kernel" in name:
        return solve_bytes(N, M, K, slots, Ncap, Mcap)
    return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    ap.add_argument("--table-bytes", type=int, default=10, choices=[10, 16])
    ap.add_argument("--jr-records", action="store_true")
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
            r = {"kernel": e.key, "calls": e.count, "ms_per_step": us / 1e3 / args.steps}
            kb = kernel_bytes(e.key, win.N, win.M, win.K, win.N, 512, args.table_bytes, args.jr_records)
            if kb is not None:
                r["bytes_per_window"] = kb
                r["gbs"] = kb * W / (r["ms_per_step"] * 1e-3) / 1e9
            rows.append(r)
    rows.sort(key=lambda r: -r["ms_per_step"])
    total = sum(r["ms_per_step"] for r in rows)
    modelled = sum(r.get("bytes_per_window", 0) for r in rows)
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "windows": W, "steps": args.steps,
           "table_bytes": args.table_bytes, "jr_records": args.jr_records,
           "kernel_ms_per_step": total, "kernels": rows, "modelled_bytes_per_window": modelled,
           "modelled_gbs": modelled * W / (total * 1e-3) / 1e9}

    g = res["gpu"]
    lines = [f"GPU: {g.get('name')}, power limit {g.get('power_limit_w')} W; cfg2, {W} windows, {args.steps} steps; "
             f"table {args.table_bytes} B / entry, jr records {'yes' if args.jr_records else 'no'}",
             "", "| kernel | calls / step | ms / step | share | KB / window (model) | GB/s | of 3.35 TB/s |",
             "|---|---|---|---|---|---|---|"]
    for r in rows:
        bw = (f"{r['bytes_per_window'] / 1e3:.0f} | {r['gbs']:.0f} | {100 * r['gbs'] / 3350:.0f} %"
              if "gbs" in r else "| |")
        lines.append(f"| `{r['kernel'][:90]}` | {r['calls'] / args.steps:g} | {r['ms_per_step']:.3f} | "
                     f"{100 * r['ms_per_step'] / total:.1f} % | {bw} |")
    lines.append(f"| total kernel time | | {total:.3f} | | {modelled / 1e3:.0f} | {res['modelled_gbs']:.0f} | "
                 f"{100 * res['modelled_gbs'] / 3350:.0f} % |")
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
