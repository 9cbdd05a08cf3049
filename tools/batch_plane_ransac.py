"""Time of pvio_b200_batch_window_plane_ransac (PlaneExtractor::work on resident slots) for n sequences of about 300
candidate tracks each, 40 % of them on a plane, with the device time of each kernel from a torch.profiler pass of its
own.  The GPU's name and power limit are read in the same run.

    python tools/batch_plane_ransac.py [--sizes 1,8,132,528] [--reps 5] [--out DIR]

Each slot holds three frames of a synthetic run and its tracks, anchored in the first frame and observed in all three.
Per size: the host wall time of the whole call (stage, 3 launches, replay, read-back), the median of --reps calls after
2 warm-up calls; the summed device time per kernel launch; and, for the host path the call replaces, the time of the
one thing it must do first -- download every slot's frames, inverse depths and anchors (pvio_b200_batch_window_download).
The host path's serial RANSAC per sequence in compiled code is not measured here.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def fill(bw, run, rec, slots, n_tracks, frac_on, seed):
    """every slot: three frames (0, 3, 6) of `run`, n_tracks tracks anchored in frame 0 -- frac_on of them on the floor
    z = -1.4, the others 0.3 .. 2 m off it -- observed in frames 1 and 2"""
    import numpy as np
    from pvio_b200.batch_window import Edit
    from synthetic import so3
    g = run.guess
    qc, pc = run.cam_pose(g.q[0], g.p[0])
    ids = {}
    for s in slots:
        bw.reset(s, run.w)
    for k, f in enumerate((0, 3, 6)):
        edits = []
        for s in slots:
            e = Edit(s).frame(np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]]), False, rec[f - 1] if k else None)
            if k == 0:
                rng = np.random.default_rng(seed + s)
                n_on = int(frac_on * n_tracks)
                z_w = np.r_[np.full(n_on, -1.4), -1.4 + rng.choice([-1, 1], n_tracks - n_on) * rng.uniform(0.3, 2, n_tracks - n_on)]
                X = np.c_[rng.uniform(3, 8, n_tracks), rng.uniform(-2, 2, n_tracks), z_w][rng.permutation(n_tracks)]
                for x in X:
                    y = so3.qrot(so3.qconj(qc), x - pc)
                    e.new.append((0, y[:2] / y[2], 1.0 / y[2]))
            else:
                e.obs = [(int(t), k, np.array([0.01 * k, 0.0])) for t in ids[s]]
            edits.append(e)
        got = bw.edit(edits)
        if k == 0:
            ids = {s: t for s, t in zip(slots, got)}
    return ids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,132,528")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tracks", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    from bench import gpu_identity
    from pvio_b200 import _lib
    from pvio_b200.batch_window import BatchWindows, PlaneRansac
    from pvio_b200.bundle_adjustor import BundleAdjustor
    from synthetic.sequence import Run

    sizes = [int(s) for s in args.sizes.split(",")]
    W = max(sizes)
    run = Run(F=8, N=8, M=40, seed=741)
    rec = _lib.PackedArgs(run.w, run.guess).keep["imu"].reshape(-1, 288)
    ba = BundleAdjustor(max_windows=W, max_frames=4, max_landmarks=args.tracks + 4, max_obs=4 * args.tracks)
    bw = BatchWindows(ba)
    ids = fill(bw, run, rec, list(range(W)), args.tracks, 0.4, 100)
    res = {"gpu": gpu_identity(torch.cuda.current_device()), "tracks": args.tracks, "on_plane": 0.4, "rows": []}
    for n in sizes:
        recs = [PlaneRansac(s, PlaneRansac.EXTRACT, ids[s]) for s in range(n)]
        out = None
        for _ in range(2):
            out = bw.plane_ransac(recs)
        assert all(o["status"] == _lib.PLANE_ACCEPTED for o in out)
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            bw.plane_ransac(recs)
            ts.append(time.perf_counter() - t0)
        dl = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            bw.download(list(range(n)), args.tracks + 4)
            dl.append(time.perf_counter() - t0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            bw.plane_ransac(recs)
            torch.cuda.synchronize()
        kern = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA and "pr_" in e.name:
                name = "pr_" + e.name.split("pr_")[1].split("(")[0].split("<")[0]
                kern[name] = kern.get(name, 0.0) + e.device_time_total / 1e3
        row = {"n": n, "wall_ms": 1e3 * float(np.median(ts)), "kernel_ms": kern,
               "iterations_mean": float(np.mean([o["iterations"] for o in out])),
               "download_ms": 1e3 * float(np.median(dl))}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"gpu": res["gpu"]}), flush=True)
    ba.close()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "batch_plane_ransac.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
