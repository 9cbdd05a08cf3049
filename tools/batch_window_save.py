"""Bytes per sequence and wall times of pvio_b200_batch_window_save / pvio_b200_batch_window_restore for n sequences, each
a cfg3-shaped resident window (N = 9 inertial frames, 300 landmarks, a prior over 8 frames, 50 kept IMU samples per
factor) with a tracker slot of batch_feature_track at 752 x 480 (two frames tracked, so both keypoint buffers are held).
Save and restore name both parts; the restore seats the blobs back in their own slots (a rollback).  Wall times are
medians over --reps calls, each ending in the call's own synchronisation; a separate torch.profiler pass gives the device
time of the pack and unpack kernels.  Prints one line per n with the GPU's name and power limit, read in the same run.

    python tools/batch_window_save.py [--n 1 8 132 528] [--reps 5]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2  # noqa: E402

from pvio_b200 import _lib  # noqa: E402
from pvio_b200.batch_window import BatchWindows, Edit, Imu  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.feature_track import batch_feature_track, min_capacity  # noqa: E402
from synthetic import synth  # noqa: E402

KD, H, W = 20.0, 480, 752
CAP = min_capacity(W, H, KD)


def frames(seed):
    rng = np.random.default_rng(seed)
    tex = cv2.GaussianBlur(rng.integers(0, 256, (H + 64, W + 64)).astype(np.float32), (0, 0), 1.6)
    tex = cv2.normalize(tex, None, 0, 255, cv2.NORM_MINMAX).astype(np.uint8)
    return [np.ascontiguousarray(tex[k:k + H, k:k + W]) for k in (0, 2)]


def seat(bw, slots, w, st, rng):
    """the cfg3 window w at state st in every slot: frames one edit at a time, then the tracks and observations, the
    prior, and 50 kept samples per IMU factor"""
    for s in slots:
        bw.reset(s, w)
    rec = _lib.imu_records(w.imu_dt, w.imu_dq, w.imu_dp, w.imu_dv, w.imu_sqrt_inv_cov, w.imu_dq_dbg, w.imu_dp_dbg,
                           w.imu_dp_dba, w.imu_dv_dbg, w.imu_dv_dba, w.imu_bg0, w.imu_ba0)
    x = np.concatenate([st.q, st.p, st.v, st.bg, st.ba], axis=1)
    for f in range(w.N):
        bw.edit([Edit(s).frame(x[f], False, rec[f - 1] if f > 0 else None) for s in slots])
    new = [(int(w.lm_anchor[m]), w.lm_z_ref[m], float(st.rho[m])) for m in range(w.M)]
    obs = [(m, int(w.obs_frame[k]), w.obs_z[k]) for m in range(w.M)
           for k in range(w.lm_obs_begin[m], w.lm_obs_begin[m + 1] if m + 1 < w.M else w.K)]
    edits = []
    for s in slots:
        e = Edit(s)
        e.new, e.obs = new, obs
        edits.append(e)
    bw.edit(edits)
    x0 = np.concatenate([w.prior_q0, w.prior_p0, w.prior_v0, w.prior_bg0, w.prior_ba0], axis=1)
    for s in slots:
        bw.set_prior(s, w.prior_S, w.prior_e, x0)
    noise = [np.eye(3) * 1e-4] * 4
    smp = [np.column_stack([np.linspace(0.25 * f, 0.25 * f + 0.245, 50), rng.normal(size=(50, 6))]) for f in range(w.N)]
    for f in range(1, w.N):
        bw.set_imu([Imu(s, f, smp[f - 1], 0.25 * f, noise) for s in slots])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    w, st, _ = synth.make_cfg3(N=9, M=300)
    imgs = frames(5)
    K = (460.0, 460.0, W / 2 - 0.5, H / 2 + 0.5)
    for n in a.n:
        ba = BundleAdjustor(max_windows=n, max_frames=9, max_landmarks=512, max_obs=4096)
        try:
            bw = BatchWindows(ba)
            slots, trk = list(range(n)), list(range(n))
            seat(bw, slots, w, st, np.random.default_rng(1))
            for c in range(0, n, 132):                       # two frames per tracker slot, in calls of at most 132
                for k in (0, 1):
                    batch_feature_track(ba, [dict(slot=t, frame_id=k + 1, image=imgs[k], K=K, map_frames=k,
                                                  max_keypoints=CAP) for t in trk[c:c + 132]], keypoint_distance=KD)
            blobs = bw.save(slots, trk)
            ts, tr = [], []
            for _ in range(a.reps + 1):
                t0 = time.perf_counter()
                blobs = bw.save(slots, trk)
                t1 = time.perf_counter()
                bw.restore(slots, blobs, trk)
                t2 = time.perf_counter()
                ts.append(t1 - t0)
                tr.append(t2 - t1)
            assert bw.save(slots, trk) == blobs
            kern = {}
            try:
                import torch
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    bw.restore(slots, bw.save(slots, trk), trk)
                    torch.cuda.synchronize()
                for ev in prof.key_averages():
                    if "bw_save_kernel" in ev.key or "bw_restore_kernel" in ev.key:
                        kern["save" if "save" in ev.key else "restore"] = ev.device_time_total / max(ev.count, 1) / 1e3
            except Exception as e:                            # the profiler pass is optional; the wall times are not
                print(f"  (no profiler pass: {e})")
            per = np.mean([len(b) for b in blobs])
            ks = " ".join(f"{k} kernel {v:.3f} ms" for k, v in sorted(kern.items())) or "kernels not profiled"
            print(f"n={n:4d}  {per / 1e6:.3f} MB per sequence  save {1e3 * np.median(ts[1:]):8.2f} ms  "
                  f"restore {1e3 * np.median(tr[1:]):8.2f} ms  (wall, median of {a.reps}; size query included in save)"
                  f"  {ks}  [{gpu}]")
        finally:
            ba.close()


if __name__ == "__main__":
    main()
