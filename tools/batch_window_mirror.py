"""Times one camera frame of n sequences through pvio_b200_batch_window_mirror_frame against the host-mirrored chain it
replaces: batch_feature_track, the keypoint mirror on the host (oracle/mirror_oracle.py), batch_window_track_frame,
batch_window_edit and batch_window_set_imu.  Both paths run the same rendered sequences (a textured plane under a
turning camera, the windows' states and IMU samples from synthetic.sequence.Run) in their own tracker and window slots;
feature_track is inside both timings.  Prints one line per n with the GPU's name and power limit.

    python tools/batch_window_mirror.py [--n 1 8 132 528] [--frames 8] [--warmup 3]"""
import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cv2  # noqa: E402

from oracle import mirror_oracle  # noqa: E402
from pvio_b200.batch_window import BatchWindows, Edit, Imu, Mirror, TrackFrame  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.feature_track import batch_feature_track, min_capacity  # noqa: E402
from synthetic.sequence import Run  # noqa: E402

KD, H, W = 30.0, 240, 320
CAP = min_capacity(W, H, KD)


def render(seed, n):
    rng = np.random.default_rng(seed)
    tex = cv2.GaussianBlur(rng.integers(0, 256, (3 * H, 3 * W)).astype(np.float32), (0, 0), 1.6)
    tex = cv2.normalize(tex, None, 0, 255, cv2.NORM_MINMAX).astype(np.uint8)
    K = (0.6 * W, 0.6 * W, W / 2 - 0.5, H / 2 + 0.25)
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    T = np.array([[1, 0, -W], [0, 1, -H], [0, 0, 1.0]])
    frames, R = [], np.eye(3)
    for _ in range(n):
        R = cv2.Rodrigues(rng.normal(0, 0.005, 3))[0] @ R
        Hm = Km @ R @ np.linalg.inv(Km) @ T
        Hm[:2, 2] += rng.normal(0, 0.4, 2)
        frames.append(cv2.warpPerspective(tex, Hm, (W, H), flags=cv2.INTER_LINEAR))
    return frames, K


class Seq:
    def __init__(self, slot, tracker, run, frames, K):
        self.slot, self.tracker, self.run, self.frames, self.K = slot, tracker, run, frames, K
        self.f = 0

    def feature(self):
        return dict(slot=self.tracker, frame_id=self.f + 1, image=self.frames[self.f], K=self.K,
                    map_frames=self.f, max_keypoints=CAP)

    def imu(self):
        s, t = self.run.truth.imu_factors[self.f - 1][:2]
        return s, t, self.run.truth.imu_noise

    def seat(self, bw, z, link):
        g = self.run.guess
        bw.reset(self.slot, self.run.w)
        e = Edit(self.slot).frame(np.concatenate([g.q[0], g.p[0], g.v[0], g.bg[0], g.ba[0]]))
        e.new = [(0, q, 1.0) for q in z]
        ids = bw.edit([e])[0]
        self.tk = {k: int(i) for k, i in enumerate(ids)}
        self.nobs = {int(i): 1 for i in ids}                 # the host chain's observation count per track
        self.z, self.next_id, self.N, self.kf, self.skipped, self.last = z, len(ids), 1, True, 0, None
        if link:
            bw.set_keypoints(self.slot, self.tracker, 1, {i: k for k, i in self.tk.items()})


def device_frame(bw, seqs):
    for s in seqs:
        s.f += 1
    batch_feature_track(bw.ba, [s.feature() for s in seqs], keypoint_distance=KD)
    bw.mirror_frame([Mirror(s.slot, s.tracker, *s.imu(), W / 2, H / 2) for s in seqs], CAP)


def host_frame(bw, seqs):
    for s in seqs:
        s.f += 1
    ft = batch_feature_track(bw.ba, [s.feature() for s in seqs], keypoint_distance=KD)
    plans, tfs = [], []
    for s, o in zip(seqs, ft):                               # the host mirror (sliding_window_tracker.cpp:52-73)
        zj = o["keypoints"]
        cont, cand = mirror_oracle.mirror_frame(o["prev_index"], s.tk)
        T = TrackFrame(s.slot, *s.imu(), W / 2, H / 2, s.kf, None if s.kf else s.last, s.skipped)
        for kj, t in cont:
            T.observe(t, zj[kj])
        for ki, kj in cand:
            T.born(s.z[ki], zj[kj])
        plans.append((cont, cand, zj))
        tfs.append(T)
    out = bw.track_frame(tfs)
    edits, imus = [], []
    for s, (cont, cand, zj), r in zip(seqs, plans, out):
        replace = not s.kf
        f = s.N - 1 if replace else s.N
        if replace:                                          # erase_frame: a track seen only there ends with it
            for t in s.tk.values():
                s.nobs[t] -= 1
            cont = [(kj, t) for kj, t in cont if s.nobs[t] > 0]
        for _, t in cont:
            s.nobs[t] += 1
        e = Edit(s.slot, replace).frame(r["state"], False, r["imu_record"])
        e.obs = [(t, f, zj[kj]) for kj, t in cont]
        born = [(ki, kj, t) for t, ((ki, kj), v) in enumerate(zip(cand, r["valid"])) if v]
        for k, (ki, kj, t) in enumerate(born):
            if replace:
                e.new.append((f, zj[kj], r["inv_depth_next"][t]))
            else:
                e.new.append((f - 1, s.z[ki], r["inv_depth"][t]))
                e.obs.append((s.next_id + k, f, zj[kj]))
        samples, t_end, noise = s.imu()
        lst = samples if s.kf else np.concatenate([s.last, samples])
        imus.append(Imu(s.slot, f, lst, t_end, noise))
        edits.append(e)
        s.tk = {kj: t for kj, t in cont}
        s.tk.update({kj: s.next_id + k for k, (ki, kj, t) in enumerate(born)})
        s.nobs.update({s.next_id + k: 1 if replace else 2 for k in range(len(born))})
        s.next_id += len(born)
        s.z, s.N, s.kf, s.skipped, s.last = zj, f + 1, r["keyframe"], r["skipped_frames"], lst
    bw.edit(edits)
    bw.set_imu(imus)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--frames", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    runs = [Run(F=a.frames + 2, N=6, M=40, seed=700 + k) for k in range(8)]
    imgs = [render(700 + k, a.frames + 1) for k in range(8)]
    for n in a.n:
        ba = BundleAdjustor(max_windows=2 * n, max_frames=a.frames + 1, max_landmarks=2048, max_obs=16384)
        try:
            bw = BatchWindows(ba)
            paths = []
            for p, link in ((0, True), (1, False)):
                seqs = [Seq(p * n + i, p * n + i, runs[i % 8], *imgs[i % 8]) for i in range(n)]
                out = batch_feature_track(ba, [s.feature() for s in seqs], keypoint_distance=KD)
                for s, o in zip(seqs, out):
                    s.seat(bw, o["keypoints"], link)
                paths.append(seqs)
            times = [[], []]
            for k in range(a.frames):
                for p, step in ((0, device_frame), (1, host_frame)):
                    ba.lib.pvio_b200_sync(ba.h)
                    t0 = time.perf_counter()
                    step(bw, paths[p])
                    ba.lib.pvio_b200_sync(ba.h)
                    if k >= a.warmup:
                        times[p].append(time.perf_counter() - t0)
            d, h = 1e3 * np.median(times[0]), 1e3 * np.median(times[1])
            print(f"n={n:4d}  mirror_frame path {d:8.2f} ms/frame  host-mirrored chain {h:8.2f} ms/frame  "
                  f"({len(times[0])} frames each, median; feature_track in both)  [{gpu}]")
        finally:
            ba.close()


if __name__ == "__main__":
    main()
