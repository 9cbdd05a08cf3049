"""The per-camera-frame PnP + new-track triangulation of n cfg3 sequences (N = 9, M = 300) on resident slots, two ways,
n = 1, 8, 132, 528:

  (a) pvio_b200_batch_window_localize: one call, the world points gathered on the device
  (b) the host path: batch_window_download, world points rebuilt on the host (Track::get_landmark_point),
      batch_pnp_solve, camera matrices from the solved states and one pvio_b200_triangulate over all sequences

Per path: wall time of one frame (the library calls and, for (b), the host gather between them; the records are built
before the clock starts), median over --reps.  Prints the card (name, power limit) and one JSON line per (path, n).
Usage: python tools/batch_window_localize.py [--n 1 8 132 528] [--reps 20]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from pvio_b200 import _lib, triangulate  # noqa: E402
from pvio_b200.batch_window import Edit, Localize  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from synthetic import so3  # noqa: E402
from synthetic.sequence import BatchPlayer, Run  # noqa: E402

N, M, KINDS, CAP = 9, 300, 4, 360


def setup(runs):
    """n slots after their first solve; the tracks first seen in the newest frame are removed, so they are born in the
    next frame"""
    n = len(runs)
    ba = BundleAdjustor(max_windows=n, max_frames=N, max_landmarks=CAP, max_obs=6000)
    player = BatchPlayer(ba, runs)
    edits = []
    for j, r in enumerate(runs):
        e = Edit(j)
        e.remove = [player.ids[j].pop(l) for l in sorted(player.ids[j]) if r.tracks[l][0][0] == N - 1]
        edits.append(e)
    player.bw.edit(edits)
    player.bw.solve(list(range(n)), max_iterations=4)
    return ba, player


def records(player):
    out = []
    for j, run in enumerate(player.runs):
        f, g = N, run.guess
        s = np.concatenate([g.q[f], g.p[f] + 1e-3, g.v[f], g.bg[f], g.ba[f]])
        L = Localize(j, s, player.rec[j][f - 1])
        obs_l = []
        for l, (fr, zs) in enumerate(run.tracks):
            if f in fr and l in player.ids[j]:
                L.observe(player.ids[j][l], zs[fr.index(f)])
                obs_l.append(l)
            elif f in fr and f - 1 in fr:
                L.born(zs[fr.index(f - 1)], zs[fr.index(f)])
        out.append((L, obs_l))
    return out


def host_path(ba, player, recs):
    """download + host gather + batch_pnp_solve + pvio_b200_triangulate"""
    n = len(recs)
    ds = player.bw.download(list(range(n)), CAP)
    pbs, keep = (_lib.CPnpProblem * n)(), []
    frames = np.zeros((n, 16))
    for j, ((L, obs_l), d) in enumerate(zip(recs, ds)):
        run, w = player.runs[j], player.runs[j].w
        row = {int(t): r for r, t in enumerate(d["ids"])}
        pts, zs = [], []
        for l, (tid, z, _) in zip(obs_l, L.obs):
            fr, kz = run.tracks[l]
            if N - 1 not in fr:
                continue
            r = row[tid]
            a = int(d["anchor"][r])
            qc, pc = run.cam_pose(d["frames"][a, 0:4], d["frames"][a, 4:7])
            za = kz[fr.index(a)]
            pts.append(so3.qrot(qc, np.array([za[0], za[1], 1.0]) / d["inv_depth"][r]) + pc)
            zs.append(z)
        x, z, last = np.array(pts).reshape(-1, 3), np.array(zs).reshape(-1, 2), np.ascontiguousarray(d["frames"][-1])
        keep += [x, z, last]
        pb = pbs[j]
        pb.n_points, pb.use_inertial = len(x), 1
        pb.points, pb.z = _lib.ptr(x), _lib.ptr(z)
        pb.cam_q_cs[:], pb.cam_p_cs[:] = list(w.cam_q_cs), list(w.cam_p_cs)
        pb.imu_q_cs[:], pb.imu_p_cs[:] = list(w.imu_q_cs), list(w.imu_p_cs)
        pb.sqrt_inv_cov[:] = list(np.asarray(w.sqrt_inv_cov, dtype=np.float64).reshape(4))
        pb.cauchy_a = w.cauchy_a
        pb.last_frame, pb.imu_data = _lib.ptr(last), _lib.ptr(L.imu)
        frames[j] = L.state
    opt = _lib.COptions(10, 1e6, 1, 0, 0.0)
    ba._ck(ba.lib.pvio_b200_batch_pnp_solve(ba.h, n, pbs, _lib.ptr(frames), 16, C.byref(opt), None))
    Ps, z, fr = [], [], []
    for j, ((L, _), d) in enumerate(zip(recs, ds)):
        run = player.runs[j]
        for x16 in (d["frames"][-1], frames[j]):
            qc, pc = run.cam_pose(x16[0:4], x16[4:7])
            R = np.array([so3.qrot(so3.qconj(qc), e) for e in np.eye(3)]).T          # q^-1 as a matrix
            Ps.append(np.c_[R, -R @ pc])
        for a, b in L.new:
            z += [a, b]
            fr += [2 * j, 2 * j + 1]
    T = len(fr) // 2
    if T:
        triangulate.triangulate(ba, np.stack(Ps), np.arange(0, 2 * T + 1, 2), np.array(fr), np.array(z))
    return frames


def timed(fn, reps):
    fn()                                              # warm-up: staging growth
    ts = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t)
    return 1e3 * float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    kinds = [Run(F=N + 4, N=N, M=M, seed=801 + i) for i in range(KINDS)]
    for n in a.n:
        ba, player = setup([kinds[i % KINDS] for i in range(n)])
        recs = records(player)
        res = {"a_localize": timed(lambda: player.bw.localize([L for L, _ in recs]), a.reps),
               "b_host": timed(lambda: host_path(ba, player, recs), a.reps)}
        n_obs = sum(len(L.obs) for L, _ in recs) / n
        n_new = sum(len(L.new) for L, _ in recs) / n
        for k, v in res.items():
            print(json.dumps(dict(path=k, n=n, card=card, ms_per_frame=round(v, 3), obs_per_seq=n_obs, new_per_seq=n_new)))
        sys.stdout.flush()
        ba.close()


if __name__ == "__main__":
    main()
