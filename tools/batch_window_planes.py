"""One keyframe cycle of n sequences with planes (N = 9, M = 300 landmarks, 2 planes x 40 tracks; the roles of
synthetic.sequence.Run.role switch along the run) through two paths, n = 1, 8, 132, 528:

  (a) resident batched slots: batch_window_solve + download + drop_victim + edit of the next frame + set_planes
  (b) the re-pack path of INTEGRATION §2c with planes: gather every window from a host model (Chain.window, plane tables
      included), batch_set_window x n, batch_upload, batch_solve, batch_download_state, batch_marginalize

Per path: wall time per keyframe inside the library calls (the Python that builds the records or gathers the windows is
reported separately), device time (CUDA events on the handle's stream around the cycle) and, in a separate pass under
torch.profiler, the host -> device bytes per keyframe.  Prints the card (name, power limit) and one JSON line per
(path, n).  Usage: python tools/batch_window_planes.py [--n 1 8 132 528] [--cycles 3]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from batch_window import Clock, h2d_bytes  # noqa: E402
from pvio_b200.bundle_adjustor import BundleAdjustor  # noqa: E402
from pvio_b200.window import State  # noqa: E402
from synthetic.sequence import BatchPlayer, Chain, Run  # noqa: E402

N, M, PLANES, KINDS = 9, 300, 2, 8
CAP = M + PLANES * 40 + 40          # live tracks per window: landmarks, plane tracks, one-observation tracks


def path_a(runs, n, cycles):
    ba = BundleAdjustor(max_windows=n, max_frames=N, max_landmarks=CAP, max_obs=6000)
    player = BatchPlayer(ba, runs)
    clock = Clock()
    clock.wrap(player.bw, ("solve", "download", "drop_victim", "edit", "set_planes"))
    js = list(range(n))

    def cycle():
        player.bw.solve(js, max_iterations=10)
        player.refresh(js, CAP)
        player.advance(js, nonkey=False)               # drop, the next frame, then set_planes of the new keyframe

    cycle()                                            # warm-up: allocations, graphs
    wall = dev = total = 0.0
    for _ in range(cycles):
        clock.s = 0.0
        t = time.perf_counter()
        ba.timer_start()
        cycle()
        dev += ba.timer_stop()
        total += time.perf_counter() - t
        wall += clock.s
    b = h2d_bytes(cycle)
    ba.close()
    return dict(wall_ms=1e3 * wall / cycles, device_ms=dev / cycles, host_python_ms=1e3 * (total - wall) / cycles,
                h2d_bytes=b)


def path_b(runs, n, cycles):
    ba = BundleAdjustor(max_windows=n, max_frames=N, max_landmarks=CAP, max_obs=6000)
    chains = [Chain(r) for r in runs]
    state = dict(k=0, resident=[False] * n)

    def cycle(clock):
        k = state["k"]
        t = time.perf_counter()
        views = [c.window(k) for c in chains]          # the host gather, plane tables included
        gather = time.perf_counter() - t
        t = time.perf_counter()
        for j, (w, st, _) in enumerate(views):
            ba.batch_set(j, w, st, resident_prior=state["resident"][j])
        ba.batch_upload(n)
        ba.batch_solve(n, max_iterations=10)
        frames, rho, _ = ba.batch_download_state(n, N, CAP)
        ba.batch_marginalize(n)
        clock[0] += time.perf_counter() - t
        clock[1] += gather
        for j, (c, (w, _, ids)) in enumerate(zip(chains, views)):
            fr = frames[j, :w.N]
            c.store(k, State(fr[:, 0:4], fr[:, 4:7], fr[:, 7:10], fr[:, 10:13], fr[:, 13:16], rho[j, :w.M].copy()), ids)
            d = 15 * (N - 1)
            c.prior = dict(frames=list(range(k + 1, k + N)), S=np.zeros((d, d)), e=np.zeros(d), x0=np.zeros((N - 1, 16)))
            state["resident"][j] = True
        state["k"] += 1

    cycle([0.0, 0.0])
    wall = dev = gather = 0.0
    for _ in range(cycles):
        clock = [0.0, 0.0]
        ba.timer_start()
        cycle(clock)
        dev += ba.timer_stop()
        wall += clock[0]
        gather += clock[1]
    b = h2d_bytes(lambda: cycle([0.0, 0.0]))
    ba.close()
    return dict(wall_ms=1e3 * wall / cycles, device_ms=dev / cycles, gather_ms=1e3 * gather / cycles, h2d_bytes=b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, nargs="+", default=[1, 8, 132, 528])
    ap.add_argument("--cycles", type=int, default=3)
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"
    kinds = [Run(F=N + 2 * a.cycles + 8, N=N, M=M, seed=795 + i, planes=PLANES) for i in range(KINDS)]
    for n in a.n:
        runs = [kinds[i % KINDS] for i in range(n)]
        res = {"a_resident": path_a(runs, n, a.cycles), "b_repack": path_b(runs, n, a.cycles)}
        for k, v in res.items():
            print(json.dumps(dict(path=k, n=n, card=card, **{x: round(y, 3) if isinstance(y, float) else y for x, y in v.items()})))
        sys.stdout.flush()


if __name__ == "__main__":
    main()
