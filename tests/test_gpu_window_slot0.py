"""The single resident window (pvio_b200_window_*) is slot 0 of the resident batched windows (pvio_b200_batch_window_*):
a sequence played through either gives the same window, and window_* keeps its own contract (ids, gone tracks, calls
before a reset) under the slot rules (slot limits, a rejected call changes nothing)."""
import numpy as np
import pytest

from pvio_b200 import _lib
from pvio_b200 import resident
from pvio_b200.batch_window import BatchWindows, Edit
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.resident import ResidentWindow
from synthetic import synth
from synthetic.sequence import ResidentPlayer, Run

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"


class Slot0Window:
    """ResidentWindow's calls (those ResidentPlayer makes) as pvio_b200_batch_window_* calls on slot 0"""

    def __init__(self, ba, win):
        self.bw = BatchWindows(ba)
        self.bw.reset(0, win)

    def append_frame(self, state16, fixed=False, imu_record=None):
        self.bw.edit([Edit(0).frame(state16, fixed, imu_record)])

    def add_tracks(self, frames, z, inv_depth):
        e = Edit(0)
        e.new = list(zip(frames, z, inv_depth))
        return self.bw.edit([e])[0]

    def add_observations(self, tracks, frames, z):
        e = Edit(0)
        e.obs = list(zip(tracks, frames, z))
        self.bw.edit([e])

    def set_prior(self, S, e, state0):
        self.bw.set_prior(0, S, e, state0)

    def solve(self, max_iterations=10):
        return self.bw.solve([0], max_iterations=max_iterations, postpass=False)[0]

    def drop_victim(self):
        self.bw.drop_victim([0])


def _handle():
    return BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=320, max_obs=2000)


def _same(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def test_window_calls_follow_batched_slot_0(monkeypatch):
    """The cfg3 ResidentPlayer through window_* on one handle and through batch_window_* slot 0 on another, 12 keyframes:
    equal iteration counts, terminations, track ids, anchors and observation counts; costs, radii, states and inverse
    depths within 1e-7.  Not bit for bit: the single-window solve of an inertial window sums fp64 terms with atomics, so
    two handles running the same calls on the same window already differ by about 1e-9 after a few keyframes.  Gone
    tracks read back as anchor -1, 0 observations and an unwritten inverse depth."""
    run = Run(F=20, N=6, M=260, seed=700)
    a, b = _handle(), _handle()
    pa = ResidentPlayer(a, run)
    monkeypatch.setattr(resident, "ResidentWindow", Slot0Window)
    pb = ResidentPlayer(b, run)
    assert isinstance(pa.rw, ResidentWindow) and isinstance(pb.rw, Slot0Window)
    gone, worst = 0, 0.0
    for k in range(12):
        sa, sb = pa.solve(6), pb.solve(6)
        for f in ("iterations", "accepted_steps", "termination", "usable"):
            assert sa[f] == sb[f], (k, f)
        for f in ("initial_cost", "final_cost", "final_radius", "final_mu"):
            worst = max(worst, abs(sa[f] - sb[f]) / max(abs(sb[f]), 1e-300))
        assert pa.ids == pb.ids, k
        ids = sorted(pa.ids.values())
        fr, rho, an, cnt = pa.rw.get(ids)
        d = pb.rw.bw.download([0], 320)[0]
        row = {int(i): r for r, i in enumerate(d["ids"])}
        live = np.array([i in row for i in ids])
        r = [row[i] for i in ids if i in row]
        assert live.sum() == len(d["ids"]), k
        assert np.array_equal(an[live], d["anchor"][r]) and np.array_equal(cnt[live], d["n_obs"][r]), k
        assert np.all(an[~live] == -1) and np.all(cnt[~live] == 0) and np.all(rho[~live] == 0.0), k
        worst = max(worst, np.abs(fr - d["frames"]).max(), np.max(np.abs(rho[live] - d["inv_depth"][r]) / np.abs(d["inv_depth"][r])))
        gone += int((~live).sum())
        pa.shift(k)
        pb.shift(k)
    print("window_* vs batch_window_* slot 0: worst summary / state / inverse-depth difference", worst)
    assert gone > 0 and worst < 1e-7
    a.close()
    b.close()


def test_window_contract_and_slot_rules():
    run = Run(F=12, N=6, M=120, seed=730)
    ba = _handle()
    player = ResidentPlayer(ba, run)
    for k in range(3):
        player.solve(4)
        player.shift(k)
    rw, bw = player.rw, BatchWindows(ba)
    t = int(rw.add_tracks([0], [np.array([0.01, 0.02])], [0.5])[0])      # a one-observation track
    ids = sorted(player.ids.values()) + [t]
    nxt = t + 1
    snap = lambda: [x.copy() for x in rw.get(ids)]
    s0 = snap()
    cnt = s0[3]
    live = [i for i, c in zip(ids, cnt) if c > 0]
    gone = [i for i, c in zip(ids, cnt) if c == 0]
    assert gone and len(live) > 2
    d = bw.download([0], 320)[0]                          # window_* and batch_window_* on slot 0: the same window
    assert np.array_equal(d["frames"], s0[0]) and [int(i) for i in d["ids"]] == live

    l0 = ba.kernel_launches                               # removing a gone track: 0, and no edit runs
    rw.remove_track(gone[0])
    assert ba.kernel_launches == l0 and _same(snap(), s0)

    n_live = len(live)
    rejected = [
        lambda: rw.remove_track(nxt),                     # ids outside [0, next id)
        lambda: rw.remove_track(-1),
        lambda: rw.get([nxt]),
        lambda: rw.get([-1]),
        lambda: rw.add_tracks([0, 9, 1], np.zeros((3, 2)), [1.0] * 3),    # the second starts outside the window
        lambda: rw.add_observations([t, t], [2, 2], np.zeros((2, 2))),    # the second is out of frame order
        lambda: rw.add_tracks([1] * (320 - n_live + 1), np.zeros((320 - n_live + 1, 2)), [1.0] * (320 - n_live + 1)),
        lambda: rw.append_frame(np.zeros(16), False, None),              # an inertial window needs the IMU record
    ]
    for i, call in enumerate(rejected):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
        assert _same(snap(), s0), i
    # live one-observation tracks count toward max_landmarks; the rejected calls used no ids
    got = rw.add_tracks([1] * (320 - n_live), np.zeros((320 - n_live, 2)), [1.0] * (320 - n_live))
    assert int(got[0]) == nxt
    with pytest.raises(PvioB200Error, match=EINVAL):
        rw.add_tracks([1], np.zeros((1, 2)), [1.0])

    rw.remove_track(t)                                    # a removed track is gone
    _, rho, an, cnt = rw.get([t])
    assert an[0] == -1 and cnt[0] == 0 and rho[0] == 0.0

    w, st, _ = synth.make_cfg2(N=5, M=40, seed=7)         # a call that packs slot 0 ends the resident window
    ba.solve(w, st, max_iterations=2)
    for call in (lambda: rw.solve(2), lambda: rw.get([]), lambda: rw.drop_victim(), lambda: bw.download([0], 320)):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
    again = ResidentWindow(ba, run.w)                     # until the next reset
    assert len(again.get()[0]) == 0

    fresh = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=32, max_obs=64)
    before = ResidentWindow.__new__(ResidentWindow)       # every call before a reset
    before.ba, before.lib, before.h = fresh, fresh.lib, fresh.h
    for call in (lambda: before.append_frame(np.zeros(16)), lambda: before.add_tracks([0], np.zeros((1, 2)), [1.0]),
                 lambda: before.add_observations([0], [0], np.zeros((1, 2))), lambda: before.remove_track(0),
                 lambda: before.set_prior(np.eye(15), np.zeros(15), np.zeros((1, 16))), lambda: before.solve(2),
                 lambda: before.drop_victim(), lambda: before.get()):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
    fresh.close()
    ba.close()


def test_visual_window_rejects_a_prior_and_more_than_96_chunks():
    ba = BundleAdjustor(max_windows=1, max_frames=16, max_landmarks=3600, max_obs=3500)
    wv, _, _ = synth.make_cfg2(N=5, M=10, seed=950)
    rw = ResidentWindow(ba, wv)
    for f in range(16):
        rw.append_frame(np.concatenate([[0, 0, 0, 1], [0.1 * f, 0, 0], np.zeros(9)]), f < 2)
    ids = rw.add_tracks([a for a in range(15) for _ in range(224)],
                        [np.array([0.01 * (i % 50), 0.02]) for _ in range(15) for i in range(224)], [0.2] * 15 * 224)
    ok = [(int(ids[a * 224 + i]), a + 1) for a in range(15) for i in range(192)]        # 15 anchors x 6 chunks
    rw.add_observations([o[0] for o in ok], [o[1] for o in ok], np.zeros((len(ok), 2)))
    snap = lambda: [x.copy() for x in rw.get(ids)]
    s0 = snap()
    more = [(int(ids[a * 224 + i]), a + 1) for a in range(15) for i in range(192, 224)]  # 105 chunks
    for call in (lambda: rw.add_observations([o[0] for o in more], [o[1] for o in more], np.zeros((len(more), 2))),
                 lambda: rw.set_prior(np.eye(15), np.zeros(15), np.zeros((1, 16)))):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
        assert _same(snap(), s0)
    ba.close()
