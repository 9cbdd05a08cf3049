"""oracle/mirror_oracle.py against a small Map / Track / Frame model of SlidingWindowTracker::mirror_frame
(sliding_window_tracker.cpp:52-73), track()'s PnP and keyframe lists (pnp.cpp:56-94, :269-277), the non-keyframe
replacement (:115-121) and Map::prune_tracks, on random keypoint chains: thinning that reorders the keypoints, lost
tracks, pruned tracks whose keypoints come back as candidates, and replace_last.

The model follows the resident slot where it departs from the reference's Map: a new track gets an id only once its
triangulation is valid (the reference numbers every created track and prunes the invalid ones, so only the gaps
differ), and a track whose only window observation was the replaced frame ends with it."""
import numpy as np
import pytest

from oracle import mirror_oracle


class Model:
    def __init__(self, rng, n):
        self.rng = rng
        self.next_id = 0
        self.tracks = {}                     # id -> {frame number: keypoint index}
        self.newest = 0                      # frame number of the window's newest frame
        self.kps = {0: n}                    # keypoint count per frame number
        self.newest_kf = True
        self.role, self.given = {}, set()

    def track_of(self, f):
        return {kps[f]: t for t, kps in self.tracks.items() if f in kps}

    def step(self, prev_index, valid_p, prune_p):
        """one camera frame: the reference's mirror_frame, lists, triangulation, replace or append, prune"""
        i, j = self.newest, self.newest + 1
        self.kps[j] = len(prev_index)
        before = self.track_of(i)
        frames_before = {t: set(k) for t, k in self.tracks.items()}
        kj_of = {int(ki): kj for kj, ki in enumerate(prev_index) if ki >= 0}
        born = []                            # mirror_frame: walk frame i, create where empty
        for ki in range(self.kps[i]):
            if ki not in kj_of:
                continue
            if ki in before:
                self.tracks[before[ki]][j] = kj_of[ki]
            else:
                born.append((ki, kj_of[ki]))
        frame_j = self.track_of(j)
        pnp = [(kj, frame_j[kj]) for kj in sorted(frame_j)
               if self.role.get(frame_j[kj], -1) == -1 or frame_j[kj] in self.given]
        frame_i = i if self.newest_kf else max(f for f in self.kps if f < i and self.kf[f])
        par = sorted([kj for kj, t in frame_j.items() if frame_i in self.tracks[t]] +
                     ([kj for _, kj in born] if frame_i == i else []))
        valid = [bool(self.rng.random() < valid_p) for _ in born]
        ends = {t for t in before.values() if frames_before[t] == {i}}
        replace = not self.newest_kf
        if replace:                          # erase frame i; a track observed there only ends with it
            for t in list(self.tracks):
                self.tracks[t].pop(i, None)
                if t in ends or not self.tracks[t]:
                    del self.tracks[t]
        for (ki, kj), v in zip(born, valid):
            if v:
                self.tracks[self.next_id] = {j: kj} if replace else {i: ki, j: kj}
                self.next_id += 1
        return dict(before=before, born=born, valid=valid, pnp=pnp, par=par, frame_i=frame_i, replace=replace,
                    ends=ends, frames_before=frames_before)

    def prune(self, p):
        for t in [t for t in self.tracks if self.rng.random() < p]:
            del self.tracks[t]


def _chain(rng, n_prev, n_new, lost_p, shuffle):
    """prev_index of a new frame: survivors of the previous frame (some lost), in previous-frame order or shuffled, then
    fresh detections (-1)"""
    keep = [ki for ki in range(n_prev) if rng.random() >= lost_p]
    if shuffle:
        rng.shuffle(keep)
    keep = keep[:n_new]
    return np.array(keep + [-1] * (n_new - len(keep)), dtype=np.int32)


@pytest.mark.parametrize("seed", range(12))
def test_oracle_follows_the_model(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(20, 70))
    m = Model(rng, n)
    m.kf = {0: True}
    # seat the window: every keypoint of frame 0 a track
    for k in range(n):
        m.tracks[m.next_id] = {0: k}
        m.next_id += 1
    replaced = 0
    for _ in range(25):
        n_new = int(rng.integers(10, 80))
        prev = _chain(rng, m.kps[m.newest], n_new, rng.uniform(0.0, 0.5), rng.random() < 0.5)
        live = list(m.tracks)
        m.role = {t: int(rng.choice([-1, -1, -2, 0])) for t in live}
        m.given = {t for t in live if m.role[t] != -1 and rng.random() < 0.5}
        track_of = m.track_of(m.newest)
        cont, cand = mirror_oracle.mirror_frame(prev, track_of)
        next_id = m.next_id
        r = m.step(prev, rng.uniform(0.3, 1.0), 0.0)
        assert r["before"] == track_of
        assert [ki for ki, _ in cand] == sorted(ki for ki, _ in cand)          # id order: ki ascending
        assert [kj for kj, _ in cont] == sorted(kj for kj, _ in cont)          # list order: kj ascending
        assert sorted(cand) == sorted(r["born"])
        assert mirror_oracle.pnp_list(cont, m.role, m.given) == r["pnp"]
        pairs, new = mirror_oracle.parallax_pairs(cont, cand, r["frames_before"], r["frame_i"], m.newest)
        assert sorted([kj for kj, _ in pairs] + [kj for _, kj in new]) == r["par"]
        kp, nid = mirror_oracle.append(cont, cand, r["valid"], next_id, r["replace"], r["ends"])
        j = m.newest + 1
        assert kp == m.track_of(j) and nid == m.next_id
        replaced += r["replace"]
        # the new frame becomes the newest: appended, or in place of a non-keyframe
        if r["replace"]:
            del m.kps[m.newest]
            m.kf.pop(m.newest)
        m.newest = j
        m.newest_kf = bool(rng.random() < 0.6)
        m.kf[j] = m.newest_kf
        m.prune(rng.uniform(0.0, 0.2))       # a pruned track's keypoint returns as a candidate next frame
    assert replaced > 0


def test_pruned_track_returns_as_candidate():
    prev = np.array([2, 0, -1, 1], dtype=np.int32)
    cont, cand = mirror_oracle.mirror_frame(prev, {0: 10, 2: 12})      # track 11 at keypoint 1 was pruned
    assert cont == [(0, 12), (1, 10)] and cand == [(1, 3)]
    kp, nid = mirror_oracle.append(cont, cand, [True], 13, False, set())
    assert kp == {0: 12, 1: 10, 3: 13} and nid == 14
    kp, nid = mirror_oracle.append(cont, cand, [False], 13, True, {12})
    assert kp == {1: 10} and nid == 13
