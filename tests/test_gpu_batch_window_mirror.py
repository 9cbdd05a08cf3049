"""pvio_b200_batch_window_set_keypoints / pvio_b200_batch_window_mirror_frame: each sequence's new camera frame taken
straight from its tracker slot.  Frames are a textured plane rendered as test_gpu_batch_feature_track renders it; the
windows' states and IMU samples come from a synthetic.sequence.Run.  Checked per frame:
  - the mirror bit for bit against oracle/mirror_oracle.py on batch_feature_track's outputs and a slot download taken
    before the call (kp_track, counts, the PnP list through the counts);
  - the track step against track_frame on the same slot with the oracle's lists, before the call;
  - the append bit for bit against twin slots that receive the call's results as ordinary edit + set_imu calls;
  - the link across prune, set_planes, drop_victim and forced non-keyframes."""
import functools

import numpy as np
import pytest

from oracle import mirror_oracle
from pvio_b200._lib import EINVAL
from oracle import tracker_oracle
from pvio_b200 import imu
from pvio_b200.batch_window import BatchWindows, Edit, Imu, Mirror, PlaneRansac, Planes, TrackFrame
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200.feature_track import batch_feature_track, min_capacity
from synthetic.sequence import Run
from test_gpu_batch_feature_track import render

pytestmark = pytest.mark.gpu
KD = 30.0
SHAPE = (240, 320)
CX, CY = 160.0, 120.0
TS = 100                                     # tracker slot of sequence j: TS + j
CAP = min_capacity(SHAPE[1], SHAPE[0], KD)
SEQ_TOL = 2e-6


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _state16(run, f):
    g = run.guess
    return np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]])


@functools.lru_cache(maxsize=None)
def _run(F, seed):
    return Run(F=F, N=6, M=40, seed=seed), render(seed, F, SHAPE)


class Seq:
    """one sequence: window slot, twin slot, tracker slot, its frames, IMU and the host's view of the link"""

    def __init__(self, j, slot, twin, F, seed):
        self.j, self.slot, self.twin, self.tracker = j, slot, twin, TS + j
        self.run, (self.frames, self.qs, self.K) = _run(F, seed)
        self.f, self.start = 0, 0
        self.roles, self.given = {}, {}

    def feature(self):
        return dict(slot=self.tracker, frame_id=self.f + 1, image=self.frames[self.f], K=self.K,
                    map_frames=min(self.f - self.start, 20), max_keypoints=CAP)

    def imu(self):
        s, t = self.run.truth.imu_factors[self.f - 1][:2]
        return s, t, self.run.truth.imu_noise

    def seat(self, bw, z):
        """a one-frame window in the slot and its twin with a track per keypoint of the tracker's newest frame, linked"""
        self.z = z
        for slot in (self.slot, self.twin):
            bw.reset(slot, self.run.w)
            e = Edit(slot).frame(_state16(self.run, self.f))
            e.new = [(0, q, 1.0) for q in z]
            ids = bw.edit([e])[0]
        self.tk = {k: int(i) for k, i in enumerate(ids)}      # keypoint of the newest frame -> track id
        self.next_id, self.N, self.newest_kf, self.skipped, self.last = len(ids), 1, True, 0, None
        self.wf = [self.f]                                     # the tracker frame of each window frame
        self.zhist = {int(i): {self.f: z[k]} for k, i in enumerate(ids)}   # track -> tracker frame -> keypoint
        self.roles, self.given = {}, {}
        bw.set_keypoints(self.slot, self.tracker, self.f + 1, {i: k for k, i in self.tk.items()})


def _start(bw, seqs):
    out = batch_feature_track(bw.ba, [s.feature() for s in seqs], keypoint_distance=KD)
    for s, o in zip(seqs, out):
        s.seat(bw, o["keypoints"])


def _advance(bw, seqs):
    for s in seqs:
        s.f += 1
    return batch_feature_track(bw.ba, [s.feature() for s in seqs], keypoint_distance=KD)


def _ends(d, N):
    return {int(i) for i, a, c in zip(d["ids"], d["anchor"], d["n_obs"]) if c == 1 and a == N - 1}


def _probe(bw, slots):
    """what the slots hold, as exactly as the calls expose it: download, IMU records, and every track with two or more
    observations triangulated over all its window keypoints (Plane::update_parameter's points: these read each stored
    keypoint and frame mask)"""
    ds = bw.download(slots, 4096)
    recs = bw.imu_records(slots)
    rf = bw.plane_ransac([PlaneRansac(s, PlaneRansac.REFIT, d["ids"][d["n_obs"] >= 2]) for s, d in zip(slots, ds)])
    return [(d, r, o["points"], o["used"]) for d, r, o in zip(ds, recs, rf)]


def _bit_equal(a, b):
    (da, ra, pa, ua), (db, rb, pb, ub) = a, b
    for k in ("ids", "anchor", "n_obs"):
        assert np.array_equal(da[k], db[k]), k
    for k in ("frames", "inv_depth"):
        assert np.array_equal(_bits(da[k]), _bits(db[k])), k
    assert np.array_equal(_bits(ra), _bits(rb))
    assert np.array_equal(_bits(pa), _bits(pb)) and np.array_equal(ua, ub)


def _kf_oracle(ba, s, d, cont, cand, zj):
    """tracker_oracle.keyframe_check on mirror_oracle.parallax_pairs from the host's keypoint history, with the step-1
    record pvio_b200_preintegrate gives at the newest frame's downloaded biases"""
    samples, t_end, noise = s.imu()
    x = d["frames"][-1]
    rec1 = imu.preintegrate(ba, [(samples, t_end, x[10:13].copy(), x[13:16].copy())], list(noise))[0]
    fi = s.wf[-1] if s.newest_kf else s.wf[-2]
    pairs, new = mirror_oracle.parallax_pairs(cont, cand, {t: set(h) for t, h in s.zhist.items()}, fi, s.wf[-1])
    zi = [s.zhist[t][fi] for _, t in pairs] + [s.z[ki] for ki, _ in new]
    zjs = [zj[kj] for kj, _ in pairs] + [zj[kj] for _, kj in new]
    w = s.run.w
    return tracker_oracle.keyframe_check(zi, zjs, rec1[1:5], w.cam_q_cs, w.imu_q_cs, w.K_fx, w.K_fy, CX, CY, s.skipped)


def _step(bw, seqs, ft, host=False, twin=True, bystanders=()):
    """one mirror_frame call over `seqs` after batch_feature_track gave `ft`.  The slot's results are checked against
    the oracle (kp_track, counts, the keyframe check), against track_frame run with the oracle's lists (on the slot
    before the call, or, host: on the twin, the host-mirrored chain), and the twin then takes the frame as an ordinary
    edit + set_imu: fed the call's outputs and the slot's inverse depths (bit for bit), or, host, track_frame's own."""
    ba = bw.ba
    pre = bw.download([s.slot for s in seqs], 4096)
    plans, recs, tfs = [], [], []
    for s, o, d in zip(seqs, ft, pre):
        prev, zj = o["prev_index"], o["keypoints"]
        cont, cand = mirror_oracle.mirror_frame(prev, s.tk)
        samples, t_end, noise = s.imu()
        pnp = mirror_oracle.pnp_list(cont, s.roles, s.given)
        plans.append((cont, cand, pnp, _ends(d, s.N), prev, zj, _kf_oracle(ba, s, d, cont, cand, zj)))
        recs.append(Mirror(s.slot, s.tracker, samples, t_end, noise, CX, CY, True, s.given))
        T = TrackFrame(s.twin if host else s.slot, samples, t_end, noise, CX, CY, s.newest_kf,
                       None if s.newest_kf else s.last, s.skipped)
        for kj, t in pnp:
            T.observe(t, zj[kj], s.given.get(t))
        for ki, kj in cand:
            T.born(s.z[ki], zj[kj])
        tfs.append(T)
    ref = bw.track_frame(tfs)
    unnamed = [s.twin for s in seqs] + list(bystanders)
    before = _probe(bw, unnamed)
    out = bw.mirror_frame(recs, CAP)
    for a, b in zip(before, _probe(bw, unnamed)):                 # slots not named keep everything
        _bit_equal(a, b)
    post = {s.slot: d for s, d in zip(seqs, bw.download([s.slot for s in seqs], 4096))}
    edits = []
    for s, o, r, (cont, cand, pnp, ends, prev, zj, kfo) in zip(seqs, out, ref, plans):
        m = len(prev)
        kp = o["kp_track"]
        assert np.all(kp[m:] == -7)
        valid = [bool(kp[kj] >= 0) for _, kj in cand]
        replace = not s.newest_kf
        want, nid = mirror_oracle.append(cont, cand, valid, s.next_id, replace, ends)
        assert {kj: int(t) for kj, t in enumerate(kp[:m]) if t >= 0} == want
        assert list(o["counts"]) == [len(cont), len(pnp), len(cand), sum(valid)]
        kf, par, npar, sk = kfo                                  # every continued track and candidate counts
        assert (o["keyframe"], o["n_parallax"], o["skipped_frames"]) == (kf, npar, sk)
        assert (np.isnan(o["parallax"]) and np.isnan(par)) or abs(o["parallax"] - par) <= 1e-12 * par
        sm, rs = o["summary"], r["summary"]
        assert sm["iterations"] == rs["iterations"]
        if len(pnp) == len(cont):            # no plane track left out: track_frame's parallax list is the same
            assert o["keyframe"] == r["keyframe"] and o["n_parallax"] == r["n_parallax"]
        assert list(r["valid"]) == valid
        tol = SEQ_TOL if host else 1e-12 * max(np.abs(r["state"]).max(), 1.0)
        assert np.abs(o["state"] - r["state"]).max() <= tol
        rho = dict(zip(post[s.slot]["ids"].tolist(), post[s.slot]["inv_depth"]))
        born = [(ki, kj, t) for t, ((ki, kj), v) in enumerate(zip(cand, valid)) if v]
        for k, (ki, kj, t) in enumerate(born):  # the inverse depths the slot took, against track_frame's
            want_rho = r["inv_depth_next"][t] if replace else r["inv_depth"][t]
            assert abs(rho[s.next_id + k] - want_rho) <= (1e-6 if host else 1e-9) * abs(want_rho)
        # the twin: the same frame as an ordinary edit + set_imu
        samples, t_end, noise = s.imu()
        lst = samples if s.newest_kf else np.concatenate([s.last, samples])
        fnew = s.N - 1 if replace else s.N
        src = r if host else o
        e = Edit(s.twin, replace).frame(src["state"], False, src["imu_record"])
        for kj, t in cont:
            if want.get(kj) == t:
                e.obs.append((t, fnew, zj[kj]))
        for k, (ki, kj, t) in enumerate(born):
            i = s.next_id + k
            x = (r["inv_depth_next"] if replace else r["inv_depth"])[t] if host else rho[i]
            e.new.append((fnew, zj[kj], x) if replace else (fnew - 1, s.z[ki], x))
            if not replace:
                e.obs.append((i, fnew, zj[kj]))
        edits.append(e)
        # the host's view of the slot after the frame
        if replace:
            s.wf[-1] = s.f
        else:
            s.wf.append(s.f)
        for kj, t in want.items():
            s.zhist.setdefault(t, {})[s.f] = zj[kj]
        for k, (ki, kj, t) in enumerate(born):
            if not replace:
                s.zhist[s.next_id + k][s.wf[-2]] = s.z[ki]
        s.tk = {kj: t for kj, t in want.items()}
        s.z, s.N = zj, fnew + 1
        s.newest_kf, s.skipped, s.last = o["keyframe"], o["skipped_frames"], lst
        s.pending = (nid, fnew, lst, t_end, noise)
    if twin:
        got = bw.edit(edits)
        imus = []
        for s, g in zip(seqs, got):
            nid, fnew, lst, t_end, noise = s.pending
            assert list(g) == list(range(s.next_id, nid))
            imus.append(Imu(s.twin, fnew, lst, t_end, noise))
        bw.set_imu(imus)
    for s in seqs:
        s.next_id = s.pending[0]
    if twin:
        for s, (a, b) in zip(seqs, zip(_probe(bw, [s.slot for s in seqs]), _probe(bw, [s.twin for s in seqs]))):
            if host:
                (da, _, _, _), (db, _, _, _) = a, b
                for k in ("ids", "anchor", "n_obs"):
                    assert np.array_equal(da[k], db[k]), k
                assert np.abs(da["frames"] - db["frames"]).max() < SEQ_TOL
            else:
                _bit_equal(a, b)
    return out


def _drop(bw, seqs, full):
    bw.drop_victim([s.slot for s in full] + [s.twin for s in full])
    for s in full:
        s.N -= 1
        s.wf.pop(0)


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=4096, max_obs=16384)
    yield b
    b.close()


def test_sequences_follow_oracle_track_frame_and_twin(ba):
    """4 sequences over 14 frames: forced non-keyframes, a prune, plane roles with and without given points, drops"""
    bw = BatchWindows(ba)
    seqs = [Seq(j, j, 4 + j, 16, 900 + j) for j in range(4)]
    _start(bw, seqs)
    replaced = dropped = pruned_back = 0
    for k in range(14):
        ft = _advance(bw, seqs)
        if k == 5:                           # prune: the pruned tracks' keypoints come back as candidates
            pruned = {}
            for s in seqs:
                ids = sorted(set(s.tk.values()))[::7][:6]
                pruned[s.j] = {ki for ki, t in s.tk.items() if t in ids}
                for slot in (s.slot, s.twin):
                    e = Edit(slot)
                    e.remove = ids
                    bw.edit([e])
                s.tk = {ki: t for ki, t in s.tk.items() if t not in ids}
                s.roles = {t: r for t, r in s.roles.items() if t not in ids}
                s.given = {t: p for t, p in s.given.items() if t not in ids}
        if k == 3:                           # plane roles: half of them with a given point
            for s in seqs:
                tr = sorted(set(s.tk.values()))[1::5][:8]
                for slot in (s.slot, s.twin):
                    p = Planes(slot)
                    for t in tr:
                        p.role(t, -2)
                    bw.set_planes([p])
                s.roles = {t: -2 for t in tr}
                s.given = {t: np.array([0.1 * t, 0.2, 3.0]) for t in tr[::2]}
        replaced += sum(not s.newest_kf for s in seqs)
        _step(bw, seqs, ft)
        if k == 5:                           # the oracle's candidates include them, and the call agreed
            for s in seqs:
                pruned_back += sum(1 for ki in ft[s.j]["prev_index"] if ki in pruned[s.j])
        full = [s for s in seqs if s.newest_kf and s.N >= 6]
        if full:
            _drop(bw, seqs, full)
            for s in full:
                _bit_equal(*_probe(bw, [s.slot, s.twin]))
            dropped += len(full)
        for s in seqs:                       # force a non-keyframe now and then: the next frame replaces it
            if k % 3 == 1 and s.newest_kf and s not in full and s.N >= 2:
                s.newest_kf = False
                bw.set_keypoints(s.slot, s.tracker, s.f + 1, {t: kj for kj, t in s.tk.items()}, False, s.skipped)
    print(f"replaced frames {replaced}, drops {dropped}, pruned keypoints back as candidates {pruned_back}")
    assert replaced > 0 and dropped > 0 and pruned_back > 0
    # a solve keeps the link: the next frame still mirrors as the oracle says
    bw.solve([s.slot for s in seqs], max_iterations=2)
    ft = _advance(bw, seqs)
    pre = bw.download([s.slot for s in seqs], 4096)
    recs = [Mirror(s.slot, s.tracker, *s.imu(), CX, CY, True, s.given) for s in seqs]
    for s, o, f, d in zip(seqs, bw.mirror_frame(recs, CAP), ft, pre):
        cont, cand = mirror_oracle.mirror_frame(f["prev_index"], s.tk)
        kp = o["kp_track"][:len(f["prev_index"])]
        valid = [bool(kp[kj] >= 0) for _, kj in cand]
        want, _ = mirror_oracle.append(cont, cand, valid, s.next_id, not s.newest_kf, _ends(d, s.N))
        assert {kj: int(t) for kj, t in enumerate(kp) if t >= 0} == want
        assert list(o["counts"][:3]) == [len(cont), len(mirror_oracle.pnp_list(cont, s.roles, s.given)), len(cand)]


def test_rejections_change_nothing(ba):
    bw = BatchWindows(ba)
    seqs = [Seq(j, j, 4 + j, 6, 950 + j) for j in range(2)]
    _start(bw, seqs)
    ft = _advance(bw, seqs)
    del ft

    def call(recs, cap=CAP):
        r, sms, out, keep = BatchWindows.mirror_records(recs, cap)
        before = bw.download([0, 1, 4, 5], 4096)
        rc = ba.lib.pvio_b200_batch_window_mirror_frame(ba.h, len(recs), r, None)
        assert rc == EINVAL
        for o in out:
            assert np.all(o["kp_track"] == -7) and np.all(o["state"] == 0.0)
        after = bw.download([0, 1, 4, 5], 4096)
        for a, b in zip(before, after):
            for k in a:
                assert np.array_equal(_bits(a[k]) if a[k].dtype == np.float64 else a[k],
                                      _bits(b[k]) if b[k].dtype == np.float64 else b[k])

    def rec(s, **kw):
        samples, t_end, noise = s.imu()
        m = Mirror(s.slot, s.tracker, samples, t_end, noise, CX, CY, True, kw.pop("given", None))
        for k, v in kw.items():
            setattr(m, k, v)
        return m

    a, b = seqs
    call([rec(b, tracker_slot=a.tracker)])                            # not the tracker slot of the link
    bw.set_keypoints(a.twin, a.tracker, a.f, {})                      # two slots linked to one tracker slot
    call([rec(a), rec(a, slot=a.twin)])                               # a tracker slot named twice
    bw.reset(a.twin, a.run.w)
    bw.edit([Edit(a.twin).frame(_state16(a.run, 0))])
    call([rec(a, slot=4)])                                            # a slot without a link
    call([rec(a)], cap=3)                                             # max_keypoints below the keypoint count
    call([rec(a, samples=np.zeros((0, 7)))])                          # no samples
    call([rec(a, given={10 ** 6: np.zeros(3)})])                      # unknown given track
    call([rec(a, given={0: np.array([np.nan, 0, 0])})])               # non-finite given point
    call([rec(a), rec(a)])                                            # a slot named twice
    # the tracker moved on without a mirror: its previous frame is not the slot's newest
    s = seqs[1]
    s.f += 1
    batch_feature_track(ba, [s.feature()], keypoint_distance=KD)
    call([rec(s)])
    # a restarted tracker slot (map_frames == 0) whose frame ids repeat the linked sequence's: the link names the old
    # sequence, so the slot stays rejected until set_keypoints links it again
    a.f, a.start = 0, 0
    batch_feature_track(ba, [a.feature()], keypoint_distance=KD)
    call([rec(a)])
    a.f = 1
    batch_feature_track(ba, [a.feature()], keypoint_distance=KD)    # previous frame id 1: the link's frame id
    call([rec(a)])
    # a window that would outgrow max_landmarks once the candidates are in: found after the gather
    small = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=8, max_obs=64)
    try:
        sb = BatchWindows(small)
        q = Seq(0, 0, 0, 4, 960)
        out = batch_feature_track(small, [q.feature()], keypoint_distance=KD)
        sb.reset(0, q.run.w)
        sb.edit([Edit(0).frame(_state16(q.run, 0))])
        sb.set_keypoints(0, q.tracker, 1, {})
        q.f = 1
        out = batch_feature_track(small, [q.feature()], keypoint_distance=KD)
        assert len(out[0]["keypoints"]) > 8
        samples, t_end, noise = q.imu()
        r, sms, o, keep = BatchWindows.mirror_records([Mirror(0, q.tracker, samples, t_end, noise, CX, CY)], CAP)
        assert small.lib.pvio_b200_batch_window_mirror_frame(small.h, 1, r, None) == EINVAL
        assert np.all(o[0]["kp_track"] == -7)
        assert sb.download([0], 64)[0]["frames"].shape == (1, 16)
    finally:
        small.close()


def test_launches_do_not_depend_on_n():
    big = BundleAdjustor(max_windows=264, max_frames=4, max_landmarks=512, max_obs=4096)
    try:
        bw = BatchWindows(big)
        counts = []
        for n in (8, 264):
            seqs = [Seq(j, j, j, 3, 1000 + j % 8) for j in range(n)]
            for s in seqs:
                s.tracker = 300 + s.j
            _start(bw, seqs)
            ft = _advance(bw, seqs)
            recs = []
            for s in seqs:
                samples, t_end, noise = s.imu()
                recs.append(Mirror(s.slot, s.tracker, samples, t_end, noise, CX, CY))
            n0 = big.kernel_launches
            out = bw.mirror_frame(recs, CAP)
            counts.append(big.kernel_launches - n0)
            assert all(o["counts"][0] + o["counts"][2] <= len(f["keypoints"]) for o, f in zip(out, ft))
        assert counts[0] == counts[1]
        print("launches per mirror_frame call:", counts)
    finally:
        big.close()


def test_host_mirrored_twin_over_a_restart(ba):
    """4 sequences against a host-mirrored twin (feature_track -> host mirror -> track_frame -> edit -> set_imu on the
    twin slot, from its own results): equal keyframe decisions, ids and track sets, states within 2e-6, over at least
    12 keyframes per sequence, non-keyframes, and one restart of a tracker slot and its windows"""
    bw = BatchWindows(ba)
    seqs = [Seq(j, j, 4 + j, 34, 980 + j) for j in range(4)]
    _start(bw, seqs)
    keyframes, replaced = [0] * 4, 0
    for k in range(33):
        if k == 16:                                              # sequence 0 starts again in its tracker slot
            s = seqs[0]
            s.f += 1
            s.start = s.f
            o = batch_feature_track(ba, [s.feature()], keypoint_distance=KD)[0]
            s.seat(bw, o["keypoints"])
            continue
        ft = _advance(bw, seqs)
        replaced += sum(not s.newest_kf for s in seqs)
        out = _step(bw, seqs, ft, host=True)
        for s, o in zip(seqs, out):
            keyframes[s.j] += o["keyframe"]
        full = [s for s in seqs if s.newest_kf and s.N >= 6]
        if full:
            _drop(bw, seqs, full)
        for s in seqs:
            if k % 4 == 2 and s.newest_kf and s not in full and s.N >= 2:
                s.newest_kf = False
                bw.set_keypoints(s.slot, s.tracker, s.f + 1, {t: kj for kj, t in s.tk.items()}, False, s.skipped)
    print(f"keyframes per sequence {keyframes}, replaced frames {replaced}")
    assert min(keyframes) >= 12 and replaced > 0
