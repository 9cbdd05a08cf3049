"""pvio_b200_batch_window_save / pvio_b200_batch_window_restore: live sequences (window slot + tracker slot) saved to
host memory and restored into other slots, into a second handle with larger capacities, and back into their own slots
(a rollback).  Inertial sequences run the full per-frame cycle of test_gpu_batch_window_mirror (feature_track ->
mirror_frame -> solve -> download -> prune -> drop_victim -> plane refit / set_planes); visual-only sequences on fp32
handles run feature_track -> localize -> edit -> set_keypoints -> solve -> prune -> plane refit.  A restored copy must
then run its cycle as the original did: bit for bit where the two runs share a handle shape, within the repository's
bar across handles with other frame capacities.
The sequences live in slots at or above half the SM count: a solve whose slot range spans that many windows gives each
window one CTA per sweep (api.cu: sweep_grid_x), whose sums do not depend on the order CTAs finish in, so two runs of the
same window agree bit for bit and a field the blob misses shows up as a difference."""
import copy

import numpy as np
import pytest

from pvio_b200._lib import EINVAL, CWindowSnapshot, ptr
from pvio_b200.batch_window import BatchWindows, Edit, Localize, Mirror, PlaneRansac, Planes
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200.feature_track import batch_feature_track
from test_gpu_batch_window_mirror import CAP, CX, CY, KD, SEQ_TOL, Seq, _advance, _bits, _start, _state16

pytestmark = pytest.mark.gpu
NMAX = (7, 9, 10, 10)                        # each inertial sequence drops its oldest keyframe at this window size
WARM = 9                                     # frames before the save
REPLAY = 6                                   # frames after it
VMAX = 8                                     # a visual-only window replaces its newest frame from this size on


def _base():
    """the first slot the sequences use: a solve over slots [0, base] takes one CTA per window and sweep"""
    torch = pytest.importorskip("torch")
    return (torch.cuda.get_device_properties(0).multi_processor_count + 1) // 2


def _handle(W, frames=10, obs=16384):
    return BundleAdjustor(max_windows=W, max_frames=frames, max_landmarks=4096, max_obs=obs)


class Where:
    """where one sequence lives: a handle's BatchWindows, a window slot and a tracker slot"""

    def __init__(self, bw, slot, tracker):
        self.bw, self.slot, self.tracker = bw, slot, tracker


def _feature(s, w):
    return dict(slot=w.tracker, frame_id=s.f + 1, image=s.frames[s.f], K=s.K, map_frames=min(s.f - s.start, 20),
                max_keypoints=CAP)


def _cycle(seqs, wheres):
    """one frame of every sequence at its Where (one handle); returns what the frame produced, for comparison between
    runs"""
    bw = wheres[0].bw
    ft = batch_feature_track(bw.ba, [_feature(s, w) for s, w in zip(seqs, wheres)], keypoint_distance=KD)
    recs = []
    for s, w in zip(seqs, wheres):
        samples, t_end = s.run.truth.imu_factors[s.f - 1][:2]
        recs.append(Mirror(w.slot, w.tracker, samples, t_end, s.run.truth.imu_noise, CX, CY, True))
    mo = bw.mirror_frame(recs, CAP)
    slots = [w.slot for w in wheres]
    bw.solve(slots, max_iterations=3)
    ds = bw.download(slots, 4096)
    out = dict(ft=ft, mirror=mo, down=ds)
    edits, planes, full = [], [], []
    for j, (s, w, o, d) in enumerate(zip(seqs, wheres, mo, ds)):
        ids = d["ids"][d["n_obs"] >= 2]
        rm = [int(i) for i in ids if i % 13 == s.f % 13]          # a prune that depends on integers only
        if rm:
            e = Edit(w.slot)
            e.remove = rm
            edits.append(e)
        if j == 1 and s.f % 4 == 0:                               # plane roles: -2 tracks
            keep = [int(i) for i in ids if i not in rm][1::6][:6]
            p = Planes(w.slot)
            for t in keep:
                p.role(t, -2)
            planes.append(p)
        if o["keyframe"] and len(d["frames"]) >= NMAX[j]:
            full.append(w.slot)
    if edits:
        bw.edit(edits)
    if planes:
        bw.set_planes(planes)
    if full:
        bw.drop_victim(full)
    d2 = bw.download(slots, 4096)
    out["ransac"] = bw.plane_ransac([PlaneRansac(w.slot, PlaneRansac.REFIT, d["ids"][d["n_obs"] >= 2][:40])
                                     for w, d in zip(wheres, d2)])
    for j, (s, w, o, d) in enumerate(zip(seqs, wheres, mo, d2)):  # a forced non-keyframe now and then
        if j == 3 and s.f % 3 == 1 and o["keyframe"] and w.slot not in full:
            live = set(d["ids"].tolist())
            kp = o["kp_track"][:len(ft[j]["keypoints"])]
            bw.set_keypoints(w.slot, w.tracker, s.f + 1, {int(t): kj for kj, t in enumerate(kp) if t in live}, False,
                             o["skipped_frames"])
            out["forced"] = True
    out["down2"] = d2
    return out


def _run(seqs, wheres, f0, frames):
    """`frames` frames of every sequence from frame f0 + 1 at its Where"""
    outs = []
    for k in range(frames):
        for s in seqs:
            s.f = f0 + 1 + k
        outs.append(_cycle(seqs, wheres))
    return outs


def _same(a, b, exact):
    """two runs of the same frames: the tracker's outputs and every integer bit for bit; states and inverse depths bit
    for bit (exact) or within the repository's bar, 2e-6 relative to the larger of 1 and the values' magnitude"""
    for x, y in zip(a, b):
        for fa, fb in zip(x["ft"], y["ft"]):
            assert np.array_equal(_bits(fa["keypoints"]), _bits(fb["keypoints"]))
            assert np.array_equal(fa["prev_index"], fb["prev_index"]) and list(fa["counts"]) == list(fb["counts"])
        for ma, mb, fa in zip(x["mirror"], y["mirror"], x["ft"]):
            m = len(fa["keypoints"])
            assert np.array_equal(ma["kp_track"][:m], mb["kp_track"][:m]) and list(ma["counts"]) == list(mb["counts"])
            assert (ma["keyframe"], ma["skipped_frames"]) == (mb["keyframe"], mb["skipped_frames"])
            if exact:
                assert np.array_equal(_bits(ma["state"]), _bits(mb["state"]))
            else:
                assert np.abs(ma["state"] - mb["state"]).max() <= SEQ_TOL * max(1.0, np.abs(ma["state"]).max())
        for key in ("down", "down2"):
            for da, db in zip(x[key], y[key]):
                for k in ("ids", "anchor", "n_obs"):
                    assert np.array_equal(da[k], db[k]), k
                for k in ("frames", "inv_depth"):
                    if exact:
                        assert np.array_equal(_bits(da[k]), _bits(db[k])), k
                    elif da[k].size:
                        assert np.abs(da[k] - db[k]).max() <= SEQ_TOL * max(1.0, np.abs(da[k]).max()), k
                if exact:
                    assert np.array_equal(da["valid"], db["valid"])
        for ra, rb in zip(x["ransac"], y["ransac"]):
            assert np.array_equal(ra["used"], rb["used"])
            if exact:
                assert np.array_equal(_bits(ra["points"]), _bits(rb["points"]))


def _agree(a, b):
    """whether two runs' states and inverse depths are equal bit for bit (their integers are checked by _same)"""
    try:
        _same(a, b, exact=True)
        return True
    except AssertionError:
        _same(a, b, exact=False)
        return False


def _probe(bw, slots):
    return bw.download(slots, 4096), bw.imu_records(slots)


def _probe_equal(a, b):
    for da, db in zip(a[0], b[0]):
        for k in da:
            assert np.array_equal(_bits(da[k]) if da[k].dtype == np.float64 else da[k],
                                  _bits(db[k]) if db[k].dtype == np.float64 else db[k]), k
    for ra, rb in zip(a[1], b[1]):
        assert np.array_equal(_bits(ra), _bits(rb))


def _sizes(bw, slots, trackers):
    recs = (CWindowSnapshot * len(slots))()
    for r, s, t in zip(recs, slots, trackers):
        r.slot, r.tracker_slot = s, t
    assert bw.lib.pvio_b200_batch_window_save(bw.h, len(slots), recs) == 0
    return [r.size for r in recs]


def _warm(seqs, bw):
    _start(bw, seqs)
    return _run(seqs, [Where(bw, s.slot, s.tracker) for s in seqs], 0, WARM - 1)


@pytest.fixture(scope="module")
def world():
    """4 linked inertial sequences after WARM frames on handle A (slots B0 .. B0 + 3, tracker slots 100..103), and a
    handle B with larger capacities"""
    B0 = _base()
    a, b = _handle(B0 + 8), _handle(B0 + 16, frames=11, obs=32768)
    bw = BatchWindows(a)
    seqs = [Seq(j, B0 + j, B0 + 7, WARM + REPLAY + 2, 1200 + j) for j in range(4)]   # seat() also seats B0 + 7
    warm = _warm(seqs, bw)
    yield a, b, bw, BatchWindows(b), seqs, warm, B0
    a.close()
    b.close()


def test_round_trip_and_rollback(world):
    a, b, bwa, bwb, seqs, warm, B0 = world
    slots, trk = [s.slot for s in seqs], [s.tracker for s in seqs]
    Ns = [len(x["frames"]) for x in bwa.download(slots, 4096)]
    print("window frames:", Ns)
    assert Ns[:3] == [6, 8, 9]
    sizes = _sizes(bwa, slots, trk)
    blobs = bwa.save(slots, trk)
    assert [len(x) for x in blobs] == sizes
    print("bytes per sequence:", sizes)
    orig = _probe(bwa, slots)
    # other slots of the same handle, and a handle with larger capacities
    copies, ca = [B0 + 4 + j for j in range(4)], [104 + j for j in range(4)]
    others, cb = [B0 + 9 + j for j in range(4)], [200 + j for j in range(4)]
    bwa.restore(copies, blobs, ca)
    _probe_equal(orig, _probe(bwa, copies))
    assert bwa.save(copies, ca) == blobs
    bwb.restore(others, blobs, cb)
    _probe_equal(orig, _probe(bwb, others))
    assert bwb.save(others, cb) == blobs
    assert _sizes(bwb, others, cb) == sizes
    _probe_equal(orig, _probe(bwa, slots))                            # the sources did not change
    # the originals run on; then roll back and replay; the copies run the same frames
    f0 = seqs[0].f
    first = _run(seqs, [Where(bwa, s.slot, s.tracker) for s in seqs], f0, REPLAY)
    bwa.restore(slots, blobs, trk)
    _probe_equal(orig, _probe(bwa, slots))
    again = _run(seqs, [Where(bwa, s.slot, s.tracker) for s in seqs], f0, REPLAY)
    copy_a = _run(seqs, [Where(bwa, t, k) for t, k in zip(copies, ca)], f0, REPLAY)
    # the bar: bit for bit where two reference runs of the same restored state (the rollback and the copy) agree bit for
    # bit, otherwise 2e-6.  The fp64 pipeline of inertial windows accumulates parts of the reduced system with atomics,
    # so its runs may differ in the last bits; the visual-only test below holds fp32 windows to the bit.
    exact = _agree(again, copy_a)
    print("inertial reference runs agree bit for bit:", exact)
    _same(first, again, exact=exact)
    _same(first, copy_a, exact=exact)
    other = _run(seqs, [Where(bwb, t, k) for t, k in zip(others, cb)], f0, REPLAY)
    _same(first, other, exact=False)                                  # other frame capacity: within the bar
    assert any(o.get("forced") for o in warm + first)                 # non-keyframes were replaced
    for s in seqs:
        s.f = f0


# ---- visual-only sequences on fp32 handles: host-driven edits on linked slots
def _vseat(bw, s, z):
    w = copy.copy(s.run.w)
    w.use_inertial = False
    bw.reset(s.slot, w)
    e = Edit(s.slot).frame(_state16(s.run, 0), fixed=True)
    e.new = [(0, q, 1.0) for q in z]
    ids = bw.edit([e])[0]
    s.tk = {k: int(i) for k, i in enumerate(ids)}                    # keypoint of the newest frame -> track id
    bw.set_keypoints(s.slot, s.tracker, 1, {i: k for k, i in s.tk.items()})


def _vcycle(seqs, wheres):
    """one frame of every visual-only sequence at its Where: the tracker step, the PnP of the continued tracks, the frame
    edit (the newest frame replaced every other frame and once the window holds VMAX frames; every other keypoint a new
    track), the link, a solve, a prune, a plane refit.  s.tk is the host's keypoint -> track map of the newest frame."""
    bw = wheres[0].bw
    slots = [w.slot for w in wheres]
    ft = batch_feature_track(bw.ba, [_feature(s, w) for s, w in zip(seqs, wheres)], keypoint_distance=KD)
    pre = bw.download(slots, 4096)
    plans, locs = [], []
    for s, w, o, d in zip(seqs, wheres, ft, pre):
        N = len(d["frames"])
        replace = N >= 2 and (s.f % 2 == 0 or N >= VMAX)
        ends = {int(i) for i, an, c in zip(d["ids"], d["anchor"], d["n_obs"]) if c == 1 and an == N - 1} if replace else set()
        cont = [(kj, s.tk[ki]) for kj, ki in enumerate(o["prev_index"]) if ki >= 0 and ki in s.tk and s.tk[ki] not in ends]
        L = Localize(w.slot, d["frames"][-1])
        for kj, t in cont:
            L.observe(t, o["keypoints"][kj])
        plans.append((replace, cont, N))
        locs.append(L)
    lo = bw.localize(locs)
    edits, news = [], []
    for s, w, o, l, (replace, cont, N) in zip(seqs, wheres, ft, lo, plans):
        zj, fnew = o["keypoints"], N - 1 if replace else N
        e = Edit(w.slot, replace).frame(l["state"])
        e.obs = [(t, fnew, zj[kj]) for kj, t in cont]
        used = {kj for kj, _ in cont}
        new = [kj for kj in range(len(zj)) if kj not in used]
        e.new = [(fnew, zj[kj], 1.0) for kj in new]
        edits.append(e)
        news.append(new)
    got = bw.edit(edits)
    for s, w, (replace, cont, N), new, ids in zip(seqs, wheres, plans, news, got):
        s.tk = {kj: t for kj, t in cont}
        s.tk.update({kj: int(i) for kj, i in zip(new, ids)})
        bw.set_keypoints(w.slot, w.tracker, s.f + 1, {t: kj for kj, t in s.tk.items()})
    bw.solve(slots, max_iterations=3)
    ds = bw.download(slots, 4096)
    edits = []
    for s, w, d in zip(seqs, wheres, ds):
        N = len(d["frames"])
        rm = [int(i) for i, an, c in zip(d["ids"], d["anchor"], d["n_obs"])
              if (c >= 2 and i % 13 == s.f % 13) or (c == 1 and an < N - 1)]      # and tracks the tracker lost at birth
        if rm:
            e = Edit(w.slot)
            e.remove = rm
            edits.append(e)
            s.tk = {k: t for k, t in s.tk.items() if t not in set(rm)}
    if edits:
        bw.edit(edits)
    d2 = bw.download(slots, 4096)
    ransac = bw.plane_ransac([PlaneRansac(w.slot, PlaneRansac.REFIT, d["ids"][d["n_obs"] >= 2][:40])
                              for w, d in zip(wheres, d2)])
    return dict(ft=ft, loc=lo, down=ds, down2=d2, ransac=ransac)


def _vrun(seqs, wheres, f0, frames, tks):
    for s, tk in zip(seqs, tks):
        s.tk = dict(tk)
    outs = []
    for k in range(frames):
        for s in seqs:
            s.f = f0 + 1 + k
        outs.append(_vcycle(seqs, wheres))
    return outs


def _vsame(a, b):
    for x, y in zip(a, b):
        for fa, fb in zip(x["ft"], y["ft"]):
            assert np.array_equal(_bits(fa["keypoints"]), _bits(fb["keypoints"]))
            assert np.array_equal(fa["prev_index"], fb["prev_index"])
        for la, lb in zip(x["loc"], y["loc"]):
            assert np.array_equal(_bits(la["state"]), _bits(lb["state"]))
        for key in ("down", "down2"):
            for da, db in zip(x[key], y[key]):
                for k in da:
                    assert np.array_equal(_bits(da[k]) if da[k].dtype == np.float64 else da[k],
                                          _bits(db[k]) if db[k].dtype == np.float64 else db[k]), (key, k)
        for ra, rb in zip(x["ransac"], y["ransac"]):
            assert np.array_equal(ra["used"], rb["used"]) and np.array_equal(_bits(ra["points"]), _bits(rb["points"]))


def test_visual_only_rollback_is_bit_exact():
    """two linked visual-only sequences on an fp32 handle: save, run REPLAY frames, roll back and replay, and run the
    copies in other slots and in a second fp32 handle with more windows and observations: every output bit for bit"""
    B0 = _base()
    v1, v2 = _handle(B0 + 4, frames=9), _handle(B0 + 12, frames=9, obs=32768)
    try:
        bw1, bw2 = BatchWindows(v1), BatchWindows(v2)
        seqs = [Seq(j, B0 + j, B0 + j, WARM + REPLAY + 2, 1300 + j) for j in range(2)]
        out = batch_feature_track(v1, [_feature(s, Where(bw1, s.slot, s.tracker)) for s in seqs], keypoint_distance=KD)
        for s, o in zip(seqs, out):
            _vseat(bw1, s, o["keypoints"])
        wh = [Where(bw1, s.slot, s.tracker) for s in seqs]
        _vrun(seqs, wh, 0, WARM - 1, [s.tk for s in seqs])
        slots, trk = [s.slot for s in seqs], [s.tracker for s in seqs]
        print("visual window frames / tracks:", [(len(d["frames"]), len(d["ids"])) for d in bw1.download(slots, 4096)])
        blobs, tks, f0 = bw1.save(slots, trk), [dict(s.tk) for s in seqs], seqs[0].f
        first = _vrun(seqs, wh, f0, REPLAY, tks)
        bw1.restore(slots, blobs, trk)
        again = _vrun(seqs, wh, f0, REPLAY, tks)
        _vsame(first, again)
        bw1.restore([B0 + 2, B0 + 3], blobs, [110, 111])
        _vsame(first, _vrun(seqs, [Where(bw1, B0 + 2 + j, 110 + j) for j in range(2)], f0, REPLAY, tks))
        bw2.restore([B0 + 7, B0 + 9], blobs, [120, 121])
        assert bw2.save([B0 + 7, B0 + 9], [120, 121]) == blobs
        _vsame(first, _vrun(seqs, [Where(bw2, B0 + 7, 120), Where(bw2, B0 + 9, 121)], f0, REPLAY, tks))
    finally:
        v1.close()
        v2.close()


def test_partial_records(world):
    a, b, bwa, bwb, seqs, warm, B0 = world
    s = seqs[0]
    blob = bwa.save([s.slot], [s.tracker])[0]
    # window only: unlinked, mirror_frame rejects it until set_keypoints
    bwb.restore([B0 + 13], [blob])
    d = bwb.download([B0 + 13], 4096)[0]
    assert np.array_equal(d["ids"], bwa.download([s.slot], 4096)[0]["ids"])
    samples, t_end = s.run.truth.imu_factors[s.f][:2]
    r, sms, out, keep = BatchWindows.mirror_records([Mirror(B0 + 13, 210, samples, t_end, s.run.truth.imu_noise, CX, CY)],
                                                    CAP)
    assert b.lib.pvio_b200_batch_window_mirror_frame(b.h, 1, r, None) == EINVAL
    # tracker only: feature_track continues from it exactly as from the original tracker slot
    bwb.restore([-1], [blob], [210])
    f = s.f + 1
    frame = dict(frame_id=f + 1, image=s.frames[f], K=s.K, map_frames=min(f - s.start, 20), max_keypoints=CAP)
    got = batch_feature_track(b, [dict(frame, slot=210)], keypoint_distance=KD)[0]
    want = batch_feature_track(a, [dict(frame, slot=s.tracker)], keypoint_distance=KD)[0]
    for k in ("keypoints", "prev_index", "counts", "info"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(_bits(got["keypoints"]), _bits(want["keypoints"]))
    bwa.restore([s.slot], [blob], [s.tracker])                       # the original back where it was
    # a record naming a part the blob lacks
    wonly = bwa.save([s.slot])[0]
    before = bwb.save([B0 + 13], [210])
    recs = (CWindowSnapshot * 1)()
    arr = np.frombuffer(wonly, dtype=np.uint8)
    recs[0].slot, recs[0].tracker_slot, recs[0].data, recs[0].capacity = B0 + 13, 210, ptr(arr), len(arr)
    assert b.lib.pvio_b200_batch_window_restore(b.h, 1, recs) == EINVAL
    assert bwb.save([B0 + 13], [210]) == before
    tonly = bwa.save([-1], [s.tracker])[0]
    arr = np.frombuffer(tonly, dtype=np.uint8)
    recs[0].data, recs[0].capacity = ptr(arr), len(arr)
    assert b.lib.pvio_b200_batch_window_restore(b.h, 1, recs) == EINVAL
    assert bwb.save([B0 + 13], [210]) == before


def test_stale_link_is_saved_unlinked(world):
    """a tracker slot that moved on twice without mirror_frame: the window's link names a frame the tracker no longer
    holds, so the blob holds no link and restores unlinked instead of being refused"""
    a, b, bwa, bwb, seqs, warm, B0 = world
    s = seqs[2]
    keep = bwa.save([s.slot], [s.tracker])[0]
    assert _get(keep, "linked") == 1
    for f in (s.f + 1, s.f + 2):
        batch_feature_track(a, [dict(slot=s.tracker, frame_id=f + 1, image=s.frames[f], K=s.K, map_frames=5,
                                     max_keypoints=CAP)], keypoint_distance=KD)
    stale = bwa.save([s.slot], [s.tracker])[0]
    assert _get(stale, "linked") == 0
    bwb.restore([B0 + 14], [stale], [211])
    assert bwb.save([B0 + 14], [211]) == [stale]
    bwa.restore([s.slot], [keep], [s.tracker])


# ---- a blob's layout, as the header describes it (offsets into a copy that the rejections edit)
_HEAD = dict(magic=(0, "<u4"), version=(4, "<u4"), size=(8, "<i8"), N=(20, "<i4"), T=(24, "<i4"), fixed=(28, "<i4"),
             next_id=(32, "<i4"), n_prior=(36, "<i4"), inertial=(40, "<i4"), n_planes=(44, "<i4"), linked=(56, "<i4"),
             n0=(60, "<i4"), n1=(64, "<i4"), w=(72, "<i4"), levels=(80, "<i4"), frame_id=(96, "<u8"),
             link_frame=(112, "<u8"))
_HEAD_BYTES = 160


def _get(blob, k):
    o, t = _HEAD[k]
    return int(np.frombuffer(blob, dtype=t, count=1, offset=o)[0])


def _put(blob, k, v):
    o, t = _HEAD[k]
    return _poke(blob, o, t, v)


def _poke(blob, off, dtype, v):
    out = bytearray(blob)
    out[off:off + np.dtype(dtype).itemsize] = np.array([v], dtype=dtype).tobytes()
    return bytes(out)


def _a16(x):
    return (x + 15) & ~15


def _sections(blob):
    """the offsets of a window + tracker blob's sections"""
    g = {k: _get(blob, k) for k in ("T", "N", "inertial", "n_prior", "n_planes", "n0", "n1")}
    T, N, F = g["T"], g["N"], max(g["N"] - 1, 0) if g["inertial"] else 0
    o, p = {}, _HEAD_BYTES

    def sec(name, n):
        nonlocal p
        o[name] = p
        p += _a16(n)
    sec("ids", 4 * T); sec("mask", 4 * T); sec("role", T); sec("nsmp", 4 * F)
    ns = np.frombuffer(blob, dtype="<i4", count=F, offset=o["nsmp"])
    d, nk = 15 * g["n_prior"], g["n0"] + g["n1"]
    sec("cst", 208); sec("tkp", 4 * T); sec("valid", T); sec("rho", 8 * T); sec("qual", 8 * T); sec("tz", 16 * T * N)
    sec("frames", 128 * N); sec("imu", 8 * 288 * F); sec("pS", 8 * d * d); sec("pe", 8 * d); sec("px0", 128 * g["n_prior"])
    sec("aux", 8 * 37 * int((ns > 0).sum())); sec("smp", 56 * int(ns.sum())); sec("planes", 32 * g["n_planes"])
    sec("kz", 16 * nk); sec("kb", 4 * nk); sec("kp", 4 * nk)
    return o


def test_rejections_change_nothing(world):
    a, b, bwa, bwb, seqs, warm, B0 = world
    s1 = seqs[1]
    blob = bwa.save([s1.slot], [s1.tracker])[0]
    tgt, ttk = B0 + 4, 104                                            # the target of the rejected restores
    bwa.restore([tgt], [blob], [ttk])
    slots, trk = [s.slot for s in seqs] + [tgt], [s.tracker for s in seqs] + [ttk]
    state = bwa.save(slots, trk)
    probe = _probe(bwa, slots)

    def rejected(blobs, slots_=(tgt,), trackers=(ttk,), handle=a):
        recs = (CWindowSnapshot * len(blobs))()
        arrs = [np.frombuffer(x, dtype=np.uint8) for x in blobs]
        for r, x, s, t in zip(recs, arrs, slots_, trackers):
            r.slot, r.tracker_slot, r.data, r.capacity = s, t, ptr(x), len(x)
        assert handle.lib.pvio_b200_batch_window_restore(handle.h, len(blobs), recs) == EINVAL
        assert bwa.save(slots, trk) == state
        _probe_equal(probe, _probe(bwa, slots))

    sec = _sections(blob)
    T, N = _get(blob, "T"), _get(blob, "N")
    assert T >= 3 and _get(blob, "linked") == 1 and _get(blob, "n_prior") > 0 and _get(blob, "n1") > 0
    assert _sections(blob)["kp"] + _a16(4 * (_get(blob, "n0") + _get(blob, "n1"))) < len(blob)
    rejected([_put(blob, "magic", 7)])
    rejected([_put(blob, "version", 2)])
    rejected([blob[:-16]])
    rejected([blob + bytes(16)])
    rejected([_put(blob, "size", len(blob) + 16) + bytes(16)])         # a consistent size, not the layout's
    rejected([_put(blob, "N", 17)])
    rejected([_put(blob, "n_prior", N + 1)])
    rejected([_put(blob, "inertial", 0)])                              # a prior on a visual-only window
    rejected([_put(blob, "n_planes", 5)])
    rejected([_put(blob, "fixed", 1 << N)])
    rejected([_put(blob, "next_id", 0)])                               # ids not below the next id
    ids = np.frombuffer(blob, dtype="<i4", count=T, offset=sec["ids"])
    rejected([_poke(blob, sec["ids"] + 4, "<i4", int(ids[0]))])        # not strictly increasing
    rejected([_poke(blob, sec["ids"], "<i4", -1)])
    rejected([_poke(blob, sec["mask"], "<u4", 0)])
    rejected([_poke(blob, sec["mask"], "<u4", 1 << N)])
    rejected([_poke(blob, sec["role"], "<i1", -3)])
    rejected([_poke(blob, sec["role"], "<i1", _get(blob, "n_planes"))])
    rejected([_poke(blob, sec["tkp"], "<i4", 1 << 20)])
    rejected([_poke(blob, sec["tkp"], "<i4", -2)])
    rejected([_poke(blob, sec["kp"], "<i4", _get(blob, "n1"))])        # prev_index past the previous frame's keypoints
    rejected([_poke(blob, sec["kp"], "<i4", -2)])
    rejected([_put(blob, "w", 5)])                                     # a pyramid the tracker does not build
    rejected([_put(blob, "levels", 9)])
    rejected([_put(blob, "link_frame", 12345)])
    rejected([_put(blob, "frame_id", 0)])
    rejected([blob, blob], (tgt, tgt), (ttk, 105))                     # a slot named twice
    rejected([blob, blob], (tgt, B0 + 5), (ttk, ttk))                  # a tracker slot named twice
    rejected([blob], (-1,), (-1,))
    # handles too small: frames, live tracks, observations; their own target slot stays as it was
    smalls = [dict(max_frames=N - 1), dict(max_obs=1)] + ([dict(max_landmarks=(T - 1) & ~3)] if T > 4 else [])
    for kw in smalls:
        small = BundleAdjustor(**dict(dict(max_windows=2, max_frames=10, max_landmarks=4096, max_obs=16384), **kw))
        try:
            sb = BatchWindows(small)
            sb.reset(0, s1.run.w)
            sb.edit([Edit(0).frame(_state16(s1.run, 0))])
            before = sb.download([0], 64)
            rejected([blob], (0,), (0,), small)
            _probe_equal((before, []), (sb.download([0], 64), []))
            recs = (CWindowSnapshot * 1)()
            recs[0].slot, recs[0].tracker_slot = -1, 0
            assert small.lib.pvio_b200_batch_window_save(small.h, 1, recs) == EINVAL   # tracker slot 0 still not live
        finally:
            small.close()
    # save: capacity below the size leaves the buffer and the size alone
    size = _sizes(bwa, [s1.slot], [s1.tracker])[0]
    buf = np.full(size, 0xAB, dtype=np.uint8)
    recs = (CWindowSnapshot * 1)()
    recs[0].slot, recs[0].tracker_slot, recs[0].data, recs[0].capacity, recs[0].size = s1.slot, s1.tracker, ptr(buf), size - 16, -5
    assert a.lib.pvio_b200_batch_window_save(a.h, 1, recs) == EINVAL
    assert recs[0].size == -5 and np.all(buf == 0xAB)


def test_launches_do_not_depend_on_n():
    big = BundleAdjustor(max_windows=528, max_frames=4, max_landmarks=512, max_obs=4096)
    try:
        bw = BatchWindows(big)
        seqs = [Seq(j, j, j, 3, 1000 + j % 8) for j in range(264)]
        for s in seqs:
            s.tracker = 300 + s.j
        _start(bw, seqs)
        _advance(bw, seqs)
        counts = []
        for n in (8, 264):
            slots, trk = list(range(n)), [300 + j for j in range(n)]
            others = list(range(n, 264))[:8]
            before = bw.download(others, 512)
            n0 = big.kernel_launches
            blobs = bw.save(slots, trk)
            n1 = big.kernel_launches
            bw.restore([264 + j for j in range(n)], blobs, [1000 + j for j in range(n)])
            counts.append((n1 - n0, big.kernel_launches - n1))
            assert bw.save([264 + j for j in range(n)], [1000 + j for j in range(n)]) == blobs
            _probe_equal((before, []), (bw.download(others, 512), []))   # slots not named keep their windows
        assert counts[0] == counts[1] and counts[0][0] == 1
        print("launches per save / restore call:", counts)
    finally:
        big.close()


def test_another_gpu(world):
    torch = pytest.importorskip("torch")
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device")
    a, b, bwa, bwb, seqs, warm, B0 = world
    slots, trk = [s.slot for s in seqs], [s.tracker for s in seqs]
    blobs = bwa.save(slots, trk)
    f0 = seqs[0].f
    first = _run(seqs, [Where(bwa, s.slot, s.tracker) for s in seqs], f0, REPLAY)
    bwa.restore(slots, blobs, trk)
    with torch.cuda.device(1):
        c = BundleAdjustor(device=1, max_windows=B0 + 8, max_frames=10, max_landmarks=4096, max_obs=16384)
        try:
            bwc = BatchWindows(c)
            bwc.restore(slots, blobs, trk)
            assert bwc.save(slots, trk) == blobs
            other = _run(seqs, [Where(bwc, s.slot, s.tracker) for s in seqs], f0, REPLAY)
        finally:
            c.close()
    _same(first, other, exact=True)                                   # the same handle shape on another device
    for s in seqs:
        s.f = f0
