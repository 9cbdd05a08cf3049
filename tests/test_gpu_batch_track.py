"""pvio_b200_batch_track_keypoints: OpenCvImage::track_keypoints (opencv_image.cpp:88-136) for many sequences in one
call, each sequence with its own pyramid cache slot.  Every pair must equal, bit for bit, what the single calls give
for its sequence on a handle of its own: LK positions, status, LK error, and the F-matrix info (iterations run, winning
iteration and model, method) -- equal info pins the schedule drawn on the device to OpenCV's, drawn on the host."""
import ctypes as C

import numpy as np
import pytest

from pvio_b200 import _lib, klt
from pvio_b200._lib import EINVAL
from synthetic import synth

METHOD = {None: 0, "ransac": 1, "lmeds": 2, "7point": 3}


def test_klt_pair_layout_matches_header():
    assert C.sizeof(_lib.CKltPair) == 96
    assert _lib.CKltPair.prev_id.offset == 16 and _lib.CKltPair.prev.offset == 32
    assert _lib.CKltPair.n_points.offset == 48 and _lib.CKltPair.prev_pts.offset == 56 and _lib.CKltPair.info.offset == 88


def _handle():
    from pvio_b200.bundle_adjustor import BundleAdjustor
    return BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)


@pytest.fixture(scope="module")
def ba():
    b = _handle()
    yield b
    b.close()


def _guess(pts, seed):
    """Initial guesses with outliers: a tenth start up to 6 px off (LK locks onto other texture), a twentieth up to
    40 px off, as the outliers of synth.make_fm_matches."""
    r = np.random.default_rng(seed)
    init = pts.copy()
    n = len(pts)
    if n:
        a = r.choice(n, max(n // 10, 1), replace=False)
        init[a] += r.uniform(-6, 6, (len(a), 2)).astype(np.float32)
        b = r.choice(n, n // 20, replace=False)
        init[b] += r.uniform(-40, 40, (len(b), 2)).astype(np.float32)
    return init


def _single(ref, prev, nxt, pts, init, prev_id, next_id, clahe_clip):
    """The reference of one step on a handle of its own: pvio_b200_klt_track_cached (LK, border) for positions, status
    and error; pvio_b200_find_fundamental_mask over its survivors for the info; pvio_b200_track_keypoints for the
    final status."""
    nx, st, err = klt.track_keypoints(ref, prev, nxt, pts, init, prev_id=prev_id, next_id=next_id, clahe_clip=clahe_clip)
    info = np.array([0, -1, -1, 0], dtype=np.int32)
    fin = st.copy()
    l = np.nonzero(st)[0]
    if len(l) >= 8:
        m, _, d = klt.find_fundamental_mask(ref, pts[l], nx[l], return_info=True)
        info = np.array([d["iterations"], d["best_iteration"], d["best_model"], METHOD[d["method"]]], dtype=np.int32)
        fin[l[m == 0]] = 0
    if len(pts):
        nx2, st2 = klt.track_keypoints_ransac(ref, prev, nxt, pts, init, prev_id=prev_id, next_id=next_id,
                                              clahe_clip=clahe_clip)
        assert np.array_equal(st2, fin) and np.array_equal(nx2, nx)
    return nx, fin, err, info


def _assert_same(got, want, what):
    for g, w, name in zip(got, want, ("next_pts", "status", "err", "info")):
        assert np.array_equal(g, w), (what, name)


def _sequences(clahe_clip, ba):
    """12 sequences of 4 frames: three shapes (160 x 120 takes OpenCV's small-image level rule), 0 / 10 / 14 / 60 / 500
    points, border points that leave fewer than 8 survivors, grid points without jitter (exact collinear triples, which
    getSubset rejects)."""
    shapes = [(752, 480), (512, 512), (160, 120)]
    counts = [0, 10, 14, 60, 500]
    seqs = []
    for i in range(12):
        size, count = shapes[i % 3], counts[i % 5]
        A, B, pts, _ = synth.make_klt_pair(seed=700 + i, size=size, n_points=max(count, 1), max_shift=6.0)
        pts = pts[:count]
        if count == 10 and i % 2 == 0:
            pts[:4, 0] = 12.0                 # inside the 20-px border: 6 survivors, RANSAC does not run
        if i % 4 == 3 and count >= 60:
            pts = (np.round((pts - 35.0) / 25.0) * 25.0 + 35.0).astype(np.float32)
        frames = [A, B, A, B]
        if clahe_clip == 0.0:
            frames = [klt.clahe(ba, f) for f in frames]
        seqs.append({"frames": frames, "pts": pts, "shape": (size[1], size[0])})
    return seqs


@pytest.mark.gpu
@pytest.mark.parametrize("clahe_clip", [6.0, 0.0])
def test_batch_matches_single_calls_through_the_cache(ba, clahe_clip):
    seqs = _sequences(clahe_clip, ba)
    slots = [int(s) for s in np.random.default_rng(3).permutation(40)[:len(seqs)] + (0 if clahe_clip else 100)]
    want = []
    for k, sq in enumerate(seqs):
        ref = _handle()
        try:
            want.append([_single(ref, sq["frames"][t], sq["frames"][t + 1], sq["pts"], _guess(sq["pts"], 10 * k + t),
                                 t + 1, t + 2, clahe_clip) for t in range(3)])
        finally:
            ref.close()
    methods = set()
    for t in range(3):
        order = np.random.default_rng(t).permutation(len(seqs))
        pairs = [{"slot": slots[k], "prev_id": t + 1, "next_id": t + 2, "prev": seqs[k]["frames"][t] if t == 0 else None,
                  "next": seqs[k]["frames"][t + 1], "pts": seqs[k]["pts"], "init": _guess(seqs[k]["pts"], 10 * k + t)}
                 for k in order]
        got = klt.batch_track_keypoints(ba, pairs, clahe_clip=clahe_clip)
        for j, k in enumerate(order):
            _assert_same(got[j], want[k][t], (clahe_clip, k, t))
            methods.add(int(got[j][3][3]))
    assert {0, 1, 2} <= methods


@pytest.mark.gpu
def test_batch_beyond_one_wave():
    """264 pairs of 500 points (132 k LK warps, 264 k RANSAC warps) tiled from 8 seeds, both frames new: staging growth
    and every per-pair offset."""
    seeds = []
    for s in range(8):
        size = (752, 480) if s % 2 == 0 else (512, 512)
        A, B, _, _ = synth.make_klt_pair(seed=800 + s, size=size)
        r = np.random.default_rng(800 + s)
        pts = np.stack([r.uniform(25, size[0] - 25, 500), r.uniform(25, size[1] - 25, 500)], 1).astype(np.float32)
        init = _guess(pts, 800 + s)
        ref = _handle()
        try:
            seeds.append((A, B, pts, init, _single(ref, A, B, pts, init, 1, 2, 6.0)))
        finally:
            ref.close()
    b = _handle()
    try:
        pairs = [{"slot": i, "prev_id": 1, "next_id": 2, "prev": seeds[i % 8][0], "next": seeds[i % 8][1],
                  "pts": seeds[i % 8][2], "init": seeds[i % 8][3]} for i in range(264)]
        got = klt.batch_track_keypoints(b, pairs, clahe_clip=6.0)
        for i in range(264):
            _assert_same(got[i], seeds[i % 8][4], i)
    finally:
        b.close()


def _pair(slot, prev_id, next_id, prev, nxt, pts, init=None, shape=None):
    return {"slot": slot, "prev_id": prev_id, "next_id": next_id, "prev": prev, "next": nxt, "pts": pts, "init": init,
            "shape": shape}


def _ref_steps(steps, clahe_clip=6.0):
    """single-call results of consecutive steps (prev, next, pts, prev_id, next_id) on a fresh handle"""
    ref = _handle()
    try:
        return [_single(ref, p, q, pts, None, i, j, clahe_clip) for p, q, pts, i, j in steps]
    finally:
        ref.close()


@pytest.mark.gpu
def test_slot_caches_are_isolated():
    A, B, pa, _ = synth.make_klt_pair(seed=901, n_points=120)
    C_, D, pc, _ = synth.make_klt_pair(seed=902, n_points=120)
    _, E, _, _ = synth.make_klt_pair(seed=903, n_points=120)
    S, T, ps, _ = synth.make_klt_pair(seed=904, size=(512, 512), n_points=120)
    s1, s2, ss, _ = synth.make_klt_pair(seed=905, size=(160, 120), n_points=20)
    b = _handle()
    try:
        # the same ids in two slots name different images; a single-call sequence runs beside them
        single0 = klt.track_keypoints(b, A, B, pa, prev_id=1, next_id=2, clahe_clip=6.0)
        g1 = klt.batch_track_keypoints(b, [_pair(5, 1, 2, C_, D, pc), _pair(2, 1, 2, A, E, pa), _pair(9, 1, 2, S, T, ps)],
                                       clahe_clip=6.0)
        single1 = klt.track_keypoints(b, None, E, pa, prev_id=2, next_id=3, clahe_clip=6.0)
        # slot 9 changes shape (its cache is dropped); slots 5 and 2 continue from their own cached frames
        g2 = klt.batch_track_keypoints(b, [_pair(9, 7, 8, s1, s2, ss), _pair(2, 2, 3, None, B, pa), _pair(5, 2, 3, None, C_, pc)],
                                       clahe_clip=6.0)
        ref_single = _ref_steps([(A, B, pa, 1, 2), (B, E, pa, 2, 3)])
        for got, want in ((single0, ref_single[0]), (single1, ref_single[1])):      # positions and LK error
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[2], want[2])
        rc = _ref_steps([(C_, D, pc, 1, 2), (D, C_, pc, 2, 3)])
        ra = _ref_steps([(A, E, pa, 1, 2), (E, B, pa, 2, 3)])
        rs = _ref_steps([(S, T, ps, 1, 2)])
        rss = _ref_steps([(s1, s2, ss, 7, 8)])
        _assert_same(g1[0], rc[0], "slot 5 first")
        _assert_same(g1[1], ra[0], "slot 2 first")
        _assert_same(g1[2], rs[0], "slot 9 first")
        _assert_same(g2[0], rss[0], "slot 9 new shape")
        _assert_same(g2[1], ra[1], "slot 2 cached")
        _assert_same(g2[2], rc[1], "slot 5 cached")
        # a 0-point pair caches its next frame
        g3 = klt.batch_track_keypoints(b, [_pair(5, 3, 4, None, E, pc[:0])], clahe_clip=6.0)
        assert len(g3[0][0]) == 0 and g3[0][3].tolist() == [0, -1, -1, 0]
        g4 = klt.batch_track_keypoints(b, [_pair(5, 4, 5, None, D, pc)], clahe_clip=6.0)
        _assert_same(g4[0], _ref_steps([(E, D, pc, 4, 5)])[0], "after a 0-point pair")
    finally:
        b.close()


@pytest.mark.gpu
def test_launch_count_does_not_grow_with_the_batch():
    A, B, pts, _ = synth.make_klt_pair(seed=910)
    _, Cn, _, _ = synth.make_klt_pair(seed=911)
    b = _handle()
    try:
        klt.batch_track_keypoints(b, [_pair(s, 1, 2, A, B, pts) for s in range(67)], clahe_clip=6.0)
        counts = []
        for slots in ([0], [1, 2], list(range(3, 67))):
            l0 = b.kernel_launches
            got = klt.batch_track_keypoints(b, [_pair(s, 2, 3, None, Cn, pts) for s in slots], clahe_clip=6.0)
            counts.append(b.kernel_launches - l0)
            assert all(np.array_equal(g[1], got[0][1]) for g in got)
        assert counts[0] == counts[1] == counts[2] and counts[0] <= 7 + 3, counts
        l0 = b.kernel_launches
        assert b.lib.pvio_b200_batch_track_keypoints(b.h, 0, None, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99) == 0
        assert b.kernel_launches == l0
    finally:
        b.close()


@pytest.mark.gpu
def test_rejected_calls_change_nothing():
    A, B, pts, _ = synth.make_klt_pair(seed=920, n_points=200)
    _, Cn, _, _ = synth.make_klt_pair(seed=921, n_points=200)
    b = _handle()
    try:
        klt.batch_track_keypoints(b, [_pair(0, 1, 2, A, B, pts), _pair(1, 1, 2, A, B, pts)], clahe_clip=6.0)

        def attempt(edit, max_level=3):
            cp, outs, keep = klt.pack_pairs([_pair(0, 2, 3, None, Cn, pts), _pair(1, 2, 3, None, Cn, pts)])
            for nx, st, err, info in outs:
                st[:] = 0xAB
                err[:] = -5.0
                info[:] = -7
            before = [[a.copy() for a in o] for o in outs]
            edit(cp)
            rc = b.lib.pvio_b200_batch_track_keypoints(b.h, 2, cp, max_level, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99)
            assert rc == EINVAL
            for o, w in zip(outs, before):
                assert all(np.array_equal(x, y) for x, y in zip(o, w))

        def setf(field, value, i=1):
            return lambda cp: setattr(cp[i], field, value)
        attempt(setf("slot", 0))                                   # a slot given twice
        attempt(setf("slot", -1))
        attempt(setf("n_points", -1))
        for field in ("prev_pts", "next_pts", "status"):
            attempt(setf(field, None))
        attempt(setf("prev_id", 99))                               # not cached in its slot, no pixels
        attempt(setf("prev_id", 0))
        attempt(setf("width", 1))
        attempt(setf("stride", 700))
        attempt(lambda cp: (setattr(cp[1], "width", 100), setattr(cp[1], "height", 100)))   # not a multiple of 8 x 8
        attempt(lambda cp: None, max_level=-1)
        attempt(lambda cp: None, max_level=8)
        # the caches are as they were: the next call still continues from frame 2 in both slots
        got = klt.batch_track_keypoints(b, [_pair(1, 2, 3, None, Cn, pts), _pair(0, 2, 3, None, Cn, pts)], clahe_clip=6.0)
        want = _ref_steps([(A, B, pts, 1, 2), (B, Cn, pts, 2, 3)])[1]
        _assert_same(got[0], want, "slot 1")
        _assert_same(got[1], want, "slot 0")
    finally:
        b.close()
