"""The frontend kernels (csrc/klt.cu, csrc/detect.cu) at their edges, against cv2 and the oracles: LK points on, near
and beyond the frame edge at odd, small and sub-window frame sizes (the edge cases of test_klt_oracle_edges.py); LK at
other levels, iteration counts and eps; CLAHE at other clip limits and tile grids on extreme frames; every entry point
that takes a row stride, on a padded frame; the batched tracker on the edge pairs; the detector at odd sizes."""
import ctypes as C

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import clahe_oracle
from oracle import detect_oracle as D
from oracle import klt_oracle as ko
from pvio_b200 import _lib, klt
from pvio_b200.detect import batch_detect_keypoints, detect_keypoints, pack_requests
from synthetic import synth
from test_gpu_batch_track import _assert_same, _handle, _single
from test_klt_oracle_edges import PARAMS, SIZES, assert_lk_parity, cv_lk, edge_case

pytestmark = pytest.mark.gpu
PAD = 13                                    # the padded frames' row stride is width + PAD; the padding holds 0xAB


@pytest.fixture(scope="module")
def ba():
    b = _handle()
    yield b
    b.close()


def _padded(img):
    h, w = img.shape
    buf = np.full((h, w + PAD), 0xAB, np.uint8)
    buf[:, :w] = img
    return buf


_p = _lib.ptr


# ---- LK at the edges --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_edge_points_match_cv2_and_oracle(ba, size):
    prev, nxt, pts, init, kinds = edge_case(size)
    got = klt.track_keypoints(ba, prev, nxt, pts, init, raw=True)
    want = cv_lk(prev, nxt, pts, init)
    assert_lk_parity(got, want, ("cv2", size))
    assert_lk_parity(got, ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init), ("oracle", size))
    assert got[1].sum() >= 4 and (got[1][kinds["outside"]] == want[1][kinds["outside"]]).all()


def test_frames_under_twelve_pixels_are_rejected(ba):
    """Below 12 px the window's reads would fold more than twice: such frames are refused, unlike cv2, which tracks them."""
    prev, nxt, pts, init, _ = edge_case((12, 12))
    rc = ba.lib.pvio_b200_klt_track(ba.h, _p(prev[:, :11].copy()), _p(nxt[:, :11].copy()), 11, 12, 11, _p(pts),
                                    _p(init.copy()), _p(np.zeros(len(pts), np.uint8)),
                                    _p(np.zeros(len(pts), np.float32)), len(pts), 3, 30, 0.01)
    assert rc == _lib.EINVAL


@pytest.mark.parametrize("name,value", PARAMS, ids=[f"{n}={v}" for n, v in PARAMS])
def test_lk_parameters_match_cv2(ba, name, value):
    """max_level 0..7, max_iter 0..150 and eps 0..25 on the odd 753 x 481 frame; the last max_iter and eps test the
    clamps (100 and 10)."""
    prev, nxt, pts, init, _ = edge_case((753, 481))
    kw = {"max_level": 3, "max_iter": 30, "eps": 0.01, name: value}
    got = klt.track_keypoints(ba, prev, nxt, pts, init, raw=True, **kw)
    assert_lk_parity(got, cv_lk(prev, nxt, pts, init, **kw), kw)
    assert_lk_parity(got, ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init, **kw), ("oracle", kw))


# ---- CLAHE ------------------------------------------------------------------------------------------------------
def _track_raw(ba, prev, nxt, pts, clip, tiles, stride=None):
    """pvio_b200_klt_track_raw with its equalised frames; `stride` set: prev / next are padded [h, stride] buffers"""
    h = prev.shape[0]
    w = prev.shape[1] if stride is None else prev.shape[1] - PAD
    cur = np.ascontiguousarray(pts, np.float32)
    out = cur.copy()
    st, err = np.zeros(len(cur), np.uint8), np.zeros(len(cur), np.float32)
    eq = [np.zeros((h, w), np.uint8) for _ in range(2)]
    ba._ck(ba.lib.pvio_b200_klt_track_raw(ba.h, _p(prev), _p(nxt), w, h, stride or w, _p(cur), _p(out), _p(st), _p(err),
                                          len(cur), 3, 30, 0.01, float(clip), tiles[0], tiles[1], _p(eq[0]), _p(eq[1])))
    return out, st, err, eq[0], eq[1]


def _clahe_frames(shape, seed):
    r = np.random.default_rng(seed)
    h, w = shape
    return {"random": r.integers(0, 256, shape, dtype=np.uint8),
            "saturated": np.where(r.random(shape) < 0.5, 0, 255).astype(np.uint8),
            "two-level": np.where(np.arange(w)[None, :] < w // 3, 40, 41).astype(np.uint8).repeat(h, 0),
            "flat0": np.zeros(shape, np.uint8),
            "flat255": np.full(shape, 255, np.uint8),
            "texture": synth.make_klt_pair(seed=seed, size=(w, h), n_points=1)[0]}


TILES = [((1, 1), (481, 753)), ((2, 3), (480, 752)), ((3, 13), (481, 753)), ((4, 6), (480, 752)), ((16, 16), (480, 752))]


@pytest.mark.parametrize("tiles,shape", TILES, ids=[f"{t[0]}x{t[1]}" for t, _ in TILES])
def test_clahe_clip_and_tiles_bit_exact(ba, tiles, shape):
    """pvio_b200_clahe and the equalised frames of pvio_b200_klt_track_raw, every pixel equal to cv2 and the oracle, at
    clip limits 0.5..40 (the clip floor max(clip * area / 256, 1) and the residual step 256 / residual)."""
    frames = _clahe_frames(shape, seed=tiles[0] * 100 + tiles[1])
    pts = np.array([[shape[1] / 2, shape[0] / 2], [30.0, 30.0]], np.float32)
    for clip in (0.5, 1.0, 2.0, 40.0):
        for name, img in frames.items():
            want = cv2.createCLAHE(clip, tiles).apply(img)
            assert np.array_equal(clahe_oracle.clahe(img, clip, tiles), want), (clip, name)
            assert np.array_equal(klt.clahe(ba, img, clip, tiles), want), (clip, name, "pvio_b200_clahe")
            other = frames["texture"] if name != "texture" else frames["random"]
            _, _, _, eq_prev, eq_next = _track_raw(ba, img, other, pts, clip, tiles)
            assert np.array_equal(eq_prev, want), (clip, name, "klt_track_raw")
            assert np.array_equal(eq_next, cv2.createCLAHE(clip, tiles).apply(other)), (clip, name, "klt_track_raw next")


# ---- row stride ----------------------------------------------------------------------------------------------------
def test_every_strided_entry_point_equals_the_contiguous_call(ba):
    """A frame stored with row stride width + 13 (padding 0xAB) gives the bits of the contiguous frame through every
    entry point that takes a stride."""
    prev, nxt, pts, init, _ = edge_case((752, 480))
    n = len(pts)
    h, w = prev.shape
    pp, pn = _padded(prev), _padded(nxt)

    def lk(stride, name):
        a, b = (pp, pn) if stride else (prev, nxt)
        out, st, err = init.copy(), np.zeros(n, np.uint8), np.zeros(n, np.float32)
        args = (_p(pts), _p(out), _p(st), _p(err), n, 3, 30, 0.01)
        s = stride or w
        ids = (11, 12) if stride else (21, 22)          # distinct ids: the strided call must not hit the cache
        if name == "klt_track":
            ba._ck(ba.lib.pvio_b200_klt_track(ba.h, _p(a), _p(b), w, h, s, *args))
            return out, st, err
        if name == "klt_track_cached":
            ba._ck(ba.lib.pvio_b200_klt_track_cached(ba.h, ids[0], _p(a), ids[1], _p(b), w, h, s, *args, 6.0, 8, 8,
                                                     20))
            return out, st, err
        assert name == "track_keypoints"
        ba._ck(ba.lib.pvio_b200_track_keypoints(ba.h, ids[0] + 100, _p(a), ids[1] + 100, _p(b), w, h, s, _p(pts), _p(out),
                                                _p(st), n, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99))
        return out, st

    for name in ("klt_track", "klt_track_cached", "track_keypoints"):
        want, got = lk(0, name), lk(w + PAD, name)
        assert all(np.array_equal(x, y) for x, y in zip(want, got)), name
        assert want[1].sum() > 20, name
    want, got = _track_raw(ba, prev, nxt, init, 6.0, (8, 8)), _track_raw(ba, pp, pn, init, 6.0, (8, 8), stride=w + PAD)
    assert all(np.array_equal(x, y) for x, y in zip(want, got)), "klt_track_raw"

    out = np.zeros_like(prev)
    ba._ck(ba.lib.pvio_b200_clahe(ba.h, _p(pp), w, h, w + PAD, 6.0, 8, 8, _p(out)))
    assert np.array_equal(out, klt.clahe(ba, prev)), "clahe"

    existing = np.ascontiguousarray(pts[::3], np.float64)
    kp = np.zeros((2048, 2))
    gftt = np.zeros((1000, 2), np.float32)
    n_out, n_g = C.c_int(), C.c_int()
    ba._ck(ba.lib.pvio_b200_detect_keypoints(ba.h, 0, _p(pn), w, h, w + PAD, 6.0, 8, 8, _p(existing), len(existing), 25.0,
                                             2048, _p(kp), C.byref(n_out), _p(gftt), C.byref(n_g)))
    want_kp, want_g = detect_keypoints(ba, nxt, existing, keypoint_distance=25.0, clahe_clip=6.0, want_gftt=True)
    assert np.array_equal(kp[:n_out.value], want_kp) and np.array_equal(gftt[:n_g.value], want_g), "detect_keypoints"
    assert n_out.value > 20

    # one pair of the batched tracker, one request of the batched detector
    pair = {"slot": 0, "prev_id": 1, "next_id": 2, "prev": prev, "next": nxt, "pts": pts, "init": init}
    want = klt.batch_track_keypoints(ba, [pair], clahe_clip=6.0)[0]
    cp, outs, keep = klt.pack_pairs([dict(pair, slot=1)])
    cp[0].prev, cp[0].next, cp[0].stride = _p(pp), _p(pn), w + PAD
    ba._ck(ba.lib.pvio_b200_batch_track_keypoints(ba.h, 1, cp, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99))
    _assert_same(outs[0], want, "batch_track_keypoints")
    req = {"slot": 2, "frame_id": 0, "image": nxt, "keypoints": existing}
    want = batch_detect_keypoints(ba, [req], clahe_clip=6.0, want_gftt=True)[0]
    cr, outs, keep2 = pack_requests([req], want_gftt=True)
    cr[0].image, cr[0].stride = _p(pn), w + PAD
    ba._ck(ba.lib.pvio_b200_batch_detect_keypoints(ba.h, 1, cr, 6.0, 8, 8))
    out, cnt, g = outs[0]
    assert np.array_equal(out[:cnt[0]], want[0]) and np.array_equal(g[:cnt[1]], want[1]), "batch_detect_keypoints"
    del keep, keep2


# ---- the batched tracker on the edge pairs -----------------------------------------------------------------------
def test_batched_edge_pairs_equal_single_calls():
    """Every edge pair in one pvio_b200_batch_track_keypoints call: the border test of each pair's own size runs in the
    batched LK kernel, and every pair gives the bits of the single cached calls on a handle of its own."""
    cases = [edge_case(size) for size in SIZES]
    want = []
    for prev, nxt, pts, init, _ in cases:
        ref = _handle()
        try:
            want.append(_single(ref, prev, nxt, pts, init, 1, 2, 0.0))
        finally:
            ref.close()
    b = _handle()
    try:
        pairs = [{"slot": 3 * i + 1, "prev_id": 1, "next_id": 2, "prev": c[0], "next": c[1], "pts": c[2], "init": c[3]}
                 for i, c in enumerate(cases)]
        got = klt.batch_track_keypoints(b, pairs, clahe_clip=0.0)
    finally:
        b.close()
    for size, g, w in zip(SIZES, got, want):
        _assert_same(g, w, size)
    assert sum(int(w[1].sum()) for w in want) > 50


# ---- the detector at odd sizes -------------------------------------------------------------------------------------
DETECT_SIZES = [(753, 481), (161, 121), (97, 203)]


def test_detector_at_odd_sizes(ba):
    """GFTT's corner set equals cv2.goodFeaturesToTrack's; the whole call equals the oracle, in order, on the same
    corners; the batched detector gives the single calls' bits.  Frames textured to the edge, equalised on the host."""
    rng = np.random.default_rng(17)
    reqs, singles = [], []
    for i, (w, h) in enumerate(DETECT_SIZES):
        img = cv2.createCLAHE(6.0, (8, 8)).apply(synth.make_klt_pair(seed=1300 + i, size=(w, h), n_points=1)[0])
        existing = np.stack([rng.uniform(0, w, 12), rng.uniform(0, h, 12)], 1)
        got, corners = detect_keypoints(ba, img, existing, keypoint_distance=25.0, want_gftt=True)
        ref = D.gftt(img)
        a, b = set(map(tuple, ref.astype(int))), set(map(tuple, corners.astype(int)))
        assert len(ref) > 20 and a == b, ((w, h), len(a), len(b), len(a & b))
        assert np.array_equal(got, D.detect_keypoints(img, existing, 25.0, corners=corners)), (w, h)
        assert len(got) > 0, (w, h)
        reqs.append({"slot": i, "image": img, "keypoints": existing})
        singles.append((got, corners))
    for (kp, g), (kp1, g1) in zip(batch_detect_keypoints(ba, reqs, want_gftt=True), singles):
        assert np.array_equal(kp, kp1) and np.array_equal(g, g1)
