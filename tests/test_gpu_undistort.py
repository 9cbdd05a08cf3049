"""Lens undistortion on the device (pvio_b200_batch_set_lens, pvio_b200_batch_undistort, and the remap inside the
batched tracker and detector).  The undistorted frames equal cv2.undistort (radtan, K and D as float32, as
EurocDatasetReader::read_image) and the oracle's equidistant remap (ImageUndistorter) bit for bit; the tracker and the
detector on raw frames of slots with a lens equal the same calls, without lenses, on frames undistorted on the host."""
import numpy as np
import pytest

from oracle import undistort_oracle as uo
from pvio_b200 import _lib, klt
from pvio_b200.detect import batch_detect_keypoints, pack_requests
from pvio_b200.undistort import EQUIDISTANT, NONE, RADTAN, batch_undistort, pack_lenses, set_lens
from pvio_b200._lib import EINVAL
from synthetic import synth

cv2 = pytest.importorskip("cv2")

EUROC = {"model": RADTAN, "width": 752, "height": 480, "K": (458.654, 457.296, 367.215, 248.375),
         "coeffs": (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)}
BARREL = {"model": RADTAN, "width": 640, "height": 480, "K": (300.0, 310.0, 320.5, 240.2), "coeffs": (-0.45, 0.2, 0.0, 0.0)}
SMALL = {"model": RADTAN, "width": 97, "height": 61, "K": (60.0, 61.0, 48.0, 30.0), "coeffs": (-0.2, 0.05, 0.001, 0.002)}
TUMVI = {"model": EQUIDISTANT, "width": 512, "height": 512,
         "K": (190.97847715128717, 190.9733070521226, 254.93170605935475, 256.8974428996504),
         "coeffs": (0.0034003170790442797, 0.001766278153469831, -0.00266312569781606, 0.0003299517423931039)}


def _handle():
    from pvio_b200.bundle_adjustor import BundleAdjustor
    return BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)


def host_undistort(img, lens):
    """what the reference's readers compute on the host"""
    if lens is None:
        return img
    if lens["model"] == RADTAN:
        fx, fy, cx, cy = lens["K"]
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
        return cv2.undistort(img, K, np.array(lens["coeffs"], np.float32))
    return uo.undistort(img, EQUIDISTANT, lens["K"], lens["coeffs"])


def _raw(lens, seed):
    return synth.make_klt_pair(seed=seed, size=(lens["width"], lens["height"]), n_points=8)[0]


@pytest.mark.gpu
def test_batch_undistort_equals_opencv():
    b = _handle()
    try:
        lenses = {3: EUROC, 7: BARREL, 9: SMALL, 11: TUMVI}
        set_lens(b, [dict(v, slot=s) for s, v in lenses.items()])
        r = np.random.default_rng(5)
        reqs, want = [], []
        for k, s in enumerate([11, 3, 9, 7, 3]):          # slot 3 twice: the call reads no cache
            L = lenses[s]
            img = _raw(L, 300 + k) if k % 2 == 0 else r.integers(0, 256, (L["height"], L["width"]), dtype=np.uint8)
            img[:20, :40] = 255
            img[-15:, -30:] = 0
            reqs.append({"slot": s, "image": img})
            want.append(host_undistort(img, L))
        l0 = b.kernel_launches
        got = batch_undistort(b, reqs)
        assert b.kernel_launches == l0 + 1
        for g, w in zip(got, want):
            assert np.array_equal(g, w)
    finally:
        b.close()


def _pairs(seqs, t, with_prev):
    return [{"slot": sq["slot"], "prev_id": t + 1, "next_id": t + 2, "prev": sq["frames"][t] if with_prev else None,
             "next": sq["frames"][t + 1], "pts": sq["pts"], "init": sq["init"][t]} for sq in seqs]


def _sequences():
    """lens and no-lens slots of three shapes, 4 raw frames each; the same sequences undistorted on the host"""
    kinds = [(2, EUROC), (5, TUMVI), (6, BARREL), (8, None), (12, EUROC), (13, None)]
    seqs, host = [], []
    for k, (slot, L) in enumerate(kinds):
        size = (L["width"], L["height"]) if L else (640, 480)
        A, B, pts, _ = synth.make_klt_pair(seed=820 + k, size=size, n_points=120, max_shift=5.0)
        r = np.random.default_rng(k)
        init = [pts + r.uniform(-2, 2, pts.shape).astype(np.float32) for _ in range(3)]
        frames = [A, B, np.roll(A, 3, axis=1), np.roll(B, -2, axis=0)]
        seqs.append({"slot": slot, "lens": L, "frames": frames, "pts": pts, "init": init})
        host.append(dict(seqs[-1], frames=[host_undistort(f, L) for f in frames]))
    return seqs, host


@pytest.mark.gpu
@pytest.mark.parametrize("clahe_clip", [6.0, 0.0])
def test_tracker_and_detector_on_raw_frames_equal_host_undistortion(clahe_clip):
    seqs, host = _sequences()
    a, b = _handle(), _handle()
    try:
        set_lens(a, [dict(sq["lens"], slot=sq["slot"]) for sq in seqs if sq["lens"]])     # new slots: no tracker call yet
        for t in range(3):
            la, lb = a.kernel_launches, b.kernel_launches
            got = klt.batch_track_keypoints(a, _pairs(seqs, t, t == 0), clahe_clip=clahe_clip)
            want = klt.batch_track_keypoints(b, _pairs(host, t, t == 0), clahe_clip=clahe_clip)
            assert a.kernel_launches - la == b.kernel_launches - lb + 1, t
            for g, w in zip(got, want):
                for x, y, name in zip(g, w, ("next_pts", "status", "err", "info")):
                    assert np.array_equal(x, y), (t, name)
            assert sum(int(g[1].sum()) for g in got) > 100
            # the detector: every slot's cached newest frame, and the raw frames uploaded again
            ex = [sq["pts"][::4].astype(np.float64) for sq in seqs]
            cached = [{"slot": sq["slot"], "frame_id": t + 2, "shape": sq["frames"][0].shape, "keypoints": e}
                      for sq, e in zip(seqs, ex)]
            up_a = [{"slot": sq["slot"], "image": sq["frames"][t], "keypoints": e} for sq, e in zip(seqs, ex)]
            up_b = [{"slot": sq["slot"], "image": sq["frames"][t], "keypoints": e} for sq, e in zip(host, ex)]
            la, lb = a.kernel_launches, b.kernel_launches
            ga = batch_detect_keypoints(a, cached + up_a, clahe_clip=clahe_clip, want_gftt=True)
            gb = batch_detect_keypoints(b, cached + up_b, clahe_clip=clahe_clip, want_gftt=True)
            assert a.kernel_launches - la == b.kernel_launches - lb + 1
            for (k1, c1), (k2, c2) in zip(ga, gb):
                assert np.array_equal(k1, k2) and np.array_equal(c1, c2)
            assert all(len(c) > 0 for _, c in ga)
        # a call in which no slot has a lens launches what the same call launches on a handle without lenses
        plain = [sq for sq in seqs if sq["lens"] is None]
        la, lb = a.kernel_launches, b.kernel_launches
        pairs = [{"slot": sq["slot"], "prev_id": 4, "next_id": 5, "prev": None, "next": sq["frames"][0], "pts": sq["pts"]}
                 for sq in plain]
        ga = klt.batch_track_keypoints(a, pairs, clahe_clip=clahe_clip)
        gb = klt.batch_track_keypoints(b, pairs, clahe_clip=clahe_clip)
        assert a.kernel_launches - la == b.kernel_launches - lb
        for g, w in zip(ga, gb):
            assert all(np.array_equal(x, y) for x, y in zip(g, w))
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_set_lens_drops_the_cache_and_clearing_restores_raw_frames():
    A, B, pts, _ = synth.make_klt_pair(seed=840, size=(752, 480), n_points=80)
    a, b = _handle(), _handle()
    try:
        klt.batch_track_keypoints(a, [{"slot": 4, "prev_id": 1, "next_id": 2, "prev": A, "next": B, "pts": pts}], clahe_clip=6.0)
        set_lens(a, [dict(EUROC, slot=4)])
        cp, outs, keep = klt.pack_pairs([{"slot": 4, "prev_id": 2, "next_id": 3, "prev": None, "next": A, "pts": pts}])
        assert a.lib.pvio_b200_batch_track_keypoints(a.h, 1, cp, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99) == EINVAL
        cr, douts, dkeep = pack_requests([{"slot": 4, "frame_id": 2, "shape": A.shape}])
        assert a.lib.pvio_b200_batch_detect_keypoints(a.h, 1, cr, 6.0, 8, 8) == EINVAL
        # cleared: uploaded frames are used as they are
        set_lens(a, [{"slot": 4, "model": NONE}])
        pair = {"slot": 4, "prev_id": 7, "next_id": 8, "prev": B, "next": A, "pts": pts}
        ga = klt.batch_track_keypoints(a, [pair], clahe_clip=6.0)
        gb = klt.batch_track_keypoints(b, [pair], clahe_clip=6.0)
        assert all(np.array_equal(x, y) for x, y in zip(ga[0], gb[0]))
        with pytest.raises(Exception):                       # no lens any more
            batch_undistort(a, [{"slot": 4, "image": A}])
        del keep, dkeep
    finally:
        a.close()
        b.close()


@pytest.mark.gpu
def test_rejections_change_nothing():
    A, B, pts, _ = synth.make_klt_pair(seed=850, size=(752, 480), n_points=80)
    small = _raw(SMALL, 851)
    b = _handle()
    try:
        set_lens(b, [dict(EUROC, slot=1), dict(SMALL, slot=2)])
        first = klt.batch_track_keypoints(b, [{"slot": 1, "prev_id": 1, "next_id": 2, "prev": A, "next": B, "pts": pts}],
                                          clahe_clip=6.0)
        assert first[0][1].sum() > 0
        ref_small = batch_undistort(b, [{"slot": 2, "image": small}])[0]

        # set_lens: one bad record among good ones changes no slot (slot 2 keeps its lens, slot 1 its cache)
        good = dict(TUMVI, slot=2)
        bads = [dict(EUROC, slot=-1), dict(EUROC, slot=65536), dict(EUROC, slot=2), dict(EUROC, slot=30, model=3),
                dict(EUROC, slot=30, width=7), dict(EUROC, slot=30, K=(float("nan"), 457.0, 367.0, 248.0)),
                dict(EUROC, slot=30, K=(0.0, 457.0, 367.0, 248.0)), dict(EUROC, slot=30, K=(458.0, -1.0, 367.0, 248.0)),
                dict(TUMVI, slot=30, coeffs=(1e308, 1e308, 0.0, 0.0))]
        for bad in bads:
            assert b.lib.pvio_b200_batch_set_lens(b.h, 2, pack_lenses([good, bad])) == EINVAL, bad
        assert b.lib.pvio_b200_batch_set_lens(b.h, -1, None) == EINVAL
        assert b.lib.pvio_b200_batch_set_lens(b.h, 1, None) == EINVAL
        assert b.lib.pvio_b200_batch_set_lens(b.h, 0, None) == 0
        assert np.array_equal(batch_undistort(b, [{"slot": 2, "image": small}])[0], ref_small)

        # batch_undistort: no lens, other shape, stride, NULL pointers; the outputs stay as they were
        def und_attempt(edit):
            img = np.ascontiguousarray(small)
            out = np.full(small.shape, 77, np.uint8)
            arr = (_lib.CUndistortRequest * 1)()
            r = arr[0]
            r.slot, r.width, r.height, r.stride = 2, small.shape[1], small.shape[0], small.shape[1]
            r.src, r.dst = _lib.ptr(img), _lib.ptr(out)
            edit(r)
            assert b.lib.pvio_b200_batch_undistort(b.h, 1, arr) == EINVAL
            assert (out == 77).all()
        und_attempt(lambda r: setattr(r, "slot", 5))
        und_attempt(lambda r: setattr(r, "slot", 65536))
        und_attempt(lambda r: setattr(r, "width", 96))
        und_attempt(lambda r: setattr(r, "height", 62))
        und_attempt(lambda r: setattr(r, "stride", 90))
        und_attempt(lambda r: setattr(r, "src", None))
        und_attempt(lambda r: setattr(r, "dst", None))
        assert b.lib.pvio_b200_batch_undistort(b.h, -1, None) == EINVAL
        assert b.lib.pvio_b200_batch_undistort(b.h, 0, None) == 0

        # tracker / detector: a frame whose shape differs from its slot's lens
        A2 = synth.make_klt_pair(seed=852, size=(640, 480))[0]
        cp, outs, keep = klt.pack_pairs([{"slot": 1, "prev_id": 2, "next_id": 3, "prev": None, "next": A, "pts": pts},
                                         {"slot": 2, "prev_id": 1, "next_id": 2, "prev": A2, "next": A2, "pts": pts}])
        for o in outs:
            o[0][:] = -5.0
            o[1][:] = 9
        before = [[x.copy() for x in o] for o in outs]
        assert b.lib.pvio_b200_batch_track_keypoints(b.h, 2, cp, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99) == EINVAL
        for o, w in zip(outs, before):
            assert all(np.array_equal(x, y) for x, y in zip(o, w))
        cr, douts, dkeep = pack_requests([{"slot": 2, "image": A2}])
        douts[0][1][:] = -9
        assert b.lib.pvio_b200_batch_detect_keypoints(b.h, 1, cr, 6.0, 8, 8) == EINVAL
        assert (douts[0][1] == -9).all()
        # nothing changed: slot 1 still tracks from its cached frame 2
        nxt = klt.batch_track_keypoints(b, [{"slot": 1, "prev_id": 2, "next_id": 3, "prev": None, "next": A, "pts": pts}],
                                        clahe_clip=6.0)
        assert nxt[0][1].sum() > 0
        del keep, dkeep
    finally:
        b.close()
