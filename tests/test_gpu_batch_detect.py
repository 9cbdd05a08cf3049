"""pvio_b200_batch_detect_keypoints: OpenCvImage::detect_keypoints (opencv_image.cpp:54-86) for many frames in one call,
on the frames the batched tracker keeps in its slots or on uploaded pixels.  Every request must equal, bit for bit,
what pvio_b200_detect_keypoints gives for that frame on a handle of its own: the keypoints and the GFTT corners, both
in order.  The single call runs the two greedy passes on the host, so it checks the device passes independently."""
import ctypes as C

import numpy as np
import pytest

from pvio_b200 import _lib, klt
from pvio_b200.detect import batch_detect_keypoints, detect_keypoints, pack_requests
from pvio_b200._lib import EINVAL
from synthetic import synth



def test_detect_request_layout_matches_header():
    R = _lib.CDetectRequest
    assert C.sizeof(R) == 88
    offsets = {"slot": 0, "width": 4, "height": 8, "stride": 12, "frame_id": 16, "image": 24, "existing": 32,
               "n_existing": 40, "max_out": 44, "keypoint_distance": 48, "keypoints_out": 56, "n_out": 64,
               "gftt_out": 72, "n_gftt": 80}
    assert {k: getattr(R, k).offset for k in offsets} == offsets


def _handle():
    from pvio_b200.bundle_adjustor import BundleAdjustor
    return BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)


def _single(img, existing, kd, clahe_clip, frame_id=0, shape=None, ref=None):
    """pvio_b200_detect_keypoints on a fresh handle (or `ref`): (keypoints, corners)"""
    own = ref is None
    ref = _handle() if own else ref
    try:
        return detect_keypoints(ref, img, existing, keypoint_distance=kd, clahe_clip=clahe_clip, frame_id=frame_id,
                                shape=shape, want_gftt=True)
    finally:
        if own:
            ref.close()


def _existing(rng, n, w, h):
    """n existing keypoints over the frame and up to 60 px beyond it, a few far outside"""
    if n == 0:
        return np.zeros((0, 2))
    e = np.stack([rng.uniform(-60, w + 60, n), rng.uniform(-60, h + 60, n)], 1)
    e[:3] = [[-1e6, 10.0], [w + 5e3, h / 2], [w / 2, -7.5]]
    return e


def _frames(clahe_clip):
    """14 frames: three shapes, 0 / 120 / 600 existing points, radius 10 / 25 / 40, a flat frame"""
    shapes = [(752, 480), (512, 512), (160, 120)]
    out = []
    for i in range(13):
        size = shapes[i % 3]
        A, B, _, _ = synth.make_klt_pair(seed=1200 + i, size=size)
        img = A if i % 2 == 0 else B
        out.append({"img": img, "n_ex": [0, 120, 600][(i + i // 3) % 3], "kd": [10.0, 25.0, 40.0][(i // 3) % 3]})
    out.append({"img": np.full((120, 160), 128, np.uint8), "n_ex": 120, "kd": 25.0})
    rng = np.random.default_rng(int(clahe_clip) + 5)
    for f in out:
        h, w = f["img"].shape
        if clahe_clip == 0.0:
            f["img"] = _clahe(f["img"])
        f["ex"] = _existing(rng, f["n_ex"], w, h)
    return out


def _clahe(img):
    b = _handle()
    try:
        return klt.clahe(b, img)
    finally:
        b.close()


@pytest.mark.gpu
@pytest.mark.parametrize("clahe_clip", [6.0, 0.0])
def test_batch_equals_single_calls(clahe_clip):
    frames = _frames(clahe_clip)
    want = [_single(f["img"], f["ex"], f["kd"], clahe_clip) for f in frames]
    assert any(len(w[0]) > 100 for w in want) and len(want[-1][1]) == 0
    assert any(0 < len(w[0]) < len(w[1]) for w in want)          # the Poisson filter and the border remove corners
    order = np.random.default_rng(11).permutation(len(frames))
    b = _handle()
    try:
        reqs = [{"slot": int(k), "image": frames[k]["img"], "keypoints": frames[k]["ex"], "keypoint_distance": frames[k]["kd"]}
                for k in order]
        got = batch_detect_keypoints(b, reqs, clahe_clip=clahe_clip, want_gftt=True)
        for j, k in enumerate(order):
            assert np.array_equal(got[j][0], want[k][0]), ("keypoints", k)
            assert np.array_equal(got[j][1], want[k][1]), ("corners", k)
        again = batch_detect_keypoints(b, reqs, clahe_clip=clahe_clip, want_gftt=True)     # reused scratch
        assert all(np.array_equal(g[0], a[0]) and np.array_equal(g[1], a[1]) for g, a in zip(got, again))
    finally:
        b.close()


def _track_pair(slot, prev_id, next_id, prev, nxt, pts):
    return {"slot": slot, "prev_id": prev_id, "next_id": next_id, "prev": prev, "next": nxt, "pts": pts}


@pytest.mark.gpu
def test_detect_through_the_slot_caches():
    import cv2
    from oracle import detect_oracle as D
    seqs = []
    for s in range(5):
        size = [(752, 480), (512, 512), (160, 120)][s % 3]
        A, B, pts, _ = synth.make_klt_pair(seed=1300 + s, size=size, n_points=200)
        _, Cn, _, _ = synth.make_klt_pair(seed=1310 + s, size=size, n_points=200)
        seqs.append((A, B, Cn, pts))
    slots = [3, 17, 0, 9, 40]
    b, control = _handle(), _handle()
    try:
        single0 = klt.track_keypoints(b, seqs[0][0], seqs[0][1], seqs[0][3], prev_id=1, next_id=2, clahe_clip=6.0)
        for hnd in (b, control):
            klt.batch_track_keypoints(hnd, [_track_pair(slots[k], 1, 2, A, B, pts) for k, (A, B, _, pts) in enumerate(seqs)],
                                      clahe_clip=6.0)
        rng = np.random.default_rng(4)
        reqs, want = [], []
        for k, (A, B, _, pts) in enumerate(seqs):
            h, w = A.shape
            for fid, img in ((2, B), (1, A)) if k % 2 == 0 else ((2, B),):
                ex = pts[::3].astype(np.float64)
                reqs.append({"slot": slots[k], "frame_id": fid, "image": None, "shape": (h, w), "keypoints": ex,
                             "keypoint_distance": 25.0})
                want.append((_single(img, ex, 25.0, 6.0), img))
        got = batch_detect_keypoints(b, reqs, clahe_clip=6.0, want_gftt=True)
        for (kp, corners), ((wkp, wc), img) in zip(got, want):
            assert np.array_equal(kp, wkp) and np.array_equal(corners, wc)
            ref = D.gftt(cv2.createCLAHE(6.0, (8, 8)).apply(img))
            assert set(map(tuple, ref.astype(int))) == set(map(tuple, corners.astype(int)))
            assert len(kp) > 0
        # no cache changed: the next tracker step equals the control handle's, which ran no detection
        step = [_track_pair(slots[k], 2, 3, None, Cn, pts) for k, (_, _, Cn, pts) in enumerate(seqs)]
        g = klt.batch_track_keypoints(b, step, clahe_clip=6.0)
        c = klt.batch_track_keypoints(control, step, clahe_clip=6.0)
        for x, y in zip(g, c):
            assert all(np.array_equal(u, v) for u, v in zip(x, y))
        # the single calls' cache still holds frame 2 of the single-call sequence
        A, B, _, pts = seqs[0]
        kp = detect_keypoints(b, None, pts[::3], keypoint_distance=25.0, clahe_clip=6.0, frame_id=2, shape=B.shape)
        assert np.array_equal(kp, _single(B, pts[::3], 25.0, 6.0)[0])
        assert len(single0[0]) == len(pts)
    finally:
        b.close()
        control.close()


@pytest.mark.gpu
def test_batch_beyond_one_wave():
    """264 frames tiled from 8 seeds, uploaded raw with device CLAHE: staging growth and every per-frame offset."""
    rng = np.random.default_rng(21)
    seeds = []
    for s in range(8):
        size = (752, 480) if s % 2 == 0 else (512, 512)
        A, _, _, _ = synth.make_klt_pair(seed=1400 + s, size=size)
        ex = _existing(rng, 150 + 20 * s, size[0], size[1])
        seeds.append((A, ex, _single(A, ex, 25.0, 6.0)))
    b = _handle()
    try:
        reqs = [{"slot": i, "image": seeds[i % 8][0], "keypoints": seeds[i % 8][1]} for i in range(264)]
        got = batch_detect_keypoints(b, reqs, clahe_clip=6.0, want_gftt=True)
        for i in range(264):
            assert np.array_equal(got[i][0], seeds[i % 8][2][0]) and np.array_equal(got[i][1], seeds[i % 8][2][1]), i
    finally:
        b.close()


@pytest.mark.gpu
def test_launch_count_does_not_grow_with_the_batch():
    A, B, pts, _ = synth.make_klt_pair(seed=1500)
    b = _handle()
    try:
        klt.batch_track_keypoints(b, [_track_pair(s, 1, 2, A, B, pts) for s in range(64)], clahe_clip=6.0)
        counts = []
        for slots in ([0], [1, 2], list(range(64))):
            l0 = b.kernel_launches
            got = batch_detect_keypoints(b, [{"slot": s, "frame_id": 2, "shape": B.shape, "keypoints": pts[::4]} for s in slots],
                                         clahe_clip=6.0)
            counts.append(b.kernel_launches - l0)
            assert all(np.array_equal(g, got[0]) for g in got) and len(got[0]) > 0
        assert counts[0] == counts[1] == counts[2] and counts[0] <= 4, counts
        l0 = b.kernel_launches
        assert b.lib.pvio_b200_batch_detect_keypoints(b.h, 0, None, 6.0, 8, 8) == 0
        assert b.kernel_launches == l0
    finally:
        b.close()


@pytest.mark.gpu
def test_rejected_calls_change_nothing():
    A, B, pts, _ = synth.make_klt_pair(seed=1600)
    b = _handle()
    try:
        klt.batch_track_keypoints(b, [_track_pair(0, 1, 2, A, B, pts)], clahe_clip=6.0)
        odd = synth.make_klt_pair(seed=1601, size=(100, 100))[0]        # not a multiple of the 8 x 8 tile grid

        def reqs():
            return [{"slot": 0, "frame_id": 2, "shape": B.shape, "keypoints": pts[::4]},
                    {"slot": 5, "image": A, "keypoints": pts[::5]}]

        def attempt(edit, clahe_clip=6.0, tiles=(8, 8), requests=None):
            cr, outs, keep = pack_requests(requests or reqs(), want_gftt=True)
            for out, cnt, gftt in outs:
                out[:] = -3.0
                cnt[:] = -9
                gftt[:] = -4.0
            before = [[a.copy() for a in o] for o in outs]
            edit(cr)
            rc = b.lib.pvio_b200_batch_detect_keypoints(b.h, 2, cr, clahe_clip, tiles[0], tiles[1])
            assert rc == EINVAL
            for o, w in zip(outs, before):
                assert all(np.array_equal(x, y) for x, y in zip(o, w))
            del keep

        def setf(field, value, i=1):
            return lambda cr: setattr(cr[i], field, value)
        attempt(setf("slot", -1))
        attempt(setf("slot", 65536))
        attempt(setf("width", 7))
        attempt(setf("height", 4, 0))
        attempt(setf("stride", 700))
        attempt(setf("n_existing", -1))
        attempt(setf("existing", None))
        attempt(setf("keypoints_out", None))
        attempt(setf("n_out", None, 0))
        attempt(setf("max_out", -1))
        attempt(setf("keypoint_distance", 0.0))
        attempt(setf("keypoint_distance", -25.0, 0))
        attempt(setf("frame_id", 3, 0))                                  # not cached in its slot, no pixels
        attempt(setf("slot", 1, 0))                                      # frame 2 is cached in slot 0 only
        attempt(lambda cr: None, clahe_clip=-1.0)
        attempt(lambda cr: None, requests=[reqs()[0], {"slot": 5, "image": odd}])
        attempt(lambda cr: None, tiles=(0, 8))
        assert b.lib.pvio_b200_batch_detect_keypoints(b.h, -1, None, 6.0, 8, 8) == EINVAL
        assert b.lib.pvio_b200_batch_detect_keypoints(b.h, 1, None, 6.0, 8, 8) == EINVAL
        # an uploaded frame without CLAHE needs no tile grid, and a cached one none at all
        ok = batch_detect_keypoints(b, [{"slot": 5, "image": odd}], clahe_clip=0.0, clahe_tiles=(0, 0))
        assert np.array_equal(ok[0], _single(odd, (), 25.0, 0.0)[0])
        # a too-small max_out: the first max_out keypoints, the full count, EINVAL -- as the single call
        full = batch_detect_keypoints(b, reqs(), clahe_clip=6.0)
        assert len(full[0]) > 10 and len(full[1]) > 10
        small = [dict(r, max_out=m) for r, m in zip(reqs(), (5, 4096))]
        cr, outs, keep = pack_requests(small)
        assert b.lib.pvio_b200_batch_detect_keypoints(b.h, 2, cr, 6.0, 8, 8) == EINVAL
        assert outs[0][1][0] == len(full[0]) and np.array_equal(outs[0][0][:5], full[0][:5])
        assert outs[1][1][0] == len(full[1]) and np.array_equal(outs[1][0][:len(full[1])], full[1])
        n = C.c_int()
        out = np.zeros((5, 2))
        rc = b.lib.pvio_b200_detect_keypoints(b.h, 0, _lib.ptr(np.ascontiguousarray(B)), B.shape[1], B.shape[0],
                                              B.shape[1], 6.0, 8, 8, _lib.ptr(np.ascontiguousarray(pts[::4], dtype=np.float64)),
                                              len(pts[::4]), 25.0, 5, _lib.ptr(out), C.byref(n), None, None)
        assert rc == EINVAL and n.value == len(full[0]) and np.array_equal(out, full[0][:5])
        del keep
    finally:
        b.close()
