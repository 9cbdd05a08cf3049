"""pvio_b200_batch_feature_track: the per-frame step of FeatureTracker::work for many sequences, with each slot's
keypoints kept on the device.  Every frame's keypoints, prev_index, counts and info must equal, bit for bit, a chain
driven from the host over the calls the step is built from: the guesses in numpy (oracle/feature_oracle.py),
pvio_b200_batch_track_keypoints, libstdc++'s std::sort and the Poisson filter on the host, then
pvio_b200_batch_detect_keypoints with the survivors, and the append."""
import numpy as np
import pytest

from oracle import feature_oracle as fo
from pvio_b200 import klt
from pvio_b200._lib import EINVAL
from pvio_b200.detect import batch_detect_keypoints
from pvio_b200.feature_track import batch_feature_track
from pvio_b200.undistort import RADTAN, set_lens

cv2 = pytest.importorskip("cv2")
Rotation = pytest.importorskip("scipy.spatial.transform").Rotation

KD = 20.0
CLIP = 6.0
EUROC = {"model": RADTAN, "width": 752, "height": 480, "K": (458.654, 457.296, 367.215, 248.375),
         "coeffs": (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05)}
LENS_SLOT = 5


def _handle():
    from pvio_b200.bundle_adjustor import BundleAdjustor
    return BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)


def render(seed, n_frames, shape, fast=(), flat=()):
    """A textured plane seen by a rotating camera with a little translation: (frames, predict_q per frame, K).
    Frames in `fast` turn ten times faster (tracks leave at the border); frames in `flat` are uniform grey."""
    h, w = shape
    rng = np.random.default_rng(seed)
    tex = cv2.GaussianBlur(rng.integers(0, 256, (3 * h, 3 * w)).astype(np.float32), (0, 0), 1.6)
    tex = cv2.normalize(tex, None, 0, 255, cv2.NORM_MINMAX).astype(np.uint8)
    K = (0.6 * w + seed % 7, 0.6 * w - seed % 5, w / 2 - 0.5, h / 2 + 0.25)
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    T = np.array([[1, 0, -w], [0, 1, -h], [0, 0, 1.0]])
    frames, qs, R = [], [], np.eye(3)
    for k in range(n_frames):
        Rk = Rotation.from_rotvec(rng.normal(0, 0.05 if k in fast else 0.005, 3)).as_matrix()
        R = Rk @ R
        qs.append(Rotation.from_matrix(Rk).as_quat())
        H = Km @ R @ np.linalg.inv(Km) @ T
        H[:2, 2] += rng.normal(0, 0.4, 2)
        img = cv2.warpPerspective(tex, H, (w, h), flags=cv2.INTER_LINEAR)
        frames.append(np.full_like(img, 128) if k in flat else img)
    return frames, qs, K


def map_frames(k, restart=None):
    """the map's frame count before frame k is put: a cap of 60 that drops to 20 at frame 12"""
    if restart is not None and k >= restart:
        k -= restart
    return 0 if k == 0 else min(k, 60 if k <= 12 else 20)


class Chain:
    """One sequence driven from the host over the tracker and detector calls of handle `ba`, slot `slot`"""

    def __init__(self, ba, slot, K):
        self.ba, self.slot, self.K = ba, slot, K
        self.z = np.zeros((0, 2))
        self.prev_index = np.zeros(0, np.int32)
        self.birth = np.zeros(0, np.int32)
        self.no, self.fid, self.img = 0, 0, None

    def step(self, img, fid, mf, q):
        K, h, w = self.K, img.shape[0], img.shape[1]
        counts, info = [0, 0, 0, 0], np.array([0, -1, -1, 0], np.int32)
        z, prev, birth = np.zeros((0, 2)), [], []
        prev_no = self.no if mf > 0 else self.no + 1
        if mf > 0:
            p0, p1 = fo.guesses(self.z, K, K, q)
            (nxt, st, _, info), = klt.batch_track_keypoints(
                self.ba, [{"slot": self.slot, "prev_id": self.fid, "next_id": fid, "prev": self.img, "next": img,
                           "pts": p0, "init": p1}], clahe_clip=CLIP)
            st = st.astype(bool)
            counts[1] = int(st.sum())
            length = np.minimum(prev_no - self.birth + 1, mf)
            st = fo.thin(nxt, st, self.prev_index != -1, length, KD)
            keep = np.nonzero(st)[0]
            counts[2] = len(keep)
            z = fo.remove_k(nxt[keep].astype(np.float64), K)
            prev, birth = list(keep), list(self.birth[keep])
        (det,) = batch_detect_keypoints(self.ba, [{"slot": self.slot, "frame_id": fid, "image": img,
                                                   "keypoints": fo.apply_k(z, K), "keypoint_distance": KD}],
                                        clahe_clip=CLIP)
        counts[3] = len(det)
        self.z = np.concatenate([z, fo.remove_k(det, K)])
        self.prev_index = np.array(prev + [-1] * len(det), np.int32)
        self.birth = np.array(birth + [prev_no + 1] * len(det), np.int32)
        self.no, self.fid, self.img = prev_no + 1, fid, img
        return {"keypoints": self.z, "prev_index": self.prev_index, "counts": counts, "info": info}


def _seqs():
    """8 sequences: EuRoC and TUM-VI shapes, slot 5 with a lens, no prediction for sequence 3, sequence 6 restarts
    at frame 10, sequence 7 loses every point at frame 9 (two flat frames: LK has no gradient to work with)"""
    out = []
    for i in range(8):
        shape = (480, 752) if i % 2 == 0 or i == LENS_SLOT else (512, 512)
        frames, qs, K = render(100 + i, 26, shape, fast=(7, 16) if i % 3 == 0 else (11,), flat=(8, 9) if i == 7 else ())
        out.append({"slot": i, "frames": frames, "qs": qs, "K": K, "predict": i != 3, "restart": 10 if i == 6 else None})
    return out


def _request(sq, k, slot=None, fid_base=0):
    return {"slot": sq["slot"] if slot is None else slot, "frame_id": fid_base + k + 1, "image": sq["frames"][k],
            "K": sq["K"], "map_frames": map_frames(k, sq["restart"]), "predict_q": sq["qs"][k] if sq["predict"] else None}


def _same(got, want, where):
    assert np.array_equal(got["keypoints"], want["keypoints"]), where
    assert np.array_equal(got["prev_index"], want["prev_index"]), where
    assert np.array_equal(got["info"], want["info"]), where
    assert list(got["counts"][1:]) == list(want["counts"][1:]), where
    assert got["counts"][0] >= got["counts"][1], where


@pytest.mark.gpu
def test_chain_equality_batch_independence_and_edges():
    seqs = _seqs()
    dev, ref, one, big = _handle(), _handle(), _handle(), _handle()
    try:
        for b in (dev, ref):
            set_lens(b, [dict(EUROC, slot=LENS_SLOT)])
        set_lens(big, [dict(EUROC, slot=s) for s in range(LENS_SLOT, 264, 8)])
        chains = [Chain(ref, sq["slot"], sq["K"]) for sq in seqs]
        got8 = []
        for k in range(26):
            reqs = [_request(sq, k) for sq in seqs]
            l0 = dev.kernel_launches
            res = batch_feature_track(dev, reqs, keypoint_distance=KD, clahe_clip=CLIP)
            if k == 3:
                launches8 = dev.kernel_launches - l0
            got8.append(res)
            for i, sq in enumerate(seqs):
                want = chains[i].step(sq["frames"][k], k + 1, reqs[i]["map_frames"], reqs[i]["predict_q"])
                _same(res[i], want, (k, i))
        # the edge cases really happened: tracks lost at the border, a restart, a sequence that lost every point
        assert any(got8[k][0]["counts"][0] < len(got8[k - 1][0]["keypoints"]) for k in (7, 16))
        assert np.all(got8[10][6]["prev_index"] == -1) and got8[10][6]["counts"][3] > 0
        assert got8[9][7]["counts"][0] == 0 and len(got8[9][7]["keypoints"]) == 0
        assert len(got8[10][7]["keypoints"]) > 0 and np.all(got8[10][7]["prev_index"] == -1)
        assert any(r["counts"][2] < r["counts"][1] for res in got8 for r in res)      # the thinning acts

        # batch independence: sequence 0 alone (with batch_track / batch_detect calls on other slots between its
        # frames), and 264 sequences (33 copies of the 8, more than one wave)
        other, _, _ = render(900, 6, (480, 752))
        for k in range(6):
            (r1,) = batch_feature_track(one, [_request(seqs[0], k)], keypoint_distance=KD, clahe_clip=CLIP)
            _same(r1, got8[k][0], ("alone", k))
            klt.batch_track_keypoints(one, [{"slot": 40, "prev_id": 7 + k, "next_id": 8 + k, "prev": other[k],
                                             "next": other[(k + 1) % 6], "pts": np.full((50, 2), 100, np.float32)}],
                                      clahe_clip=CLIP)
            batch_detect_keypoints(one, [{"slot": 40, "frame_id": 8 + k, "shape": (480, 752)},
                                         {"slot": 41, "image": other[k]}], clahe_clip=CLIP)
        for k in range(5):
            reqs = [_request(seqs[s % 8], k, slot=s) for s in range(264)]
            l0 = big.kernel_launches
            res = batch_feature_track(big, reqs, keypoint_distance=KD, clahe_clip=CLIP)
            if k == 3:
                assert big.kernel_launches - l0 == launches8
            for s in range(264):
                _same(res[s], got8[k][s % 8], ("264", k, s))

        # an evicted previous frame: the call is rejected and changes no slot
        klt.batch_track_keypoints(dev, [{"slot": 2, "prev_id": 5001, "next_id": 5002, "prev": other[0], "next": other[1],
                                         "pts": np.zeros((0, 2), np.float32)}], clahe_clip=CLIP)
        f26, q26, _ = render(100 + 1, 28, (512, 512), fast=(11,))
        extra = dict(_request(seqs[1], 25), frame_id=27, image=f26[26], map_frames=20, predict_q=q26[26])
        n0 = dev.kernel_launches
        with pytest.raises(RuntimeError):
            batch_feature_track(dev, [extra, dict(_request(seqs[2], 25), frame_id=27, map_frames=20)],
                                keypoint_distance=KD, clahe_clip=CLIP)
        assert dev.kernel_launches == n0
        (r,) = batch_feature_track(dev, [extra], keypoint_distance=KD, clahe_clip=CLIP)
        _same(r, chains[1].step(f26[26], 27, 20, q26[26]), "after a rejected call")
    finally:
        for b in (dev, ref, one, big):
            b.close()


@pytest.mark.gpu
def test_rejections_on_the_device():
    frames, qs, K = render(7, 2, (480, 752))
    b = _handle()
    try:
        req = {"slot": 0, "frame_id": 1, "image": frames[0], "K": K, "map_frames": 0}
        lib = b.lib
        from pvio_b200.feature_track import pack_frames
        for bad in ([req, dict(req)],                                       # a slot twice
                    [dict(req, map_frames=1)],                              # nothing cached in the slot
                    [dict(req, max_keypoints=100)]):                        # below the bound
            cf, _, keep = pack_frames(bad, KD)
            assert lib.pvio_b200_batch_feature_track(b.h, len(bad), cf, 3, 30, 0.01, CLIP, 8, 8, 20, 1.0, 0.99, KD) == EINVAL
        batch_feature_track(b, [req], keypoint_distance=KD, clahe_clip=CLIP)
        cf, _, keep = pack_frames([dict(req, map_frames=1)], KD)           # the slot's newest frame id again
        assert lib.pvio_b200_batch_feature_track(b.h, 1, cf, 3, 30, 0.01, CLIP, 8, 8, 20, 1.0, 0.99, KD) == EINVAL
        (r,) = batch_feature_track(b, [dict(req, frame_id=2, image=frames[1], map_frames=1, predict_q=qs[1])],
                                   keypoint_distance=KD, clahe_clip=CLIP)
        assert r["counts"][0] > 0 and np.all(r["prev_index"][:r["counts"][2]] >= 0)
    finally:
        b.close()
