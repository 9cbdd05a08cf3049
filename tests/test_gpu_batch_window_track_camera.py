"""pvio_b200_batch_window_track_camera: each sequence's new camera frame tracked with the IMU keypoint prediction made
on the device, then taken into its window slot.  Each sequence runs on slot A (tracker slot TA) with the call and on
twin slot B (tracker slot TB) with the host chain it replaces: batch_feature_track with the call's predict_q, then
mirror_frame with the same samples.  Frames are the textured plane of test_gpu_batch_feature_track.render seen by a
camera whose rotation follows the sequence's IMU samples (gyro readings scaled up on fast-turn frames), so the
prediction is what moves the keypoints.  Checked per frame, bit for bit: predict_q against oracle/delta_key_q.py on the
integrated dq, the feature outputs, every mirror_frame output, and the save blobs of (A, TA) and (B, TB).  Solves and
drops run on A, and B takes A's sequences through save / restore: a solve's or a marginalisation's last bits (the
signs of the prior's square-root rows) may depend on the slot it runs in."""
import cv2
import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from oracle import imu_oracle
from oracle.delta_key_q import delta_key_q
from pvio_b200._lib import EINVAL, IMU_DQ
from pvio_b200.batch_window import BatchWindows, Camera, Edit, Mirror
from pvio_b200.bundle_adjustor import BundleAdjustor
from pvio_b200.feature_track import batch_feature_track, min_capacity
from synthetic.sequence import Run

pytestmark = pytest.mark.gpu
KD = 30.0
SHAPE = (240, 320)
CAP = min_capacity(SHAPE[1], SHAPE[0], KD)
TA, TB, TC = 100, 200, 300
FAST = 12.0                                  # gyro scale of a fast-turn frame: turns of 10 to 20 degrees


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _state16(run, f):
    g = run.guess
    return np.concatenate([g.q[f], g.p[f], g.v[f], g.bg[f], g.ba[f]])


def render_run(run, seed, fast):
    """(frames, samples per frame, K): the camera of body rotation q_0 * dq_1 * ... * dq_k, dq_k the integration of
    frame k's samples at zero biases, the samples' gyro readings scaled by FAST on the frames in `fast`"""
    h, w = SHAPE
    rng = np.random.default_rng(seed)
    tex = cv2.GaussianBlur(rng.integers(0, 256, (3 * h, 3 * w)).astype(np.float32), (0, 0), 1.6)
    tex = cv2.normalize(tex, None, 0, 255, cv2.NORM_MINMAX).astype(np.uint8)
    K = (0.6 * w + seed % 7, 0.6 * w - seed % 5, w / 2 - 0.5, h / 2 + 0.25)
    Km = np.array([[K[0], 0, K[2]], [0, K[1], K[3]], [0, 0, 1]])
    T = np.array([[1, 0, -w], [0, 1, -h], [0, 0, 1.0]])
    cov = [np.asarray(c, dtype=np.float64).reshape(3, 3) for c in run.truth.imu_noise]
    cam = Rotation.from_quat(run.w.cam_q_cs)
    qb = Rotation.from_quat(run.truth.q[0])
    R0 = (qb * cam).as_matrix()
    frames, samples = [], [None]
    for k in range(len(run.truth.q)):
        if k > 0:
            s, t = run.truth.imu_factors[k - 1][:2]
            s = np.array(s, dtype=np.float64)
            if k in fast:
                s[:, 1:4] *= FAST
            qb = qb * Rotation.from_quat(imu_oracle.integrate(s, t, np.zeros(3), np.zeros(3), *cov)["dq"])
            samples.append((s, t))
        Rk = (qb * cam).as_matrix().T @ R0    # camera-0 rays into camera k
        frames.append(cv2.warpPerspective(tex, Km @ Rk @ np.linalg.inv(Km) @ T, (w, h), flags=cv2.INTER_LINEAR))
    return frames, samples, K


class Seq:
    def __init__(self, j, a, b, F, seed, fast=()):
        self.j, self.a, self.b, self.ta, self.tb, self.tc = j, a, b, TA + j, TB + j, TC + j
        self.run = Run(F=F, N=6, M=40, seed=seed)
        self.frames, self.samples, self.K = render_run(self.run, seed, fast)
        self.run.w.K_fx, self.run.w.K_fy = self.K[0], self.K[1]      # one Frame::K for the tracker and the window
        self.f, self.newest_kf, self.skipped, self.tk = 0, True, 0, {}

    def feature(self, tracker, q=None):
        return dict(slot=tracker, frame_id=self.f + 1, image=self.frames[self.f], K=self.K, map_frames=min(self.f, 20),
                    max_keypoints=CAP, predict_q=q)

    def imu(self):
        s, t = self.samples[self.f]
        return s, t, self.run.truth.imu_noise

    def camera(self, given=None, **kw):
        samples, t_end, noise = self.imu()
        c = Camera(self.a, self.ta, self.f + 1, self.frames[self.f], self.K, min(self.f, 20), samples, t_end, noise,
                   True, given)
        for k, v in kw.items():
            setattr(c, k, v)
        return c


def _start(bw, seqs, extra=()):
    """the first frame in both tracker slots (and the `extra` ones), one-frame windows with a track per keypoint, linked"""
    for s in seqs:
        for tr in extra:
            batch_feature_track(bw.ba, [s.feature(tr + s.j)], keypoint_distance=KD)
        for slot, tr in ((s.a, s.ta), (s.b, s.tb)):
            z = batch_feature_track(bw.ba, [s.feature(tr)], keypoint_distance=KD)[0]["keypoints"]
            bw.reset(slot, s.run.w)
            e = Edit(slot).frame(_state16(s.run, 0))
            e.new = [(0, q, 1.0) for q in z]
            ids = bw.edit([e])[0]
            s.tk = {int(i): k for k, i in enumerate(ids)}
            bw.set_keypoints(slot, tr, 1, s.tk)


def _same_blobs(bw, seqs, k):
    A = bw.save([s.a for s in seqs], [s.ta for s in seqs])
    B = bw.save([s.b for s in seqs], [s.tb for s in seqs])
    for j, (x, y) in enumerate(zip(A, B)):
        assert x == y, f"frame {k}, sequence {j}: the save blobs differ"


def _take_a(bw, seqs):
    """B takes A's sequences (window and tracker slot)"""
    bw.restore([s.b for s in seqs], bw.save([s.a for s in seqs], [s.ta for s in seqs]), [s.tb for s in seqs])


def _twin_step(bw, seqs, outs, given=None):
    """the host chain on the twins with the call's predict_q; checks every output bit for bit"""
    ft = batch_feature_track(bw.ba, [s.feature(s.tb, o["predict_q"]) for s, o in zip(seqs, outs)], keypoint_distance=KD)
    recs = []
    for s in seqs:
        samples, t_end, noise = s.imu()
        recs.append(Mirror(s.b, s.tb, samples, t_end, noise, s.K[2], s.K[3], True, (given or {}).get(s.j)))
    mo = bw.mirror_frame(recs, CAP)
    for o, f, m in zip(outs, ft, mo):
        n = o["n_keypoints"]
        assert n == len(f["keypoints"])
        assert np.array_equal(_bits(o["keypoints"]), _bits(f["keypoints"]))
        assert np.array_equal(o["prev_index"], f["prev_index"])
        assert np.array_equal(o["feature_counts"], f["counts"]) and np.array_equal(o["info"], f["info"])
        assert np.array_equal(o["kp_track"][:n], m["kp_track"][:n]) and np.array_equal(o["counts"], m["counts"])
        for key in ("state", "predicted", "imu_record"):
            assert np.array_equal(_bits(o[key]), _bits(m[key])), key
        for key in ("keyframe", "n_parallax", "skipped_frames"):
            assert o[key] == m[key], key
        assert np.array_equal(_bits([o["parallax"]]), _bits([m["parallax"]]))
        assert o["summary"]["iterations"] == m["summary"]["iterations"]


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=16, max_frames=9, max_landmarks=4096, max_obs=16384)
    yield b
    b.close()


def test_call_equals_the_host_chain_on_twins(ba):
    """8 inertial sequences over 22 frames: keyframe solves, a prune edit, drops, forced non-keyframes, given points and
    fast turns, bit for bit against the host chain; on the fast turns the prediction keeps more points through LK and
    F-RANSAC than the same frames tracked without it (tracker slots TC)"""
    bw = BatchWindows(ba)
    fast = (7, 13, 18)
    seqs = [Seq(j, j, 8 + j, 24, 1200 + j, fast) for j in range(8)]
    _start(bw, seqs, extra=(TC,))
    kf_checked = replaced = dropped = solved = n_given = 0
    lk_pred = lk_plain = 0
    for k in range(22):
        for s in seqs:
            s.f += 1
        given = {}
        if k in (3, 4, 9, 15):                   # given (plane-cast) points for a few tracks of the newest frame
            for s in seqs:
                given[s.j] = {t: np.array([0.05 * t, -0.1, 2.5]) for t in sorted(s.tk)[1::9][:5]}
                n_given += len(given[s.j])
        was_kf = [s.newest_kf for s in seqs]
        outs = bw.track_camera([s.camera(given.get(s.j)) for s in seqs], CAP, keypoint_distance=KD)
        plain = batch_feature_track(ba, [s.feature(s.tc) for s in seqs], keypoint_distance=KD)
        for s, o, kf, p in zip(seqs, outs, was_kf, plain):
            if kf:                               # the step-1 record is the edit's: its dq made predict_q
                want = delta_key_q(s.run.w.cam_q_cs, s.run.w.imu_q_cs, o["imu_record"][IMU_DQ:IMU_DQ + 4])
                assert np.array_equal(_bits(o["predict_q"]), _bits(want))
                kf_checked += 1
            else:
                replaced += 1
            if s.f in fast:                      # kept after LK, the border test and F-RANSAC
                lk_pred += int(o["feature_counts"][1])
                lk_plain += int(p["counts"][1])
        _twin_step(bw, seqs, outs, given)
        for s, o in zip(seqs, outs):
            s.newest_kf, s.skipped = o["keyframe"], o["skipped_frames"]
            s.tk = {int(t): kj for kj, t in enumerate(o["kp_track"][:o["n_keypoints"]]) if t >= 0}
        _same_blobs(bw, seqs, k)
        if k == 6:                               # a prune edit on both: removal only, the link stays
            for s in seqs:
                ids = [int(i) for i in bw.download([s.a], 4096)[0]["ids"][::7][:5]]
                for slot in (s.a, s.b):
                    e = Edit(slot)
                    e.remove = ids
                    bw.edit([e])
                s.tk = {t: kj for t, kj in s.tk.items() if t not in ids}
        took = False
        if k % 4 == 1:                           # a keyframe solve: the next prediction starts from its state
            bw.solve([s.a for s in seqs], max_iterations=3)
            solved += 1
            took = True
        full = [s for s in seqs if s.newest_kf and bw.download([s.a], 4096)[0]["frames"].shape[0] >= 6]
        if full:
            bw.drop_victim([s.a for s in full])
            dropped += len(full)
            took = True
        if took:
            _take_a(bw, seqs)
        if k % 4 == 2:                           # force a non-keyframe: the next frame replaces it
            for s in seqs:
                if s.newest_kf and s not in full:
                    d = bw.download([s.a], 4096)[0]
                    if d["frames"].shape[0] >= 2:
                        s.newest_kf = False
                        live = set(int(i) for i in d["ids"])
                        pairs = {t: kj for t, kj in s.tk.items() if t in live}
                        for slot, tr in ((s.a, s.ta), (s.b, s.tb)):
                            bw.set_keypoints(slot, tr, s.f + 1, pairs, False, s.skipped)
        _same_blobs(bw, seqs, k)
    print(f"predict_q checked {kf_checked}, replaced {replaced}, dropped {dropped}, solves {solved}, "
          f"given points {n_given}, kept after F-RANSAC on fast turns: {lk_pred} predicted, {lk_plain} not")
    assert kf_checked > 0 and replaced > 0 and dropped > 0 and solved > 0 and n_given > 0
    assert lk_pred > lk_plain


def _call_rejected(bw, seqs, recs):
    """a rejected call: EINVAL, no output written, every named slot's blob (window and tracker) unchanged"""
    before = bw.save([s.a for s in seqs], [s.ta for s in seqs])
    r, sms, out, keep = BatchWindows.camera_records(recs, CAP)
    assert bw.lib.pvio_b200_batch_window_track_camera(bw.h, len(recs), r, 3, 30, 0.01, 6.0, 8, 8, 20, 1.0, 0.99, KD,
                                                      None) == EINVAL
    for o in out:
        assert np.all(o["kp_track"] == -7) and np.all(o["keypoints"] == -7.0) and np.all(o["prev_index"] == -7)
        assert o["n_keypoints"][0] == -7 and not o["state"].any() and not o["predict_q"].any()
        assert not o["predicted"].any() and not o["feature_counts"].any() and not o["counts"].any()
    assert bw.save([s.a for s in seqs], [s.ta for s in seqs]) == before


def test_rejections_change_nothing_and_the_next_call_is_unaffected(ba):
    """every rejection, after several tracked frames (the tracker slots hold a previous frame), leaves both slots and
    the outputs as they were, and the next call equals the host chain"""
    bw = BatchWindows(ba)
    seqs = [Seq(j, j, 8 + j, 8, 1300 + j) for j in range(2)]
    _start(bw, seqs)
    for _ in range(3):
        for s in seqs:
            s.f += 1
        outs = bw.track_camera([s.camera() for s in seqs], CAP, keypoint_distance=KD)
        _twin_step(bw, seqs, outs)
        for s, o in zip(seqs, outs):
            s.tk = {int(t): kj for kj, t in enumerate(o["kp_track"][:o["n_keypoints"]]) if t >= 0}
    a, b = seqs
    a.f = b.f = a.f + 1
    call = lambda recs: _call_rejected(bw, seqs, recs)                 # noqa: E731
    call([a.camera(map_frames=0)])                                     # a sequence start
    call([a.camera(K=(a.K[0] * 1.01,) + tuple(a.K[1:]))])              # fx not the slot's
    call([a.camera(tracker_slot=b.ta)])                                # not the link's tracker slot
    call([a.camera(), a.camera()])                                     # a slot named twice
    call([a.camera(), b.camera(slot=a.a)])
    call([a.camera(samples=np.zeros((0, 7)))])                         # no samples
    call([a.camera(given={10 ** 6: np.zeros(3)})])                     # unknown given track
    call([a.camera(frame_id=a.f)])                                     # the tracker's newest frame id
    vo = Run(F=4, N=6, M=40, seed=1310).w                              # a visual-only slot
    vo.use_inertial, vo.K_fx, vo.K_fy = False, a.K[0], a.K[1]
    bw.reset(15, vo)
    bw.edit([Edit(15).frame(_state16(a.run, 0))])
    bw.set_keypoints(15, a.ta, a.f, {})
    call([a.camera(slot=15)])
    outs = bw.track_camera([s.camera() for s in seqs], CAP, keypoint_distance=KD)
    _twin_step(bw, seqs, outs)
    _same_blobs(bw, seqs, "after the rejections")


def test_capacity_found_after_the_gather_rejects_without_a_trace():
    """a handle with a small max_landmarks, after tracked frames (the tracker slot holds a previous frame): the
    candidates overflow the window after the gather; the window and tracker blob stay byte for byte, no output is
    written, and the next frame tracks on TA exactly as on its untouched twin TB"""
    small = BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=8, max_obs=64)
    try:
        bw = BatchWindows(small)
        s = Seq(0, 0, 1, 8, 1400)
        for _ in range(3):
            for tr in (s.ta, s.tb):
                batch_feature_track(small, [s.feature(tr)], keypoint_distance=KD)
            s.f += 1
        s.f -= 1
        for slot in (s.a, s.b):
            bw.reset(slot, s.run.w)
            bw.edit([Edit(slot).frame(_state16(s.run, 0))])
        bw.set_keypoints(s.a, s.ta, s.f + 1, {})
        bw.set_keypoints(s.b, s.tb, s.f + 1, {})
        s.f += 1
        before = bw.save([s.a], [s.ta])
        _call_rejected(bw, [s], [s.camera()])
        assert bw.save([s.a], [s.ta]) == before == bw.save([s.b], [s.tb])
        f = batch_feature_track(small, [s.feature(s.ta)], keypoint_distance=KD)[0]
        g = batch_feature_track(small, [s.feature(s.tb)], keypoint_distance=KD)[0]
        assert np.array_equal(_bits(f["keypoints"]), _bits(g["keypoints"])) and np.array_equal(f["prev_index"], g["prev_index"])
    finally:
        small.close()


def test_mixed_batches_and_launches():
    """a record gives the same bits alone, in a batch of 8 and in a batch of 264; the launches at n = 8 and n = 264
    are equal"""
    big = BundleAdjustor(max_windows=540, max_frames=4, max_landmarks=512, max_obs=4096)
    try:
        bw = BatchWindows(big)
        counts, res = {}, {}
        for n, off in ((1, 530), (8, 0), (264, 264)):
            seqs = [Seq(j, off + j, off + j, 3, 1500 + j % 8) for j in range(n)]
            for s in seqs:
                s.ta = 1000 + off + s.j
                batch_feature_track(big, [s.feature(s.ta)], keypoint_distance=KD)
                bw.reset(s.a, s.run.w)
                bw.edit([Edit(s.a).frame(_state16(s.run, 0))])
                bw.set_keypoints(s.a, s.ta, 1, {})
                s.f = 1
            n0 = big.kernel_launches
            res[n] = bw.track_camera([s.camera() for s in seqs], CAP, keypoint_distance=KD)
            counts[n] = big.kernel_launches - n0
        assert counts[8] == counts[264], counts
        print("launches per track_camera call:", counts)
        for other in (res[8][:1], res[264][:1], res[264][8:9]):
            o, r = other[0], res[1][0]
            for key in ("keypoints", "state", "predicted", "predict_q", "imu_record"):
                assert np.array_equal(_bits(o[key]), _bits(r[key])), key
            assert np.array_equal(o["kp_track"], r["kp_track"]) and np.array_equal(o["prev_index"], r["prev_index"])
    finally:
        big.close()
