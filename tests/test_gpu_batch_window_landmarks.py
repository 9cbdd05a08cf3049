"""pvio_b200_batch_window_landmarks: every row's world point against landmark_oracle.landmark_point's arithmetic at the
slot's downloaded state and the keypoints the test fed, the point covariance against landmark_oracle.point_covariance
(dense), the points of slots driven through mirror_frame (no host keypoint) and through replace_last edits, Var(rho) bit for bit against pvio_b200_batch_window_covariance, the selection modes, the numeric status, the
rejections, that the call changes no slot, and its launch count."""
import numpy as np
import pytest

import landmark_oracle as lo
from oracle.lie import qrot
from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows, Edit
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from synthetic import synth
from test_gpu_batch_window_covariance import _feed, _repack, _snap, _tracks, _visual
from test_gpu_batch_window_mirror import Seq, _advance, _drop, _start, _step

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"
# |C - C_ref|_ij / sqrt(C_ref,ii C_ref,jj) of the point covariances against the dense oracle: inertial windows run the
# fp64 pipeline, visual-only ones fp32 Jacobians.  Set from the first H100 run (DESIGN 5b): worst seen 2.2e-5 (fp64,
# the size of the inverse-depth variance error of test_gpu_batch_window_covariance), 8.9e-6 (fp32)
BAR_FP64, BAR_FP32 = 1e-4, 2e-3


def _point(w, fr, z, rho):
    """Track::get_landmark_point() from a downloaded frame state fr [16], the anchor keypoint z and rho"""
    y = np.array([z[0], z[1], 1.0]) / rho
    return qrot(fr[0:4], qrot(w.cam_q_cs, y) + w.cam_p_cs) + fr[4:7]


def _check_points(w, d, model, out):
    """every row's point at the downloaded state and the fed keypoints; ids in id order; roles of the model"""
    assert np.array_equal(out["ids"], d["ids"])
    rho = dict(zip((int(i) for i in d["ids"]), d["inv_depth"]))
    for t, x, r in zip(out["ids"], out["point"], out["role"]):
        m = model[int(t)]
        ref = _point(w, d["frames"][m["frames"][0]], m["zs"][0], rho[int(t)])
        assert np.linalg.norm(x - ref) <= 1e-12 * np.linalg.norm(ref), (t, x, ref)
        assert r == m["role"]


def _check_cov(bw, slot, w, model, fixed, bar, prior=None):
    d = bw.download([slot], 600)[0]
    out = bw.landmarks([slot], covariance=True)[0]
    assert out["status"] == _lib.OK
    _check_points(w, d, model, out)
    ids = [int(i) for i in out["ids"]]
    var = bw.covariance([slot], [[]], [ids])[0]["inv_depth_var"]
    assert np.array_equal(var, out["inv_depth_var"], equal_nan=True)         # the same arithmetic, bit for bit
    imu = bw.imu_records([slot])[0] if w.use_inertial else None
    wr, sr, lms = _repack(w, d, model, imu, fixed, prior)
    lm_of = {t: k for k, t in enumerate(lms)}
    ref = lo.point_covariance(wr, sr, [lm_of.get(t) for t in ids])
    worst = 0.0
    for t, C, R in zip(ids, out["point_cov"], ref):
        lm = model[t]["role"] < 0 and len(model[t]["frames"]) >= 2
        assert np.isnan(C).all() == (not lm) and np.isnan(R).all() == (not lm)
        if lm:
            assert np.array_equal(C, C.T)
            s = np.sqrt(np.diag(R))
            worst = max(worst, float(np.max(np.abs(C - R) / np.outer(s, s))))
    print(f"slot {slot}: {len(ids)} rows, {len(lms)} landmarks, point covariance error {worst:.3g}")
    assert worst < bar, worst
    return out


def test_inertial_points_and_covariance_before_and_after_a_drop():
    """cfg4 windows (gauge prior, plane tracks with set_planes inverse depths, role -2 tracks, one-observation plane
    tracks), solved; then after drop_victim (re-anchored rows) with the new prior"""
    res = BundleAdjustor(max_windows=3, max_frames=9, max_landmarks=600, max_obs=4000)
    bw = BatchWindows(res)
    wins = [synth.make_cfg4(seed=990 + i, N=(7, 9)[i], M=150)[:2] for i in range(2)]
    models = [_feed(bw, i + 1, w, st, _tracks(w)) for i, (w, st) in enumerate(wins)]
    d0 = bw.download([1], 600)[0]                       # before any solve: the fed state
    _check_points(wins[0][0], d0, models[0], bw.landmarks([1])[0])
    assert any(len(m["frames"]) == 1 for m in models[0].values()) and any(m["role"] >= 0 for m in models[0].values())
    bw.solve([1, 2], max_iterations=4)
    for i, (w, _) in enumerate(wins):
        _check_cov(bw, i + 1, w, models[i], [0] * w.N, BAR_FP64)
    S, e = bw.drop_victim([1, 2], want=True, max_frames=9)
    for i, ((w, _), m) in enumerate(zip(wins, models)):
        for t in list(m):
            if m[t]["frames"][0] == 0:
                m[t]["frames"].pop(0); m[t]["zs"].pop(0)
            if not m[t]["frames"]:
                del m[t]
                continue
            m[t]["frames"] = [f - 1 for f in m[t]["frames"]]
        dk = 15 * (w.N - 1)
        _check_cov(bw, i + 1, w, m, [0] * (w.N - 1), BAR_FP64, prior=(S[i, :dk * dk].reshape(dk, dk), e[i, :dk]))
    res.close()


def test_visual_selection_and_numeric_status():
    """cfg2 windows with two fixed frames on an fp32 handle: the oracle; named tracks give the all-tracks rows; a
    too-small capacity is rejected; a slot with an unobserved free frame is ENUMERIC with NaN covariances and finite
    points while the other record of the call is unaffected"""
    res = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=600, max_obs=4000)
    bw = BatchWindows(res)
    w, m = _visual(bw, 0)
    bw.solve([0], max_iterations=3)
    full = _check_cov(bw, 0, w, m, list(w.frame_fixed), BAR_FP32)
    ids = list(full["ids"])
    pick = [ids[k] for k in (7, 2, 30, 11, 0)]
    named = bw.landmarks([0], [pick], covariance=True)[0]
    rows = [ids.index(t) for t in pick]
    assert np.array_equal(named["ids"], pick) and np.array_equal(named["role"], full["role"][rows])
    for k in ("point", "point_cov", "inv_depth_var"):
        assert np.array_equal(named[k], full[k][rows], equal_nan=True), k
    pts = bw.landmarks([0])[0]                          # points only: the same points
    assert "point_cov" not in pts and np.array_equal(pts["point"], full["point"])
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.landmarks([0], capacity=len(ids) - 1)
    free = [f for f in range(w.N) if not w.frame_fixed[f]]
    _visual(bw, 3, skip=free[-1])
    r = bw.landmarks([3, 0], covariance=True)
    assert r[0]["status"] == _lib.ENUMERIC and len(r[0]["ids"]) > 0
    assert np.isnan(r[0]["point_cov"]).all() and np.isnan(r[0]["inv_depth_var"]).all()
    assert np.isfinite(r[0]["point"]).all()
    assert r[1]["status"] == _lib.OK
    for k in ("ids", "point", "role", "point_cov", "inv_depth_var"):
        assert np.array_equal(r[1][k], full[k], equal_nan=True), k
    res.close()


def _call(bw, recs):
    """the C call on raw records (for the rejections the Python method never builds)"""
    arr = (_lib.CWindowLandmarks * len(recs))(*recs)
    bw.ba._ck(bw.lib.pvio_b200_batch_window_landmarks(bw.h, len(recs), arr))
    return arr


def test_no_side_effects_rejections_and_launch_count():
    """every slot's download and save blob are byte-identical after the call and after every rejection, and a
    rejection writes no output; the launch count is the same at 8 and 264 records, 1 for points only and 5 with the
    covariance"""
    W = 265                                               # the last slot stays empty (not resident)
    res = BundleAdjustor(max_windows=W, max_frames=6, max_landmarks=200, max_obs=1200)
    bw = BatchWindows(res)
    w, st = synth.make_cfg2(seed=997, N=5, M=60)[:2]
    tr = _tracks(w, planes=False)
    for s in range(W - 1):
        _feed(bw, s, w, st, [dict(t) for t in tr])
    bw.solve([0, 1, 2], max_iterations=2)
    ids = [int(i) for i in bw.download([0], 200)[0]["ids"]]
    e = Edit(0)                                           # a dead track: live once, removed by an edit
    e.remove = [ids[-1]]
    bw.edit([e])
    dead, ids = ids[-1], ids[:-1]
    assert [int(i) for i in bw.download([0], 200)[0]["ids"]] == ids
    before = _snap(bw, [0, 1, 2])
    bw.landmarks([0, 1], [ids[:10], None], covariance=True)
    bw.landmarks([2, 0])
    pt = np.full((4, 3), 7.0)
    sentinel = pt.copy()

    def rec(slot=0, tracks=ids[:4], n=None, cap=0, point=pt, cov=None):
        r = _lib.CWindowLandmarks()
        t = None if tracks is None else np.ascontiguousarray(tracks, dtype=np.int32)
        r.slot, r.n_tracks, r.capacity = slot, (len(t) if n is None else n), cap
        _lib.set_ptrs(r, tracks=t, point=point, point_cov=cov)
        r._keep = t
        return r

    bad = [[rec(), rec()],                                   # slot twice
           [rec(slot=W)],                                    # slot out of range
           [rec(slot=W - 1)],                                # not resident
           [rec(tracks=[ids[0], ids[0]])],                   # track twice
           [rec(tracks=[ids[1], dead])],                     # dead track (removed, below the slot's next id)
           [rec(tracks=[10 ** 6])],                          # unknown track (never issued)
           [rec(tracks=None, n=4)],                          # tracks missing
           [rec(point=None)],                                # point missing
           [rec(tracks=None, n=-1, cap=len(ids) - 1)],       # capacity too small
           [rec(n=-2)]]                                      # track count out of range
    for recs in bad:
        with pytest.raises(PvioB200Error, match=EINVAL):
            _call(bw, recs)
        assert np.array_equal(pt, sentinel)
    after = _snap(bw, [0, 1, 2])
    for x, y in zip(before[0], after[0]):
        for k in x:
            assert np.array_equal(x[k], y[k]), k
    assert before[1] == after[1]
    for cov, want in ((False, 1), (True, 5)):
        counts = []
        for n in (8, W - 1):
            l0 = res.kernel_launches
            bw.landmarks(list(range(n)), [ids[:3]] * 4 + [None] * (n - 4), covariance=cov)
            counts.append(res.kernel_launches - l0)
        assert counts[0] == counts[1] == want, (cov, counts)
    res.close()


def _check_mirrored(bw, s, slot):
    """every row's point of a mirror-driven slot (or its twin) against the keypoints mirror_oracle gave the host's
    history: the row's anchor window frame -> its tracker frame -> the keypoint the track had there"""
    d = bw.download([slot], 4096)[0]
    out = bw.landmarks([slot], capacity=4096)[0]
    assert np.array_equal(out["ids"], d["ids"])
    w = s.run.w
    for t, a, rho, x in zip(d["ids"], d["anchor"], d["inv_depth"], out["point"]):
        ref = _point(w, d["frames"][a], s.zhist[int(t)][s.wf[a]], rho)
        assert np.linalg.norm(x - ref) <= 1e-12 * np.linalg.norm(ref), (slot, t, x, ref)
    return len(out["ids"])


def test_points_of_mirrored_slots_and_replace_last_edits():
    """sequences whose frames come straight from their tracker slots (mirror_frame: the host holds no keypoint), with
    forced non-keyframes and drops; each slot's points against mirror_oracle's keypoints after every frame.  Each
    sequence's twin slot takes the same frames as host edits, a non-keyframe's successor as a replace_last edit whose new
    tracks are anchored in the replaced frame; its points are checked the same way."""
    res = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=4096, max_obs=16384)
    bw = BatchWindows(res)
    seqs = [Seq(j, j, 4 + j, 12, 930 + j) for j in range(2)]
    _start(bw, seqs)
    replaced_born = drops = 0
    for k in range(10):
        ft = _advance(bw, seqs)
        replace = [not s.newest_kf for s in seqs]
        out = _step(bw, seqs, ft)
        for s, r, o in zip(seqs, replace, out):
            _check_mirrored(bw, s, s.slot)
            _check_mirrored(bw, s, s.twin)
            replaced_born += int(r and o["counts"][3] > 0)
        full = [s for s in seqs if s.newest_kf and s.N >= 6]
        if full:
            _drop(bw, seqs, full)
            drops += len(full)
            for s in full:                   # re-anchored rows
                _check_mirrored(bw, s, s.slot)
                _check_mirrored(bw, s, s.twin)
        for s in seqs:                       # force a non-keyframe now and then: the next frame replaces it
            if k % 3 == 1 and s.newest_kf and s not in full and s.N >= 2:
                s.newest_kf = False
                bw.set_keypoints(s.slot, s.tracker, s.f + 1, {t: kj for kj, t in s.tk.items()}, False, s.skipped)
    print(f"replace_last frames with new tracks {replaced_born}, drops {drops}")
    assert replaced_born > 0 and drops > 0
    res.close()
