"""pvio_b200_batch_window_plane_ransac: PlaneExtractor::work and Plane::update_parameter(true) on resident slots, the
points built on the device from each slot's own track table.  Checked against a host gather from the slot download,
against pvio_b200_triangulate and the fp64 triangulation oracle, against the serial RANSAC of oracle/plane_oracle.py
iteration by iteration, at its edges, in mixed batches, and along sequences with a plane in view."""
import numpy as np
import pytest

from oracle import plane_oracle as po
from oracle import tri_oracle as to
from pvio_b200 import _lib, triangulate
from pvio_b200._lib import EINVAL
from pvio_b200.batch_window import Edit, PlaneRansac, Planes
from pvio_b200.bundle_adjustor import BundleAdjustor
from synthetic import so3
from synthetic.sequence import BatchPlayer, Run

pytestmark = pytest.mark.gpu
EXTRACT, REFIT = PlaneRansac.EXTRACT, PlaneRansac.REFIT
RUNS = [dict(F=14, N=8, M=200, seed=741 + j, planes=1, tracks_per_plane=150, plane_landmarks=True) for j in range(4)]
SPARE = 4                                  # a slot built track by track for the edge cases
KEYFRAMES = 3


def _handle():
    return BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=512, max_obs=6000)


def _play(ba, calls=None):
    """4 sequences with the floor in view through KEYFRAMES keyframes (solve, drop, next frame); calls(player) between
    the solve and the drop of every keyframe"""
    player = BatchPlayer(ba, [Run(**kw) for kw in RUNS])
    js = list(range(len(RUNS)))
    for _ in range(KEYFRAMES):
        player.bw.solve([player.slots[j] for j in js], max_iterations=6)
        if calls:
            calls(player)
        player.advance(js)
    return player


@pytest.fixture(scope="module")
def setup():
    ba = _handle()
    player = _play(ba)
    yield ba, player
    ba.close()


# ------------------------------------------------------------------------ host views of a slot
def _host(player, j):
    """(run, download, model tracks by id) of run j"""
    d = player.bw.download([player.slots[j]], 512)[0]
    return player.runs[j], d, player.model.m[player.slots[j]].tracks


def _extract_ids(player, j, seed=0):
    """every live track of run j in a shuffled order (Map order is not id order)"""
    _, d, _ = _host(player, j)
    return np.random.default_rng(seed + j).permutation(d["ids"]).astype(np.int32)


def _refit_ids(player, j):
    """the tracks of run j on the floor, in id order"""
    run, d, tr = _host(player, j)
    return np.array([i for i in d["ids"] if tr[int(i)]["l"] is not None and tr[int(i)]["l"] >= run.w.M], dtype=np.int32)


def _host_gather(player, j, ids, mode):
    """per candidate: enough_baseline, the point (get_landmark_point from the download, or try_triangulate through the
    oracle over the window views) and the views"""
    run, d, tr = _host(player, j)
    row = {int(t): r for r, t in enumerate(d["ids"])}
    fr = d["frames"]
    used, pts, views = [], np.full((len(ids), 3), np.nan), []
    for i, t in enumerate(ids):
        t, r = int(t), row[int(t)]
        frames, zs = tr[t]["frames"], tr[t]["zs"]
        assert frames[0] == d["anchor"][r]
        ok = po.enough_baseline([fr[f, 4:7] for f in frames], d["inv_depth"][r])
        cams = [run.cam_pose(fr[f, 0:4], fr[f, 4:7]) for f in frames]
        views.append((cams, zs))
        if ok and mode == EXTRACT:
            qc, pc = cams[0]
            rho = d["inv_depth"][r]
            pts[i] = so3.qrot(qc, np.array([zs[0][0] / rho, zs[0][1] / rho, 1.0 / rho])) + pc
        elif ok:
            p = po.refit_point(cams, zs)
            ok = p is not None
            if ok:
                pts[i] = p
        used.append(ok)
    return np.array(used), pts, views


def _check_against_oracle(o, mode):
    """the record's RANSAC on its returned points against the serial oracle"""
    P = o["points"][o["used"]]
    assert o["n_points"] == len(P)
    ref = po.plane_ransac(P, mode)
    assert o["status"] == ref["status"]
    if ref["status"] == po.FEW_POINTS:
        assert (o["counts"] == -1).all() and (o["schedule"] == -1).all() and o["best_it"] == -1
        assert np.isnan(o["normal"]).all() and np.isnan(o["reference"]).all() and not o["inlier"].any()
        return ref
    np.testing.assert_array_equal(o["schedule"], po.lotbox_schedule(len(P), 0, 3, 1000))
    np.testing.assert_array_equal(o["counts"][:ref["iterations"]], ref["counts"])
    full = [int(po.inlier_mask(P, *po.plane_solve(*P[s]), po.THRESHOLD[mode]).sum()) for s in o["schedule"]]
    np.testing.assert_array_equal(o["counts"], full)
    assert (o["iterations"], o["best_it"], o["inliers"]) == (ref["iterations"], ref["best_it"], ref["inliers"])
    np.testing.assert_array_equal(o["inlier"][o["used"]], ref["mask"])
    assert not o["inlier"][~o["used"]].any()
    if ref["status"] == po.ACCEPTED:
        np.testing.assert_array_equal(o["reference"], po.centroid(P, ref["mask"]))
        np.testing.assert_allclose(o["normal"], ref["plane"][:3], rtol=0, atol=1e-10)
        assert abs(o["distance"] - ref["plane"][3]) <= 1e-10
        assert o["distance"] >= 0
    elif mode == REFIT:                        # the raw model, an undefined reference point
        np.testing.assert_array_equal(o["normal"], ref["normal"])
        assert o["distance"] == ref["distance"] and np.isnan(o["reference"]).all()
    else:
        assert np.isnan(o["normal"]).all() and np.isnan(o["distance"])
    return ref


# ------------------------------------------------------------------------ gather
def test_gather_matches_the_host_gather(setup):
    ba, player = setup
    recs = [PlaneRansac(player.slots[j], EXTRACT, _extract_ids(player, j)) for j in range(4)]
    recs += [PlaneRansac(player.slots[j], REFIT, _refit_ids(player, j)) for j in range(4)]
    out = player.bw.plane_ransac(recs, schedules=True)
    for rec, o in zip(recs, out):
        j = player.slots.index(rec.slot)
        used, pts, views = _host_gather(player, j, rec.tracks, rec.mode)
        np.testing.assert_array_equal(o["used"], used)
        assert used.sum() >= 50
        assert np.isnan(o["points"][~used]).all()
        scale = np.abs(pts[used]).max()
        if rec.mode == EXTRACT:
            np.testing.assert_allclose(o["points"][used], pts[used], rtol=1e-12, atol=1e-12 * scale)
            continue
        np.testing.assert_allclose(o["points"][used], pts[used], rtol=1e-7, atol=1e-7 * scale)   # SVD vs Jacobi
        # the same views through pvio_b200_triangulate: one camera per (used candidate, view)
        Ps, begin, fr, zs = [], [0], [], []
        for (cams, z), u in zip(views, used):
            if not u:
                continue
            for (q, p), zz in zip(cams, z):
                fr.append(len(Ps)); Ps.append(to.projection_matrix(q, p)); zs.append(zz)
            begin.append(len(fr))
        tp, tv, _ = triangulate.triangulate(ba, np.array(Ps), np.array(begin), np.array(fr), np.array(zs))
        assert tv.all()
        np.testing.assert_allclose(o["points"][used], tp, rtol=1e-8, atol=1e-8 * scale)


def test_ransac_matches_the_oracle(setup):
    ba, player = setup
    recs = [PlaneRansac(player.slots[j], EXTRACT, _extract_ids(player, j, seed)) for j in range(4) for seed in (0, 9)]
    recs += [PlaneRansac(player.slots[j], REFIT, _refit_ids(player, j)) for j in range(4)]
    for rec, o in zip(recs, player.bw.plane_ransac(recs, schedules=True)):
        ref = _check_against_oracle(o, rec.mode)
        assert ref["status"] == po.ACCEPTED


# ------------------------------------------------------------------------ edges, on a slot built track by track
def _spare(ba, player, points, dup=()):
    """reset the spare slot to three frames of run 0 (0, 3, 6: a baseline above 0.5) and one track per world point,
    anchored in frame 0 (z, inverse depth from the point), observed in frames 1 and 2; dup: (i, j) pairs of tracks made
    identical to track i.  Returns the track ids."""
    run, bw = player.runs[0], player.bw
    bw.reset(SPARE, run.w)
    ids = None
    for k, f in enumerate((0, 3, 6)):
        e = Edit(SPARE).frame(player.state16(0, f), False, player.rec[0][f - 1] if k else None)
        if k == 0:
            qc, pc = run.cam_pose(run.guess.q[f], run.guess.p[f])
            z, rho = [], []
            for x in points:
                y = so3.qrot(so3.qconj(qc), x - pc)
                z.append(y[:2] / y[2]); rho.append(1.0 / y[2])
            for i, j in dup:
                z[j], rho[j] = z[i], rho[i]
            e.new = [(0, zz, r) for zz, r in zip(z, rho)]
        else:
            e.obs = [(int(t), k, np.array([0.01 * k, 0.0])) for t in ids]
        got = bw.edit([e])[0]
        if k == 0:
            ids = got
    return ids


def _floor(rng, n_on, n_off):
    """n_on points on the floor z = -1.4 ahead of run 0's first camera, n_off points 0.3 .. 2 m off it"""
    on = np.c_[rng.uniform(3, 8, n_on), rng.uniform(-2, 2, n_on), np.full(n_on, -1.4)]
    off = np.c_[rng.uniform(3, 8, n_off), rng.uniform(-2, 2, n_off), -1.4 + rng.choice([-1, 1], n_off) * rng.uniform(0.3, 2, n_off)]
    return np.vstack([on, off])


def test_edges_extraction_point_counts(setup):
    ba, player = setup
    ids = _spare(ba, player, _floor(np.random.default_rng(3), 20, 0))
    recs = [PlaneRansac(SPARE, EXTRACT, ids[:k]) for k in (0, 2, 3)]
    out = player.bw.plane_ransac(recs, schedules=True)
    assert [o["n_points"] for o in out] == [0, 2, 3]
    assert [o["status"] for o in out] == [_lib.PLANE_FEW_POINTS, _lib.PLANE_FEW_POINTS, _lib.PLANE_REJECTED]
    for o in out:
        _check_against_oracle(o, EXTRACT)
    assert out[2]["inliers"] == 3 and out[2]["iterations"] == 1     # ratio 1: one iteration


@pytest.mark.parametrize("n_on", [30, 31])
def test_edges_thirty_and_thirty_one_inliers(setup, n_on):
    ba, player = setup
    ids = _spare(ba, player, _floor(np.random.default_rng(11), n_on, 70))
    o = player.bw.plane_ransac([PlaneRansac(SPARE, EXTRACT, ids)], schedules=True)[0]
    _check_against_oracle(o, EXTRACT)
    assert o["inliers"] == n_on and o["inlier"][:n_on].all()
    assert o["status"] == (_lib.PLANE_ACCEPTED if n_on == 31 else _lib.PLANE_REJECTED)


def test_edges_degenerate_sample(setup):
    ba, player = setup
    first = po.lotbox_schedule(40, 0, 3, 1)[0]                      # iteration 0's sample of 40 points
    pts = _floor(np.random.default_rng(5), 10, 30)
    ids = _spare(ba, player, pts, dup=[(int(first[0]), int(first[1])), (int(first[0]), int(first[2]))])
    o = player.bw.plane_ransac([PlaneRansac(SPARE, EXTRACT, ids)], schedules=True)[0]
    _check_against_oracle(o, EXTRACT)
    assert o["counts"][0] == 40 and o["best_it"] == 0 and o["inliers"] == 40 and o["iterations"] == 1
    assert o["status"] == _lib.PLANE_ACCEPTED and o["inlier"].all()


def test_edges_refit_49_50_and_rejected(setup):
    ba, player = setup
    ids = _refit_ids(player, 0)
    o = player.bw.plane_ransac([PlaneRansac(player.slots[0], REFIT, ids)])[0]
    good = ids[o["used"]]
    assert len(good) >= 50
    out = player.bw.plane_ransac([PlaneRansac(player.slots[0], REFIT, good[:k]) for k in (49, 50)], schedules=True)
    assert [x["n_points"] for x in out] == [49, 50]
    assert out[0]["status"] == _lib.PLANE_FEW_POINTS and np.isnan(out[0]["normal"]).all()
    assert out[1]["status"] != _lib.PLANE_FEW_POINTS
    for x in out:
        _check_against_oracle(x, REFIT)
    # a refit over off-plane landmarks: rejected, the raw model with a NaN reference point
    run, d, tr = _host(player, 0)
    lm = np.array([i for i in d["ids"] if tr[int(i)]["l"] is not None and tr[int(i)]["l"] < run.w.M], dtype=np.int32)
    o = player.bw.plane_ransac([PlaneRansac(player.slots[0], REFIT, lm)], schedules=True)[0]
    ref = _check_against_oracle(o, REFIT)
    assert ref["status"] == po.REJECTED and np.isfinite(o["normal"]).all() and np.isnan(o["reference"]).all()


# ------------------------------------------------------------------------ batch behaviour
def _mixed(player, n):
    recs = []
    for i in range(n):
        j = i % 4
        if i % 3 == 2:
            recs.append(PlaneRansac(player.slots[j], REFIT, _refit_ids(player, j)))
        else:
            ids = _extract_ids(player, j, seed=i)
            recs.append(PlaneRansac(player.slots[j], EXTRACT, ids[: 40 + (7 * i) % max(len(ids) - 40, 1)]))
    return recs


def _same(a, b):
    for k in a:
        if isinstance(a[k], np.ndarray):
            np.testing.assert_array_equal(a[k], b[k], err_msg=k)
        else:
            assert a[k] == b[k] or (a[k] != a[k] and b[k] != b[k]), k


def test_mixed_batch_equals_each_record_alone(setup):
    ba, player = setup
    recs = _mixed(player, 132)
    batch = player.bw.plane_ransac(recs, schedules=True)
    for r, o in zip(recs, batch):
        _same(o, player.bw.plane_ransac([r], schedules=True)[0])


def test_three_launches_whatever_n(setup):
    ba, player = setup
    for n in (8, 264):
        recs = _mixed(player, n)
        n0 = ba.kernel_launches
        player.bw.plane_ransac(recs)
        assert ba.kernel_launches - n0 == 3
    n0 = ba.kernel_launches
    assert player.bw.plane_ransac([]) == [] and ba.kernel_launches == n0


def test_slots_are_untouched(setup):
    """downloads, IMU records and the post-pass flags are bit-identical before and after a mixed call, and the slots
    then solve"""
    ba, player = setup
    slots = [player.slots[j] for j in range(4)]
    before = player.bw.download(slots, 512), player.bw.imu_records(slots)
    player.bw.plane_ransac(_mixed(player, 24))
    after = player.bw.download(slots, 512), player.bw.imu_records(slots)
    for x, y in zip(before[0], after[0]):
        for k in x:
            np.testing.assert_array_equal(x[k], y[k], err_msg=k)
    for x, y in zip(before[1], after[1]):
        np.testing.assert_array_equal(x, y)


def _raw(ba, recs, n=None):
    arr = (_lib.CWindowPlaneRansac * max(len(recs), 1))(*recs)
    return ba.lib.pvio_b200_batch_window_plane_ransac(ba.h, len(recs) if n is None else n, arr)


@pytest.mark.parametrize("spoil", ["slot_range", "slot_not_resident", "unknown", "dead", "twice", "mode", "null_tracks",
                                   "null_info", "too_many"])
def test_rejections_change_no_output(setup, spoil):
    ba, player = setup
    s = player.slots[1]
    ids = _extract_ids(player, 1)
    info, plane = np.full(5, 7, dtype=np.int32), np.full(7, 7.0)
    used, inl = np.full(len(ids), 7, dtype=np.uint8), np.full(len(ids), 7, dtype=np.uint8)
    good = _lib.CWindowPlaneRansac(slot=player.slots[0], mode=EXTRACT, n_tracks=len(ids))
    keep = [ids.copy()]
    _lib.set_ptrs(good, tracks=keep[0], info=np.zeros(5, dtype=np.int32), plane=np.zeros(7),
                  used=np.zeros(len(ids), dtype=np.uint8), inlier=np.zeros(len(ids), dtype=np.uint8))
    t = ids.copy()
    r = _lib.CWindowPlaneRansac(slot=s, mode=EXTRACT, n_tracks=len(t))
    _lib.set_ptrs(r, tracks=t, info=info, plane=plane, used=used, inlier=inl)
    n = None
    if spoil == "slot_range":
        r.slot = 99
    elif spoil == "slot_not_resident":
        r.slot = 7
    elif spoil == "unknown":
        t[3] = 10 ** 6
    elif spoil == "dead":
        live = set(int(i) for i in ids)
        t[3] = next(i for i in range(int(ids.max())) if i not in live)
    elif spoil == "twice":
        t[5] = t[2]
    elif spoil == "mode":
        r.mode = 2
    elif spoil == "null_tracks":
        r.tracks = None
    elif spoil == "null_info":
        r.info = None
    elif spoil == "too_many":
        n = 65536
    recs = [good, r] if n is None else [r] * 65536
    n0 = ba.kernel_launches
    assert _raw(ba, recs, n) == EINVAL
    assert ba.kernel_launches == n0
    assert (info == 7).all() and (plane == 7.0).all() and (used == 7).all() and (inl == 7).all()
    del keep


# ------------------------------------------------------------------------ sequences with the floor in view
def _valid_ids(player, j):
    """the extractor's candidates as the host filters them (plane_extractor.cpp:45-47): live tracks that the last solve
    kept (TF_VALID) with quality < 2.0, in a shuffled order"""
    _, d, _ = _host(player, j)
    ok = (d["valid"] == 1) & (d["quality"] < 2.0)
    return np.random.default_rng(j).permutation(d["ids"][ok]).astype(np.int32)


def test_sequences_find_and_refit_the_floor(setup):
    ba, player = setup
    recs = [PlaneRansac(player.slots[j], EXTRACT, _valid_ids(player, j)) for j in range(4)]
    found = player.bw.plane_ransac(recs)
    planes, truth = [], []
    for j, (rec, o) in enumerate(zip(recs, found)):
        run, d, tr = _host(player, j)
        # the floor's normal in the estimate's frame, through the window's oldest frame: the estimate may sit rotated
        # against the truth by what the gauge and the IMU factors leave free
        R = so3.qmat(d["frames"][0, 0:4]) @ so3.qmat(run.truth.q[player.k[j]]).T
        truth.append(R @ np.array([0.0, 0.0, 1.0]))
        assert o["status"] == _lib.PLANE_ACCEPTED
        on = np.array([tr[int(t)]["l"] >= run.w.M for t in rec.tracks]) & o["used"]
        n = o["normal"] * np.sign(o["normal"] @ truth[-1])
        angle = np.degrees(np.arccos(min(1.0, n @ truth[-1])))
        assert on.sum() >= 50 and o["inlier"][on].mean() >= 0.9 and angle < 1.0, (on.sum(), o["inlier"][on].mean(), angle)
        planes.append(Planes(player.slots[j], np.r_[o["normal"], o["distance"]][None]))
        for t in np.sort(rec.tracks[o["inlier"]]):
            planes[-1].role(int(t), 0)
    player.bw.set_planes(planes)
    refits = [PlaneRansac(p.slot, REFIT, np.array(p.tracks, dtype=np.int32)) for p in planes]
    for f, o, t in zip(found, player.bw.plane_ransac(refits, schedules=True), truth):
        _check_against_oracle(o, REFIT)
        assert o["status"] == _lib.PLANE_ACCEPTED
        # a looser bar: the refit triangulates over every window view, and the newest frame holds the state the player
        # fed (not localized against the solved window), which biases the triangulated floor by a few centimetres
        assert np.degrees(np.arccos(min(1.0, abs(o["normal"] @ f["normal"])))) < 2.0
        assert abs(o["normal"] @ t) > np.cos(np.radians(2.0)) and abs(o["distance"] - f["distance"]) < 0.2
    player.bw.set_planes([_unset(p) for p in planes])


def _unset(p):
    """the record that gives the tracks of a Planes record back their landmark role and removes the plane"""
    q = Planes(p.slot, np.zeros((0, 4)))
    for t in p.tracks:
        q.role(t, -1)
    return q
