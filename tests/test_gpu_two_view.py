"""pvio_b200_batch_two_view: init_sfm's two-view step (initializer.cpp:102-161) on the device, against the serial CPU
oracle (oracle/twoview_oracle.py) on synthetic two-view scenes: general depth, a dominant plane, a pure rotation and
too little parallax; 0 to 1000 matches; 0 to 50 % outliers.  The device's sample schedules must equal the oracle's
exactly; the homography counts must equal the oracle's on every iteration; the essential counts too, except on
iterations the oracle flags as borderline (an eigenvalue with 1e-11 < |imag| < 1e-9, or a match within 1e-9 relative
of the threshold), at most 1 % of them; the final answer must equal the serial loop's."""
import numpy as np
import pytest

from oracle import twoview_oracle as tv
from pvio_b200 import _lib
from pvio_b200.two_view import batch_two_view, two_view
from pvio_b200._lib import EINVAL
from synthetic import synth

pytestmark = pytest.mark.gpu

SCENES = [
    dict(seed=40, n=150, outlier_frac=0.0, kind="general"),
    dict(seed=41, n=300, outlier_frac=0.3, kind="general"),
    dict(seed=42, n=1000, outlier_frac=0.5, kind="general"),
    dict(seed=43, n=50, outlier_frac=0.1, kind="general"),
    dict(seed=44, n=200, outlier_frac=0.1, kind="plane"),
    dict(seed=45, n=120, outlier_frac=0.0, kind="rotation", noise_px=0.0, ill_posed=True),
    dict(seed=46, n=120, outlier_frac=0.2, kind="rotation"),
    dict(seed=47, n=100, outlier_frac=0.0, kind="small", ill_posed=True),
    dict(seed=48, n=5, outlier_frac=0.0, kind="general"),
    dict(seed=49, n=30, outlier_frac=0.0, kind="general"),
    dict(seed=50, n=4, outlier_frac=0.0, kind="general"),
    dict(seed=51, n=0, outlier_frac=0.0, kind="general"),
]


@pytest.fixture(scope="module")
def ba():
    from pvio_b200.bundle_adjustor import BundleAdjustor
    b = BundleAdjustor(max_windows=1, max_frames=4, max_landmarks=16, max_obs=64)
    yield b
    b.close()


def _problem(sc, **kw):
    s = synth.make_two_view(**{k: v for k, v in sc.items() if k != "ill_posed"})
    d = dict(p1=s["p1"], p2=s["p2"], fx=s["fx"], fy=s["fy"])
    d.update(kw)
    return d


def _all_counts(kind, d, schedule):
    """Every iteration of the schedule as the device evaluates it: (counts rows, borderline flags)."""
    thr_h, thr_e = tv.thresholds(d["fx"])
    p1, p2 = np.asarray(d["p1"], dtype=np.float64), np.asarray(d["p2"], dtype=np.float64)
    rows, border = [], []
    for idx in schedule:
        models, masks, b = tv.iteration(kind, p1, p2, idx, thr_h if kind == "H" else thr_e)
        rows.append([len(models)] + [int(m.sum()) for m in masks])
        border.append(b)
    return rows, border


@pytest.mark.parametrize("sc", SCENES, ids=[f"{s['kind']}-{s['n']}-{s['outlier_frac']}-{s['seed']}" for s in SCENES])
def test_two_view_equals_the_serial_oracle(ba, sc):
    d = _problem(sc)
    got = two_view(ba, diagnostics=True, **d)
    ref = tv.two_view(d["p1"], d["p2"], d["fx"], d["fy"])
    n = sc["n"]
    assert got["status"] == ref["status"]
    assert got["parallax"] == pytest.approx(ref["parallax"], rel=1e-12)
    if n < 5:                                   # no RANSAC below 5 matches: too few matches, nothing evaluated
        assert got["status"] == tv.STATUS_FEW_MATCHES
        assert got["h_iterations"] == 0 and got["e_iterations"] == 0 and got["candidate"] == -1
        assert got["h_best_it"] == -1 and got["e_best_it"] == -1 and got["triangulated"] == 0
        assert not got["h_mask"].any() and not got["e_mask"].any() and not got["point_status"].any()
        assert np.all(got["H"] == 0) and np.all(got["E"] == 0) and np.all(got["points"] == 0)
        return
    # schedules
    np.testing.assert_array_equal(got["h_schedule"], tv.lotbox_schedule(n, 648, 4, 1000))
    np.testing.assert_array_equal(got["e_schedule"], tv.lotbox_schedule(n, 648, 5, 1000))
    # every iteration's counts.  Without a baseline (a pure rotation, or 2 cm against depths of 3 to 12 m) the 5-point
    # problem has no well-defined solution: its real roots are as ill-conditioned as the eigen-solvers that find them,
    # so there only the homography, the gates and the status are compared.
    ill = sc.get("ill_posed", False)
    rows, _ = _all_counts("H", d, got["h_schedule"])
    np.testing.assert_array_equal(got["h_counts"], [r[1] for r in rows])          # every iteration, no exception
    if not ill:
        rows, border = _all_counts("E", d, got["e_schedule"])
        dev, skipped = got["e_counts"], 0
        for it, (r, b) in enumerate(zip(rows, border)):
            drow = [int(dev[it, 0])] + [int(c) for c in dev[it, 1:1 + dev[it, 0]]]
            if drow != r:
                assert b, f"E iteration {it}: device {drow}, oracle {r}"
                skipped += 1
        assert skipped <= 0.01 * len(rows), f"{skipped} of {len(rows)} borderline E iterations differ"
        print(f"{sc}: {skipped} borderline E iterations differ")
    # the serial loops' results
    for k, r in (("h", ref["h"]),) + ((() if ill else (("e", ref["e"]),))):
        assert got[k + "_inliers"] == r["inliers"]
        assert got[k + "_iterations"] == r["iterations"]
        assert got[k + "_best_it"] == r["best_it"]
        np.testing.assert_array_equal(got[k + "_mask"], r["mask"])
    if ill:
        # init_sfm's status there is decided before the essential matrix counts (the homography's pure-rotation test,
        # or the parallax gate), and equals the oracle's above.  The device's E path must still be self-consistent.
        assert ref["status"] in (tv.STATUS_PURE_ROTATION, tv.STATUS_LOW_PARALLAX)
        for k in ("H", "R", "T", "points"):
            assert np.all(np.isfinite(got[k])), k
        ec = got["e_counts"]
        assert 0 <= got["e_best_it"] < got["e_iterations"] <= 1000
        assert 0 <= got["e_best_model"] < ec[got["e_best_it"], 0] <= 10
        assert got["e_inliers"] == ec[got["e_best_it"], 1 + got["e_best_model"]] == int(got["e_mask"].sum())
        assert np.all(ec[: got["e_iterations"], 1:][np.arange(10) >= ec[: got["e_iterations"], :1]] == 0)
        assert 0 <= got["candidate"] < 8 and got["triangulated"] == int(got["point_status"].sum())
        return
    assert got["e_best_model"] == ref["e"]["best_k"]
    assert got["candidate"] == ref["candidate"]
    assert got["triangulated"] == ref["triangulated"]
    np.testing.assert_allclose(got["R"], ref["R"], rtol=0, atol=1e-9)
    np.testing.assert_allclose(got["T"], ref["T"], rtol=0, atol=1e-9)
    np.testing.assert_array_equal(got["point_status"], ref["point_status"])
    st = ref["point_status"]
    scale = np.maximum(np.linalg.norm(ref["points"][st], axis=1, keepdims=True), 1.0)
    assert np.all(np.abs(got["points"][st] - ref["points"][st]) <= 1e-8 * scale)
    assert np.all(got["points"][~st] == 0)


def test_batch_equals_each_problem_alone(ba):
    rng = np.random.default_rng(60)
    kinds = ["general", "plane", "rotation", "small"]
    probs = []
    for i in range(132):
        sc = dict(seed=1000 + i, n=int(rng.choice([0, 3, 5, 40, 80, 150, 400])), outlier_frac=float(rng.uniform(0, 0.5)),
                  kind=kinds[i % 4])
        probs.append(_problem(sc, seed=int(rng.integers(0, 5000)), max_iteration=int(rng.choice([200, 1000]))))
    batch = batch_two_view(ba, probs, diagnostics=True)
    for i, d in enumerate(probs):
        one = batch_two_view(ba, [d], diagnostics=True)[0]
        for k, v in one.items():
            if isinstance(v, np.ndarray):
                np.testing.assert_array_equal(batch[i][k], v, err_msg=f"problem {i} {k}")
            else:
                assert batch[i][k] == v, f"problem {i} {k}"


def test_rejected_calls_change_nothing(ba):
    d = _problem(dict(seed=70, n=100))
    good = two_view(ba, **d)
    bad = [dict(d, fx=0.0), dict(d, confidence=0.0), dict(d, max_iteration=0), dict(d, min_triangulation=-1)]
    for b in bad:
        recs = (_lib.CTwoView * 2)()
        info = np.full(10, 77, np.int32)
        p1 = np.ascontiguousarray(d["p1"])
        p2 = np.ascontiguousarray(d["p2"])
        for r, src in zip(recs, (d, b)):
            r.n_matches, r.seed, r.p1, r.p2 = 100, 648, _lib.ptr(p1), _lib.ptr(p2)
            r.fx, r.fy, r.min_matches, r.min_triangulation = src["fx"], d["fy"], 50, src.get("min_triangulation", 20)
            r.min_parallax, r.confidence, r.max_iteration = 10.0, src.get("confidence", 0.999), src.get("max_iteration", 1000)
            r.info = _lib.ptr(info)
        assert ba.lib.pvio_b200_batch_two_view(ba.h, 2, recs) == EINVAL
        assert np.all(info == 77)
    recs = (_lib.CTwoView * 1)()
    recs[0].n_matches, recs[0].fx, recs[0].fy, recs[0].confidence, recs[0].max_iteration = 10, 400.0, 400.0, 0.9, 10
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 1, recs) == EINVAL            # NULL keypoints with n > 0
    recs[0].n_matches = -1
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 1, recs) == EINVAL
    assert ba.lib.pvio_b200_batch_two_view(ba.h, -1, recs) == EINVAL
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 0, None) == 0
    # the call's limits: at most 65535 problems, at most 2^31 - 1 matches in all (the keypoints are never read)
    p1 = np.ascontiguousarray(d["p1"])
    many = (_lib.CTwoView * 65536)()
    for r in many:
        r.fx, r.fy, r.confidence, r.max_iteration = 400.0, 400.0, 0.9, 10
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 65536, many) == EINVAL
    big = (_lib.CTwoView * 128)()
    for r in big:
        r.n_matches, r.p1, r.p2 = 1 << 24, _lib.ptr(p1), _lib.ptr(p1)
        r.fx, r.fy, r.confidence, r.max_iteration = 400.0, 400.0, 0.9, 10
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 128, big) == EINVAL
    big[0].n_matches = (1 << 24) + 1
    assert ba.lib.pvio_b200_batch_two_view(ba.h, 1, big) == EINVAL
    again = two_view(ba, **d)
    for k, v in good.items():
        if isinstance(v, np.ndarray):
            np.testing.assert_array_equal(again[k], v)
        else:
            assert again[k] == v
