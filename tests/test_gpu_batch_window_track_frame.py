"""pvio_b200_batch_window_track_frame: the start of SlidingWindowTracker::track on resident inertial slots -- integrate
the new frame's samples, predict its state, PnP + triangulation as localize, the keyframe check, and the merged record
after a non-keyframe -- with the slot's newest frame as map->last_frame().  Checked against pvio_b200_preintegrate,
tracker_oracle.predict, localize and tracker_oracle.keyframe_check, and along whole sequences against a host twin."""
import numpy as np
import pytest

from oracle import lie, tracker_oracle
from pvio_b200 import _lib, imu
from pvio_b200.batch_window import BatchWindows, Edit, Localize, TrackFrame
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200._lib import EINVAL
from synthetic.sequence import BatchPlayer, Run
from test_gpu_batch_window_localize import _downloads, _given_point, _near_threshold, _cam_matrix, _same_download

pytestmark = pytest.mark.gpu
SEQ_TOL = 2e-6
CX, CY = 376.0, 240.0


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _samples(run, f, first=None):
    """the raw samples of the factors from absolute frame `first` (default f - 1) to f back to back, and f's time"""
    fs = run.truth.imu_factors
    first = f - 1 if first is None else first
    return np.concatenate([fs[k][0] for k in range(first, f)]), fs[f - 1][1]


def _track(p, j, f, newest_abs, kf=True, skipped=0, samples=None, obs=True, born=True, prev=None):
    """the TrackFrame of absolute frame f of run j after the slot's newest frame newest_abs: its samples (the newest
    frame's own, from the window frame before it, `prev`, as the merge list when it is not a keyframe), its keypoints
    on live tracks and the tracks born in it"""
    run = p.runs[j]
    s, t = _samples(run, f) if samples is None else samples
    merge = None if kf else _samples(run, newest_abs, prev)[0]
    T = TrackFrame(p.slots[j], s, t, run.truth.imu_noise, CX, CY, kf, merge, skipped)
    obs_l, new_l = [], []
    for l, (fr, zs) in enumerate(run.tracks):
        if f not in fr:
            continue
        z = zs[fr.index(f)]
        if l in p.ids[j]:
            if obs:
                T.observe(p.ids[j][l], z, _given_point(run, l) if p.roles[j].get(l, -1) != -1 else None)
                obs_l.append(l)
        elif born and newest_abs in fr:
            T.born(zs[fr.index(newest_abs)], z)
            new_l.append(l)
    return T, obs_l, new_l


def _host_records(ba, T, newest16):
    """pvio_b200_preintegrate at the newest frame's biases: the step-1 record and, after a non-keyframe, the merged one"""
    bg, bav = newest16[10:13].copy(), newest16[13:16].copy()
    fs = [(T.samples, T.t_end, bg, bav)]
    if T.merge is not None:
        fs.append((np.concatenate([T.merge, T.samples]), T.t_end, bg, bav))
    recs = imu.preintegrate(ba, fs, [n.reshape(3, 3) for n in T.noise])
    return recs[0], (recs[1] if T.merge is not None else recs[0])


def _oracle_check(run, model, T, rec1, frame_i, newest, skipped):
    """tracker_oracle.keyframe_check of a record from the slot's host model (keypoints per window frame)"""
    zi, zj = [], []
    for tid, z, _ in T.obs:
        t = model.tracks[tid]
        if frame_i in t["frames"]:
            zi.append(t["zs"][t["frames"].index(frame_i)]); zj.append(z)
    if frame_i == newest:
        for a, b in T.new:
            zi.append(a); zj.append(b)
    w = run.w
    return tracker_oracle.keyframe_check(zi, zj, rec1[1:5], w.cam_q_cs, w.imu_q_cs, w.K_fx, w.K_fy, CX, CY, skipped)


RUNS = [dict(F=20, N=6, M=220, seed=760), dict(F=20, N=8, M=240, seed=762, planes=2), dict(F=20, N=9, M=260, seed=764),
        dict(F=20, N=2, M=150, seed=766)]


@pytest.fixture(scope="module")
def setup():
    """four resident inertial slots (N = 6, 8 with planes, 9, 2) after their first solve; slot 4 is visual-only"""
    runs = [Run(**kw) for kw in RUNS]
    ba = BundleAdjustor(max_windows=6, max_frames=9, max_landmarks=400, max_obs=3000)
    player = BatchPlayer(ba, runs)
    w = runs[0].w
    use = w.use_inertial
    w.use_inertial = False
    player.bw.reset(4, w)
    w.use_inertial = use
    edits = []                      # the tracks first seen in the newest frame leave: they are born in the next frame
    for j, r in enumerate(player.runs):
        e = Edit(player.slots[j])
        e.remove = [player.ids[j].pop(l) for l in sorted(player.ids[j]) if r.tracks[l][0][0] == r.N - 1]
        edits.append(e)
    player.bw.edit(edits)
    player.model.edit(edits)
    player.bw.solve(list(range(4)), max_iterations=4)
    yield ba, player
    ba.close()


def _frame(p, j):
    run = p.runs[j]
    return p.k[j] + run.N, p.k[j] + run.N - 1


# ------------------------------------------------------------------------ 1, 2: records and prediction
@pytest.mark.parametrize("kind", ["one", "own", "long"])
@pytest.mark.parametrize("kf", [True, False], ids=["keyframe", "nonkey"])
def test_records_and_prediction(setup, kind, kf):
    """imu_record equals pvio_b200_preintegrate at the newest frame's downloaded biases bit for bit (the new frame's own
    list after a keyframe, the merged list otherwise) for 1, 50 and 400 samples and N = 2, 6, 8, 9; predicted equals
    tracker_oracle.predict from the downloaded newest state and the step-1 record within 1e-13 max(1, |x|)"""
    ba, p = setup
    js = [0, 1, 2, 3]
    recs = []
    for j in js:
        f, newest = _frame(p, j)
        s, t = _samples(p.runs[j], f + 7, f - 1) if kind == "long" else _samples(p.runs[j], f)
        if kind == "one":
            s = s[:1]
        recs.append(_track(p, j, f, newest, kf=kf, samples=(s, t))[0])
    assert {len(r.samples) for r in recs} == {dict(one=1, own=50, long=400)[kind]}
    ds = p.bw.download([p.slots[j] for j in js], 400)
    out = p.bw.track_frame(recs)
    for T, d, o in zip(recs, ds, out):
        rec1, edit = _host_records(ba, T, d["frames"][-1])
        assert np.array_equal(_bits(o["imu_record"]), _bits(edit))
        want = tracker_oracle.predict(d["frames"][-1], rec1)
        assert np.all(np.abs(o["predicted"] - want) <= 1e-13 * np.maximum(1.0, np.abs(want)))


# ------------------------------------------------------------------------ 3: PnP and triangulation as localize
@pytest.mark.parametrize("js", [[1], [0, 1, 2]], ids=["n1", "n3"])
def test_pnp_and_triangulation_equal_localize(setup, js):
    """localize fed the call's predicted state and pvio_b200_preintegrate's record: the same iterations, accepted steps
    and termination, states and costs within 1e-12, the same validity and inverse depths within 1e-9"""
    ba, p = setup
    recs = [_track(p, j, *_frame(p, j))[0] for j in js]
    ds = p.bw.download([p.slots[j] for j in js], 400)
    out = p.bw.track_frame(recs)
    locs = []
    for T, d, o in zip(recs, ds, out):
        rec1, _ = _host_records(ba, T, d["frames"][-1])
        L = Localize(T.slot, o["predicted"], rec1)
        L.obs, L.new = T.obs, T.new
        locs.append(L)
    ref = p.bw.localize(locs)
    checked = 0
    for j, T, d, o, r in zip(js, recs, ds, out, ref):
        for k in ("iterations", "accepted_steps", "termination", "usable"):
            assert o["summary"][k] == r["summary"][k], k
        for k in ("initial_cost", "final_cost"):
            assert abs(o["summary"][k] - r["summary"][k]) <= 1e-12 * abs(r["summary"][k]), k
        assert np.abs(o["state"] - r["state"]).max() <= 1e-12 * max(np.abs(r["state"]).max(), 1.0)
        assert np.array_equal(np.isnan(o["points"]), np.isnan(r["points"]))
        run = p.runs[j]
        Ps = (_cam_matrix(run, d["frames"][-1])[0], _cam_matrix(run, r["state"])[0])
        for t in range(len(T.new)):
            if _near_threshold(Ps, T.new[t]):
                continue
            checked += 1
            assert o["valid"][t] == r["valid"][t], t
            if r["valid"][t]:
                assert abs(o["inv_depth"][t] - r["inv_depth"][t]) <= 1e-9 * abs(r["inv_depth"][t])
                assert abs(o["inv_depth_next"][t] - r["inv_depth_next"][t]) <= 1e-9 * abs(r["inv_depth_next"][t])
    assert checked > 0


# ------------------------------------------------------------------------ 4: keyframe check
def _crafted(ba, p, j, pars, kf=True, skipped=0, obs=False):
    """a record of slot j whose new tracks (born) give exactly the parallaxes `pars` when frame_i is the newest frame"""
    f, newest = _frame(p, j)
    T = _track(p, j, f, newest, kf=kf, skipped=skipped, obs=obs, born=False)[0]
    d = p.bw.download([p.slots[j]], 400)[0]
    rec1, _ = _host_records(ba, T, d["frames"][-1])
    w = p.runs[j].w
    q = lie.qmul(lie.qmul(lie.qmul(lie.qmul(lie.qconj(w.cam_q_cs), w.imu_q_cs), rec1[1:5]), lie.qconj(w.imu_q_cs)), w.cam_q_cs)
    qij = lie.qconj(q)
    rng = np.random.default_rng(len(pars) + skipped)
    for P in pars:
        zi = rng.uniform(-0.3, 0.3, 2)
        y = lie.qrot(qij, np.array([zi[0], zi[1], 1.0]))
        T.born(zi, y[:2] / y[2] + np.array([P / w.K_fx, 0.0]))
    return T, rec1


def _pcts(m, P):
    """m parallaxes whose element m * 4 / 5 in ascending order is P"""
    k = m * 4 // 5
    return np.concatenate([np.linspace(0.2 * P, 0.9 * P, k), np.full(m - k, P)])


CASES = [("p30", _pcts(80, 30.0), 0, False), ("p49.9", _pcts(80, 49.9), 0, False), ("p50.1", _pcts(80, 50.1), 0, True),
         ("p80", _pcts(80, 80.0), 0, True), ("m49", np.full(49, 5.0), 3, True), ("m50", np.full(50, 5.0), 3, False),
         ("skip9", np.full(60, 30.0), 9, False), ("skip10", np.full(60, 30.0), 10, True),
         ("skip11", np.full(60, 30.0), 11, True), ("m5000", _pcts(5000, 42.0), 2, False)]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_keyframe_check_on_crafted_lists(setup, case):
    ba, p = setup
    _, pars, skipped, want_kf = case
    j = 0
    T, rec1 = _crafted(ba, p, j, pars, skipped=skipped)
    N = p.runs[j].N
    o = p.bw.track_frame([T])[0]
    kf, par, m, sk = _oracle_check(p.runs[j], p.model.m[p.slots[j]], T, rec1, N - 1, N - 1, skipped)
    assert (o["keyframe"], o["n_parallax"], o["skipped_frames"]) == (kf, m, sk) and m == len(pars)
    assert kf == want_kf
    if m < 50:
        assert np.isnan(o["parallax"]) and np.isnan(par)
    else:
        assert abs(o["parallax"] - par) <= 1e-12 * par


def test_keyframe_check_after_a_non_keyframe(setup):
    """newest frame not a keyframe: frame_i is frame N - 2, observed tracks without a keypoint there are left out and
    the new tracks do not count (they have their keypoint in the newest frame)"""
    ba, p = setup
    for j in (0, 2):
        f, newest = _frame(p, j)
        T = _track(p, j, f, newest, kf=False)[0]
        N = p.runs[j].N
        model = p.model.m[p.slots[j]]
        n_out = sum(1 for tid, _, _ in T.obs if N - 2 not in model.tracks[tid]["frames"])
        assert len(T.new) > 0
        d = p.bw.download([p.slots[j]], 400)[0]
        rec1, _ = _host_records(ba, T, d["frames"][-1])
        o = p.bw.track_frame([T])[0]
        kf, par, m, sk = _oracle_check(p.runs[j], model, T, rec1, N - 2, N - 1, 0)
        assert m == len(T.obs) - n_out
        assert (o["keyframe"], o["n_parallax"], o["skipped_frames"]) == (kf, m, sk)
        assert (np.isnan(o["parallax"]) and np.isnan(par)) or abs(o["parallax"] - par) <= 1e-12 * par


# ------------------------------------------------------------------------ 5: no writes, rejections
def test_no_slot_changes(setup):
    ba, p = setup
    before = _downloads(p.bw, [0, 1, 2, 3, 4], 400)
    imu_before = p.bw.imu_records([0, 1, 2, 3])
    p.bw.track_frame([_track(p, j, *_frame(p, j), kf=(j % 2 == 0))[0] for j in range(4)])
    assert _same_download(before, _downloads(p.bw, [0, 1, 2, 3, 4], 400))
    assert all(np.array_equal(_bits(a), _bits(b)) for a, b in zip(imu_before, p.bw.imu_records([0, 1, 2, 3])))


def _arr(keep, a):
    a = np.ascontiguousarray(a)
    keep.append(a)
    return _lib.ptr(a)


def _sp_visual(r, keep):
    r.slot, r.n_obs, r.n_new = 4, 0, 0


def _sp_no_samples(r, keep):
    r.n_samples = 0


def _sp_sample(r, keep):
    s = np.ctypeslib.as_array(r.samples, shape=(r.n_samples, 7)).copy()
    s[3, 4] = np.nan
    r.samples = _arr(keep, s)


def _sp_t_end(r, keep):
    r.t_end = np.inf


def _sp_noise(r, keep):
    n = np.ctypeslib.as_array(r.noise_cov, shape=(36,)).copy()
    n[30] = np.nan
    r.noise_cov = _arr(keep, n)


def _sp_cx(r, keep):
    r.cy = np.nan


def _sp_flag(r, keep):
    r.newest_is_keyframe = 2


def _sp_no_merge(r, keep):
    r.newest_is_keyframe, r.n_merge, r.merge_samples = 0, 0, None


def _sp_merge_given(r, keep):
    r.n_merge, r.merge_samples = r.n_samples, r.samples


def _sp_skipped_null(r, keep):
    r.skipped_frames = None


def _sp_skipped_negative(r, keep):
    r.skipped_frames = _arr(keep, np.array([-1], dtype=np.int32))


def _sp_unknown_track(r, keep):
    t = np.ctypeslib.as_array(r.obs_track, shape=(r.n_obs,)).copy()
    t[0] = 10 ** 6
    r.obs_track = _arr(keep, t)


def _sp_record_null(r, keep):
    r.imu_record = None


SPOILERS = [_sp_visual, _sp_no_samples, _sp_sample, _sp_t_end, _sp_noise, _sp_cx, _sp_flag, _sp_no_merge,
            _sp_merge_given, _sp_skipped_null, _sp_skipped_negative, _sp_unknown_track, _sp_record_null]


@pytest.mark.parametrize("spoil", SPOILERS, ids=[s.__name__[4:] for s in SPOILERS])
def test_rejections_change_nothing(setup, spoil):
    ba, p = setup
    built = [_track(p, j, *_frame(p, j))[0] for j in (0, 2)]
    recs, sms, out, keep = BatchWindows.track_frame_records(built)
    for o in out:
        for k in ("state", "points", "predicted", "imu_record", "parallax", "inv_depth", "inv_depth_next"):
            o[k][...] = 7.0
        o["valid"][...] = 7
        o["keyframe"][...] = 7
        o["n_parallax"][...] = 7
        o["skipped_frames"][...] = 3
    for s in sms:
        s.iterations = 777
    spoil(recs[1], keep)
    before = _downloads(p.bw, [0, 1, 2, 3, 4], 400)
    n0 = ba.kernel_launches
    assert ba.lib.pvio_b200_batch_window_track_frame(ba.h, 2, recs, None) == EINVAL
    assert ba.kernel_launches == n0
    for o, s in zip(out, sms):
        for k in ("state", "points", "predicted", "imu_record", "parallax", "inv_depth", "inv_depth_next"):
            assert np.all(o[k] == 7.0), k
        assert np.all(o["valid"] == 7) and o["keyframe"][0] == 7 and o["n_parallax"][0] == 7
        assert o["skipped_frames"][0] == 3 and s.iterations == 777
    assert _same_download(before, _downloads(p.bw, [0, 1, 2, 3, 4], 400))
    p.bw.track_frame(built)                                           # the handle is still usable


def test_non_keyframe_needs_two_frames(setup):
    ba, p = setup
    f, newest = _frame(p, 3)
    T = _track(p, 3, f, newest, kf=False)[0]
    one = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=400, max_obs=3000)
    try:
        bw = BatchWindows(one)
        bw.reset(0, p.runs[3].w)
        bw.edit([Edit(0).frame(np.concatenate([p.runs[3].guess.q[0], p.runs[3].guess.p[0], p.runs[3].guess.v[0],
                                               p.runs[3].guess.bg[0], p.runs[3].guess.ba[0]]))])
        T.slot, T.obs, T.new = 0, [], []
        with pytest.raises(PvioB200Error):
            bw.track_frame([T])
        T.newest_is_keyframe, T.merge = True, None
        assert len(bw.track_frame([T])) == 1
    finally:
        one.close()


# ------------------------------------------------------------------------ 6: launches
def test_launches_independent_of_n(setup):
    ba, p = setup
    counts = []
    for js in ([0], [0, 1, 2, 3]):
        recs = [_track(p, j, *_frame(p, j), kf=(j != 1))[0] for j in js]
        n0 = ba.kernel_launches
        p.bw.track_frame(recs)
        counts.append(ba.kernel_launches - n0)
    assert counts[0] == counts[1] <= 5
    n0 = ba.kernel_launches
    assert p.bw.track_frame([]) == [] and ba.kernel_launches == n0


# ------------------------------------------------------------------------ 7: sequences
class _Twin:
    """one way of running the tracking cycle on the slots of a BatchPlayer with raw samples: `device` takes each frame's
    records, prediction, PnP and keyframe decision from track_frame, otherwise from pvio_b200_preintegrate,
    tracker_oracle.predict, localize and tracker_oracle.keyframe_check"""

    def __init__(self, ba, kws, slots, device):
        self.ba, self.device = ba, device
        self.p = BatchPlayer(ba, [Run(**kw) for kw in kws], slots=slots)
        self.win = [list(range(r.N)) for r in self.p.runs]            # absolute frame of each window frame
        self.newest_kf = [True] * len(kws)
        self.skipped = [0] * len(kws)

    def step(self, js):
        p = self.p
        built = []
        for j in js:
            f, newest = self.win[j][-1] + 1, self.win[j][-1]
            built.append(_track(p, j, f, newest, kf=self.newest_kf[j], skipped=self.skipped[j], prev=self.win[j][-2]))
        res = []
        if self.device:
            for (T, _, _), o in zip(built, p.bw.track_frame([b[0] for b in built])):
                res.append(o)
        else:
            ds = p.bw.download([p.slots[j] for j in js], 400)
            locs, recs = [], []
            for (T, _, _), d in zip(built, ds):
                rec1, edit = _host_records(self.ba, T, d["frames"][-1])
                L = Localize(T.slot, tracker_oracle.predict(d["frames"][-1], rec1), rec1)
                L.obs, L.new = T.obs, T.new
                locs.append(L)
                recs.append((rec1, edit))
            for j, (T, _, _), o, (rec1, edit) in zip(js, built, p.bw.localize(locs), recs):
                N = len(self.win[j])
                kf, par, m, sk = _oracle_check(p.runs[j], p.model.m[p.slots[j]], T, rec1,
                                               N - 1 if self.newest_kf[j] else N - 2, N - 1, self.skipped[j])
                o.update(imu_record=edit, keyframe=kf, parallax=par, n_parallax=m, skipped_frames=sk)
                res.append(o)
        self.apply(js, built, res)
        return res

    def apply(self, js, built, res):
        """append after a keyframe newest frame (drop first when the window is full, then solve), replace the newest
        frame otherwise (the merged record).  The factors keep the records the calls return: re-integrating them before
        each solve (set_imu) amplifies rounding differences between the two paths by 1e3 to 1e5 per keyframe on these
        synthetic runs (DESIGN 9), beyond the 2e-6 bar"""
        p = self.p
        app = [j for j in js if self.newest_kf[j]]
        full = [j for j in app if len(self.win[j]) == p.runs[j].N]
        if full:
            p.bw.drop_victim([p.slots[j] for j in full])
            p.model.drop_victim([p.slots[j] for j in full])
            p.refresh(full, 400)                                      # tracks the drop ended leave the edit
            for j in full:
                self.win[j].pop(0)
        edits, born = [], []
        for j, (T, obs_l, new_l), o in zip(js, built, res):
            run, replace = p.runs[j], not self.newest_kf[j]
            f, N = self.win[j][-1] + 1, len(self.win[j])
            e = Edit(p.slots[j], replace).frame(o["state"], False, o["imu_record"])
            fw = N - 1 if replace else N
            tr = p.model.m[p.slots[j]].tracks              # a replace ends the tracks seen in the erased frame only
            for l in (l for l in obs_l if l in p.ids[j] and not (replace and tr[p.ids[j][l]]["frames"] == [N - 1])):
                e.obs.append((p.ids[j][l], fw, run.tracks[l][1][run.tracks[l][0].index(f)]))
            ls = []
            for (zl, zn), v, r, rn, l in zip(T.new, o["valid"], o["inv_depth"], o["inv_depth_next"], new_l):
                if v:
                    e.new.append((N - 1, zn, rn) if replace else (N - 1, zl, r))
                    ls.append(l)
            edits.append(e)
            born.append(ls)
            if replace:
                self.win[j][-1] = f
            else:
                self.win[j].append(f)
        got = p.bw.edit(edits)
        p.model.edit(edits)
        follow = []
        for j, e, ls, ids in zip(js, edits, born, got):
            fe = Edit(p.slots[j])
            for l, i in zip(ls, ids):
                p.ids[j][l], p.roles[j][l] = int(i), -1
                if not e.replace_last:
                    f = self.win[j][-1]
                    fe.obs.append((int(i), len(self.win[j]) - 1, p.runs[j].tracks[l][1][p.runs[j].tracks[l][0].index(f)]))
            follow.append(fe)
        p.bw.edit(follow)
        p.model.edit(follow)
        if app:
            p.bw.solve([p.slots[j] for j in app], max_iterations=10)
        p.refresh(js, 400)
        for j, o in zip(js, res):
            self.newest_kf[j], self.skipped[j] = bool(o["keyframe"]), int(o["skipped_frames"])


def test_sequences_follow_the_host_twin():
    """4 inertial sequences (N = 6, 8, 9, 6; the second with planes): the device path is driven by track_frame's own
    decisions only (a keyframe: the next frame is appended; a non-keyframe: the next frame replaces it with the merged
    record), a host twin runs the same cycle with pvio_b200_preintegrate, tracker_oracle.predict, localize and
    tracker_oracle.keyframe_check; they agree on every decision, iteration count and landmark set, states within 2e-6"""
    kws = [dict(F=40, N=6, M=220, seed=780), dict(F=40, N=8, M=260, seed=782, planes=2),
           dict(F=40, N=9, M=260, seed=784), dict(F=40, N=6, M=220, seed=786)]
    ba = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=400, max_obs=3000)
    twins = [_Twin(ba, kws, list(range(4)), True), _Twin(ba, kws, list(range(4, 8)), False)]
    for t in twins:
        t.p.bw.solve(t.p.slots, max_iterations=10)
    worst, decisions, keyframes = 0.0, {True: 0, False: 0}, [0] * 4
    while min(keyframes) < 11:
        js = [j for j in range(4) if twins[0].win[j][-1] + 2 < kws[j]["F"]]
        if not js:
            break
        rd, rh = twins[0].step(js), twins[1].step(js)
        for j, a, b in zip(js, rd, rh):
            assert a["keyframe"] == b["keyframe"] and a["n_parallax"] == b["n_parallax"], j
            assert a["skipped_frames"] == b["skipped_frames"], j
            assert a["summary"]["iterations"] == b["summary"]["iterations"], j
            assert np.array_equal(a["valid"], b["valid"]), j
            worst = max(worst, np.abs(a["state"] - b["state"]).max())
            assert np.abs(a["state"] - b["state"]).max() < SEQ_TOL, j
            decisions[a["keyframe"]] += 1
            keyframes[j] += a["keyframe"]
        assert [dict(twins[0].p.ids[j]) for j in range(4)] == [dict(twins[1].p.ids[j]) for j in range(4)]
        for a, b in zip(twins[0].p.bw.download(twins[0].p.slots, 400), twins[1].p.bw.download(twins[1].p.slots, 400)):
            assert np.array_equal(a["ids"], b["ids"])
            worst = max(worst, np.abs(a["frames"] - b["frames"]).max())
            assert np.abs(a["frames"] - b["frames"]).max() < SEQ_TOL
    print(f"largest state difference between the two paths: {worst:.3e}; keyframes {decisions[True]}, "
          f"non-keyframes {decisions[False]}; keyframes per sequence {keyframes}")
    assert min(keyframes) >= 11 and decisions[True] >= 3 and decisions[False] >= 3
    ba.close()
