"""IMU samples kept on the device with their factors in the resident slots (pvio_b200_batch_window_set_imu): every factor
that holds samples is re-integrated at its first frame's current biases before each solve, as BundleAdjustor::solve
re-integrates the window's factors (bundle_adjustor.cpp:220-231)."""
import ctypes as C

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import imu_oracle
from pvio_b200 import _lib, imu
from pvio_b200.batch_window import BatchWindows, Imu
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200._lib import EINVAL
from synthetic import synth
from synthetic.sequence import BatchPlayer, Chain, Run

pytestmark = pytest.mark.gpu
SEQ_TOL = 2e-6


def _noise(run):
    return run.truth.imu_noise


def _expected(ba, frames, lists, noise):
    """pvio_b200_preintegrate of each (frame i, samples, t_end) at frame i's biases in `frames`"""
    fs = [(s, t, frames[i][10:13].copy(), frames[i][13:16].copy()) for i, s, t in lists]
    return imu.preintegrate(ba, fs, noise)


def _factor(run, g, first=None):
    """samples of the factors from absolute frame `first` (default g - 1) to g back to back, and the time of frame g"""
    fs = run.truth.imu_factors
    first = g - 1 if first is None else first
    return np.concatenate([fs[k][0] for k in range(first, g)]), fs[g - 1][1]


def _bits(a):
    """bit patterns: a degenerate factor (one sample) has a singular covariance and NaN in its square-root information"""
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


def _frames(bw, slots):
    return [d["frames"] for d in bw.download(slots, 400)]


# ------------------------------------------------------------------------ 1: records
def test_records_equal_preintegrate_bit_for_bit():
    """Slots with N = 2, 3, 6, 9 and factors of 1, 50 and 400 samples: after a solve every factor with samples holds
    pvio_b200_preintegrate of its samples at its first frame's pre-solve biases, bit for bit; a factor without samples
    keeps its edit record bit for bit; and one factor matches the fp64 oracle."""
    runs = [Run(F=12, N=2, M=120, seed=740), Run(F=12, N=3, M=150, seed=741), Run(F=14, N=6, M=200, seed=742),
            Run(F=16, N=9, M=260, seed=743)]
    ba = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=400, max_obs=3000)
    p = BatchPlayer(ba, runs)
    # per slot: window frame -> its list: "own" (the factor's 50 samples), "one" (its first sample only, integrated
    # up to the frame), "long" (400: the eight factors from absolute frame 1 to 9), "ragged" (own, uneven times)
    plan = {0: {1: "long"}, 1: {1: "one", 2: "own"}, 2: {2: "own", 4: "long", 5: "ragged"},
            3: {1: "one", 2: "own", 3: "long", 7: "own"}}
    recs, lists = [], {j: [] for j in range(4)}
    for j, fr in plan.items():
        run = runs[j]
        for f, kind in fr.items():
            s, t = _factor(run, 9, 1) if kind == "long" else _factor(run, f)
            if kind == "one":
                s = s[:1]
            elif kind == "ragged":
                s = s.copy()
                s[1::3, 0] += 1e-3
            recs.append(Imu(j, f, s, t, _noise(run)))
            lists[j].append((f - 1, s, t))
    assert {len(r.samples) for r in recs} == {1, 50, 400}
    p.bw.set_imu(recs)
    before = p.bw.imu_records(range(4))
    frames = _frames(p.bw, range(4))
    want = {j: _expected(ba, frames[j], lists[j], _noise(runs[j])) for j in range(4) if lists[j]}
    p.bw.solve(list(range(4)), max_iterations=4)
    got = p.bw.imu_records(range(4))
    for j in range(4):
        assert got[j].shape == (runs[j].N - 1, 288)
        held = set(plan[j])
        for k, (i, _, _) in enumerate(lists[j]):
            assert np.array_equal(_bits(got[j][i]), _bits(want[j][k])), (j, i)
        for f in range(1, runs[j].N):
            if f not in held:                              # no samples: the edit record, untouched
                assert np.array_equal(_bits(got[j][f - 1]), _bits(before[j][f - 1])), (j, f)
                assert np.array_equal(_bits(got[j][f - 1]), _bits(p.rec[j][f - 1])), (j, f)
    assert np.isnan(got[1][0][11:236]).any()               # the one-sample factor, as the reference's would be
    # one factor (slot 3, frame 3, 400 samples) against the oracle
    _, s, t = lists[3][2]
    bg, bav = frames[3][2][10:13], frames[3][2][13:16]
    ref = imu_oracle.record(imu_oracle.integrate(s, t, bg, bav, *_noise(runs[3])), bg, bav)
    r = got[3][2]
    for a, b in ((0, 11), (236, 281)):                     # deltas and bias Jacobians
        assert np.max(np.abs(r[a:b] - ref[a:b])) <= 1e-12 * np.max(np.abs(ref[a:b]))
    assert np.array_equal(r[281:287], ref[281:287])
    U, U0 = r[11:236].reshape(15, 15), ref[11:236].reshape(15, 15)
    assert np.max(np.abs(U - U0)) <= 1e-7 * np.max(np.abs(U0))   # the square-root information: test_gpu_imu's bar
    ba.close()


# ------------------------------------------------------------------------ 2: oracle
def test_solve_matches_the_oracle_at_the_presolve_biases():
    """One cfg3 window in a resident slot whose states carry biases away from those its edit records were integrated
    at: the slot solves with its factors re-integrated at the pre-solve biases, as ba_oracle.solve does with records
    imu_oracle integrates there -- the same iterations, accepted steps and termination, states within 1e-5."""
    w, st, truth = synth.make_cfg3(N=9, M=150, seed=745)
    rng = np.random.default_rng(745)
    st.bg = st.bg + rng.normal(0, 2e-3, 3)
    st.ba = st.ba + rng.normal(0, 5e-2, 3)
    assert np.array_equal(w.prior_frames, np.arange(w.n_prior))
    ba = BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=160, max_obs=2000)
    bw = BatchWindows(ba)
    bw.reset(1, w)
    rec = _lib.PackedArgs(w, st).keep["imu"].reshape(-1, 288)          # integrated at the edit-time biases
    from pvio_b200.batch_window import Edit
    ids = {}
    for f in range(w.N):
        x = np.concatenate([st.q[f], st.p[f], st.v[f], st.bg[f], st.ba[f]])
        e = Edit(1).frame(x, bool(w.frame_fixed[f]), rec[f - 1] if f > 0 else None)
        new = []
        for l in range(w.M):
            if int(w.lm_anchor[l]) == f:
                e.new.append((f, w.lm_z_ref[l], st.rho[l])); new.append(l)
            for k in range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1]):
                if int(w.obs_frame[k]) == f:
                    e.obs.append((ids[l], f, w.obs_z[k]))
        for l, i in zip(new, bw.edit([e])[0]):
            ids[l] = int(i)
    x0 = np.concatenate([w.prior_q0, w.prior_p0, w.prior_v0, w.prior_bg0, w.prior_ba0], axis=1)
    bw.set_prior(1, w.prior_S, w.prior_e, x0)
    bw.set_imu([Imu(1, f, truth.imu_factors[f - 1][0], truth.imu_factors[f - 1][1], truth.imu_noise)
                for f in range(1, w.N)])
    sm = bw.solve([1], max_iterations=10, postpass=False)[0]
    d = bw.download([1], 160)[0]
    # the oracle's window: records at the pre-solve biases
    refs = [imu_oracle.record(imu_oracle.integrate(s, t, st.bg[i], st.ba[i], *truth.imu_noise), st.bg[i], st.ba[i])
            for i, (s, t, _, _) in enumerate(truth.imu_factors)]
    _set_records(w, np.array(refs))
    ref_st, ref_sum = bo.solve(w, st, max_iter=10)
    assert sm["iterations"] == ref_sum["iterations"]
    assert sm["accepted_steps"] == sum(ref_sum["accepted"])
    assert (sm["termination"] == 0) == (ref_sum["termination"] == "CONVERGENCE")
    fr = d["frames"]
    move = np.linalg.norm(ref_st.p - st.p)
    assert np.linalg.norm(fr[:, 4:7] - ref_st.p) < 1e-5 * max(move, 1e-3) + 1e-9
    for a, b, ref, x in ((0, 4, ref_st.q, st.q), (7, 10, ref_st.v, st.v), (10, 13, ref_st.bg, st.bg), (13, 16, ref_st.ba, st.ba)):
        assert np.linalg.norm(fr[:, a:b] - ref) < 1e-5 * max(np.linalg.norm(ref - x), 1e-3) + 1e-9
    row = {int(t): r for r, t in enumerate(d["ids"])}
    rho = np.array([d["inv_depth"][row[ids[l]]] for l in range(w.M)])
    assert np.linalg.norm(rho - ref_st.rho) < 1e-5 * np.linalg.norm(ref_st.rho - st.rho) + 1e-9
    ba.close()


def _set_records(w, rec):
    w.imu_dt, w.imu_dq, w.imu_dp, w.imu_dv = rec[:, 0].copy(), rec[:, 1:5].copy(), rec[:, 5:8].copy(), rec[:, 8:11].copy()
    w.imu_sqrt_inv_cov = rec[:, 11:236].reshape(-1, 15, 15).copy()
    for k, a in (("dq_dbg", 236), ("dp_dbg", 245), ("dp_dba", 254), ("dv_dbg", 263), ("dv_dba", 272)):
        setattr(w, "imu_" + k, rec[:, a:a + 9].reshape(-1, 3, 3).copy())
    w.imu_bg0, w.imu_ba0 = rec[:, 281:284].copy(), rec[:, 284:287].copy()


# ------------------------------------------------------------------------ 3: bookkeeping
def test_samples_follow_drops_replacements_and_growth():
    """A drop shifts every factor's samples with its frame, a replace_last and a set_imu with the merged list give the
    merged factor; growing the sample stride through one slot leaves another slot's samples; window_solve on slot 0
    re-integrates too."""
    runs = [Run(F=16, N=6, M=200, seed=750), Run(F=16, N=8, M=240, seed=751), Run(F=16, N=6, M=200, seed=752)]
    ba = BundleAdjustor(max_windows=3, max_frames=8, max_landmarks=400, max_obs=3000)
    p = BatchPlayer(ba, runs, imu_samples=True)
    p.imu_samples = False                                  # the edits below name their samples themselves
    lists = {j: [(f - 1,) + _factor(r, f) for f in range(1, r.N)] for j, r in enumerate(runs)}

    def check(js, solve):
        frames = _frames(p.bw, js)
        want = [_expected(ba, fr, [(i, s, t) for i, s, t in lists[j]], _noise(runs[j])) for j, fr in zip(js, frames)]
        solve()
        for j, wj, g in zip(js, want, p.bw.imu_records(js)):
            assert np.array_equal(_bits(g[:len(wj)]), _bits(wj)), j

    check([0, 1, 2], lambda: p.bw.solve([0, 1, 2], max_iterations=3))
    # drop in slots 0 and 1: their lists shift; then slot 0's newest frame is replaced by the next one (merged samples)
    p.bw.drop_victim([0, 1])
    p.model.drop_victim([0, 1])
    p.refresh([0, 1], 400)
    p.k[0] += 1; p.k[1] += 1
    for j in (0, 1):
        lists[j] = [(i - 1, s, t) for i, s, t in lists[j][1:]]
    r0, N0 = runs[0], runs[0].N
    g = p.k[0] + N0 - 1                                    # a non-keyframe g, then g + 1 replaces it at index N0 - 1
    fake = p.frame_edit(0, g, N0 - 1)
    p._apply([fake], [0])
    p.bw.set_imu([Imu(0, N0 - 1, *_factor(r0, g), _noise(r0))])
    for l in fake.landmarks:                               # its new tracks die with it
        del p.ids[0][l]
    p._apply([p.frame_edit(0, g + 1, N0 - 1, replace_last=True)], [0])
    s, t = _factor(r0, g + 1, g - 1)                       # the merged list of the two factors
    p.bw.set_imu([Imu(0, N0 - 1, s, t, _noise(r0))])
    lists[0].append((N0 - 2, s, t))
    # slot 1 takes its next frame, and its newest factor a list of 400 samples: the stride grows
    r1, N1 = runs[1], runs[1].N
    g1 = p.k[1] + N1 - 1
    p._apply([p.frame_edit(1, g1, N1 - 1)], [1])
    s1, t1 = _factor(r1, g1, g1 - 8)
    p.bw.set_imu([Imu(1, N1 - 1, s1, t1, _noise(r1))])
    lists[1].append((N1 - 2, s1, t1))
    check([2], lambda: p.bw.solve([2], max_iterations=3))  # slot 2's samples survived the growth
    check([0, 1], lambda: p.bw.solve([0, 1], max_iterations=3))
    # window_solve on slot 0
    sm = _lib.CSummary()
    opt = _lib.COptions(3, 1e6, 1, 0, 0.0)
    check([0], lambda: ba._ck(ba.lib.pvio_b200_window_solve(ba.h, C.byref(opt), C.byref(sm))))
    # slot 2: a non-keyframe with samples, replaced by a frame without a set_imu: the replaced samples leave, the new
    # factor keeps its edit record
    r2, N2 = runs[2], runs[2].N
    g2 = p.k[2] + N2
    fake = p.frame_edit(2, g2, N2)
    p._apply([fake], [2])
    p.bw.set_imu([Imu(2, N2, *_factor(r2, g2), _noise(r2))])
    for l in fake.landmarks:
        del p.ids[2][l]
    p._apply([p.frame_edit(2, g2 + 1, N2, replace_last=True)], [2])
    check([2], lambda: p.bw.solve([2], max_iterations=3))
    got = p.bw.imu_records([2])[0]
    assert got.shape == (N2, 288) and np.array_equal(_bits(got[-1]), _bits(p.rec[2][g2]))
    # a reset clears the samples: the slot solves with its edit records only
    p.bw.reset(2, runs[2].w)
    assert p.bw.imu_records([2])[0].shape == (0, 288)
    ba.close()


# ------------------------------------------------------------------------ 4: nothing else changes
def _build():
    """a handle of 8 resident slots: 4 inertial sequences (slots 0 .. 3), 4 visual windows (4 .. 7)"""
    runs = [Run(F=14, N=6, M=200, seed=760), Run(F=14, N=8, M=220, seed=761), Run(F=14, N=6, M=200, seed=762),
            Run(F=14, N=7, M=200, seed=763)]
    ba = BundleAdjustor(max_windows=8, max_frames=8, max_landmarks=200, max_obs=2000)
    p = BatchPlayer(ba, runs)
    from pvio_b200.batch_window import Edit
    for i in range(4):
        w, st = synth.make_cfg2(N=6 + (i % 3), M=90 + 10 * i, seed=900 + i, staggered=True)[:2]
        p.bw.reset(4 + i, w)
        ids = {}
        for f in range(w.N):
            e = Edit(4 + i).frame(np.concatenate([st.q[f], st.p[f], st.v[f], st.bg[f], st.ba[f]]), bool(w.frame_fixed[f]))
            new = []
            for l in range(w.M):
                if int(w.lm_anchor[l]) == f:
                    e.new.append((f, w.lm_z_ref[l], st.rho[l])); new.append(l)
                for k in range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1]):
                    if int(w.obs_frame[k]) == f:
                        e.obs.append((ids[l], f, w.obs_z[k]))
            for l, t in zip(new, p.bw.edit([e])[0]):
                ids[l] = int(t)
    return ba, p, runs


def test_slots_without_samples_and_launch_counts_are_unchanged():
    """Slots without samples beside slots with samples solve as on a handle that never saw set_imu: visual windows bit
    for bit, inertial ones bit for bit when two reference handles agree (otherwise within 2e-6).  A solve makes the
    launches of the reference when no named slot holds samples, one more otherwise, for n = 1 and n = 8."""
    (ra, pa, runs), (rb, pb, _), (rc, pc, _) = _build(), _build(), _build()
    all8 = list(range(8))
    for js in ([1], all8):                                 # before any set_imu: the same launches
        la, lb = ra.kernel_launches, rb.kernel_launches
        pa.bw.solve(js, max_iterations=3); pb.bw.solve(js, max_iterations=3); pc.bw.solve(js, max_iterations=3)
        assert rb.kernel_launches - lb == ra.kernel_launches - la
    n0 = rb.kernel_launches
    pb.bw.set_imu([Imu(j, f, *_factor(runs[j], f), _noise(runs[j])) for j in (0, 2) for f in range(1, runs[j].N)])
    assert rb.kernel_launches - n0 == 1                    # one launch per set_imu call
    for js, extra in (([1], 0), ([5], 0), ([0], 1), (all8, 1)):
        la, lb = ra.kernel_launches, rb.kernel_launches
        pa.bw.solve(js, max_iterations=3); pb.bw.solve(js, max_iterations=3); pc.bw.solve(js, max_iterations=3)
        assert rb.kernel_launches - lb == ra.kernel_launches - la + extra, js
    da, db, dc = pa.bw.download(all8, 400), pb.bw.download(all8, 400), pc.bw.download(all8, 400)
    for s in (1, 3, 4, 5, 6, 7):
        gap_ac = max(np.abs(da[s]["frames"] - dc[s]["frames"]).max(), np.abs(da[s]["inv_depth"] - dc[s]["inv_depth"]).max())
        gap_ab = max(np.abs(da[s]["frames"] - db[s]["frames"]).max(), np.abs(da[s]["inv_depth"] - db[s]["inv_depth"]).max())
        print(f"slot {s}: two reference handles differ by {gap_ac:.3e}, the handle with samples by {gap_ab:.3e}")
        assert gap_ab == 0.0 if gap_ac == 0.0 else gap_ab < SEQ_TOL, s
    assert np.abs(da[0]["frames"] - db[0]["frames"]).max() > 0.0          # slot 0 did re-integrate
    for h in (ra, rb, rc):
        h.close()


# ------------------------------------------------------------------------ 5: rejections
def test_rejections_change_nothing():
    ba, p, runs = _build()
    all8 = list(range(8))
    p.bw.set_imu([Imu(1, 2, *_factor(runs[1], 2), _noise(runs[1]))])
    keep = []

    def rec(slot=0, frame=1, n=None, samples=True, t_end=0.25, noise=True, spoil=None):
        s, t = _factor(runs[0], 1)
        s = s.copy()
        nz = np.array([np.asarray(c, dtype=np.float64).reshape(9) for c in _noise(runs[0])])
        if spoil == "sample":
            s[7, 3] = np.nan
        if spoil == "noise":
            nz[2, 4] = np.inf
        keep.extend([s, nz])
        r = _lib.CWindowImu()
        r.slot, r.frame, r.n_samples, r.t_end = slot, frame, len(s) if n is None else n, t_end if spoil != "t_end" else np.inf
        r.samples = _lib.ptr(s) if samples else None
        r.noise_cov = _lib.ptr(nz) if noise else None
        return r

    def arr(*rs):
        a = (_lib.CWindowImu * len(rs))()
        for i, r in enumerate(rs):
            a[i] = r
        return a

    bad = {
        "slot out of range": [rec(slot=8)], "negative slot": [rec(slot=-1)],
        "visual-only slot": [rec(slot=5)], "frame 0": [rec(frame=0)], "frame N": [rec(frame=runs[0].N)],
        "pair named twice": [rec(frame=2), rec(slot=2), rec(frame=2)], "no samples": [rec(n=0)],
        "null samples": [rec(samples=False)], "null noise": [rec(noise=False)], "nan sample": [rec(spoil="sample")],
        "inf t_end": [rec(spoil="t_end")], "inf noise": [rec(spoil="noise")],
        "a good record before a bad one": [rec(frame=3), rec(slot=1, frame=9)],
    }
    ba2 = BundleAdjustor(max_windows=8, max_frames=8, max_landmarks=200, max_obs=2000)   # slot 0 never reset there
    r_nr = arr(rec())
    assert ba2.lib.pvio_b200_batch_window_set_imu(ba2.h, 1, r_nr) == EINVAL
    ba2.close()
    before, imus = p.bw.download(all8, 400), p.bw.imu_records([0, 1, 2, 3])
    for name, rs in bad.items():
        n0 = ba.kernel_launches
        assert ba.lib.pvio_b200_batch_window_set_imu(ba.h, len(rs), arr(*rs)) == EINVAL, name
        assert ba.kernel_launches == n0, name
    assert ba.lib.pvio_b200_batch_window_set_imu(ba.h, -1, arr(rec())) == EINVAL
    assert ba.lib.pvio_b200_batch_window_set_imu(ba.h, 1, None) == EINVAL
    n0 = ba.kernel_launches
    assert ba.lib.pvio_b200_batch_window_set_imu(ba.h, 0, None) == 0 and ba.kernel_launches == n0
    after, imus2 = p.bw.download(all8, 400), p.bw.imu_records([0, 1, 2, 3])
    for a, b in zip(before, after):
        for k in a:
            assert np.array_equal(a[k], b[k]), k
    for a, b in zip(imus, imus2):
        assert np.array_equal(a, b)
    # no rejected record left samples behind: against a handle that never saw set_imu, a solve of slot 0 makes no
    # re-integration launch, one of slot 1 (which holds samples) one
    ref, pr, _ = _build()
    for js, extra in (([0], 0), ([1], 1)):
        n0, r0 = ba.kernel_launches, ref.kernel_launches
        p.bw.solve(js, max_iterations=2)
        pr.bw.solve(js, max_iterations=2)
        assert ba.kernel_launches - n0 == ref.kernel_launches - r0 + extra, js
    ref.close()
    with pytest.raises(PvioB200Error):
        p.bw.imu_records([5])                              # a visual-only slot has no IMU records
    with pytest.raises(PvioB200Error):
        p.bw.imu_records([0, 0])
    ba.close()


# ------------------------------------------------------------------------ 6: sequences
class _ReChain(Chain):
    """The re-pack twin of BundleAdjustor::solve: before every solve each factor of the window is re-integrated at its
    frame i's current biases with pvio_b200_preintegrate"""

    def __init__(self, run, handle):
        super().__init__(run)
        self.handle = handle

    def window(self, k):
        w, st, lm = super().window(k)
        fs = [(s, t, self.bg[k + i].copy(), self.ba[k + i].copy())
              for i, (s, t, _, _) in enumerate(self.run.truth.imu_factors[k:k + self.run.N - 1])]
        _set_records(w, imu.preintegrate(self.handle, fs, self.run.truth.imu_noise))
        return w, st, lm


def test_sequences_follow_the_reintegrating_twin():
    """4 inertial sequences (N = 6, 8, 9, 6; the second with planes) take two solved keyframes with a marginalisation, a
    drop and a replaced non-keyframe between them.  With samples they follow a re-pack twin that re-integrates every
    factor at its first frame's biases before each ba_solve + ba_marginalize (what BundleAdjustor::solve does): equal
    iterations, anchors and landmarks, states within 2e-6.  The same sequences without samples depart from that twin
    by more than 100x that bar.  Further on, the synthetic runs' re-integrated sequences amplify rounding differences
    by 1e3 - 1e5 per keyframe (the twin against itself as much as against the slots), so the bar holds for these two."""
    kws = [dict(F=20, N=6, M=220, seed=770), dict(F=22, N=8, M=260, seed=772, planes=2),
           dict(F=23, N=9, M=260, seed=774), dict(F=20, N=6, M=220, seed=776)]
    mk = lambda: [Run(**kw) for kw in kws]                 # noqa: E731
    ba = BundleAdjustor(max_windows=8, max_frames=9, max_landmarks=400, max_obs=3000)
    one = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=400, max_obs=3000)
    runs = mk()
    with_s = BatchPlayer(ba, runs, slots=range(4), imu_samples=True)
    without = BatchPlayer(ba, mk(), slots=range(4, 8))
    refs = [_ReChain(r, one) for r in runs]
    js = list(range(4))
    gap_with, gap_without, fails = 0.0, 0.0, []
    for step in range(2):
        sm_w = with_s.bw.solve(with_s.slots, max_iterations=10)   # the reference's solver_iteration_limit
        without.bw.solve(without.slots, max_iterations=10)
        dw = with_s.refresh(js, 400)
        do = without.refresh(js, 400)
        for j in js:
            k = with_s.k[j]
            wr, sr, lm = refs[j].window(k)
            out, summ = one.solve(wr, sr, max_iterations=10, postpass=False)
            S, e = one.marginalize_frame(wr, out, index=0)
            refs[j].store(k, out, lm)
            refs[j].set_prior(k, S, e, out)
            ok_it = sm_w[j]["iterations"] == summ["iterations"] and sm_w[j]["accepted_steps"] == summ["accepted_steps"]
            row = {int(t): r for r, t in enumerate(dw[j]["ids"])}
            rows = [row[with_s.ids[j][l]] for l in lm]
            ok_lm = np.array_equal(dw[j]["anchor"][rows], wr.lm_anchor) and np.all(dw[j]["n_obs"][rows] >= 2)
            if not (ok_it and ok_lm):
                fails.append((step, j, sm_w[j]["iterations"], summ["iterations"]))
            refv = np.concatenate([out.q, out.p, out.v, out.bg, out.ba], axis=1)
            gap_with = max(gap_with, np.abs(dw[j]["frames"] - refv).max(),
                           np.max(np.abs(dw[j]["inv_depth"][rows] - out.rho) / np.abs(out.rho)))
            gap_without = max(gap_without, np.abs(do[j]["frames"] - refv).max())
        with_s.advance(js, nonkey=True)
        without.advance(js, nonkey=True)
    ba.close()
    one.close()
    print(f"largest difference to the re-integrating twin: with samples {gap_with:.3e}, without {gap_without:.3e}")
    assert not fails, fails
    assert gap_with < SEQ_TOL
    assert gap_without > 100 * SEQ_TOL
