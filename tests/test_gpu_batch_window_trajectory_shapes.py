"""pvio_b200_batch_window_trajectory and pvio_b200_batch_window_smoothed_trajectory at every window size, sample count,
time layout and slot history the handle accepts, against oracle/trajectory_oracle.trajectory and
trajectory_smoothing_oracle.smoothed, with a 50-digit judge (trajectory_mp_oracle) on the far, epoch-time and
400-sample windows.

- Sizes: cfg3 windows of N = 1 (a prior only) to 16 frames on a max_frames 16 handle, so bw_trajectory_kernel runs 0 to
  15 warps.  With covariances N <= 11; from N = 12 the covariance system does not fit cov_kernel's shared memory and a
  call that asks for it is refused whole.
- Which factors hold samples: none, the first, the last, all but the first, all but the last, every other one, one in
  the middle, at N = 7 and 16.  That moves the frames of the joint covariance block the kernels index.
- Every factor has its own noise: a scaled copy of EuRoC's, or full symmetric 3 x 3 blocks in a random rotation.
- Sample counts 1, 2, 3, 50 and 250 (1 kHz) in one window, 400 per factor (2 s at 200 Hz), a factor whose store row
  grows after the slot was queried.
- Times: every sample time and t_end and each +- 1e-9, 5e-8 and 2e-7 s (both sides of the 1e-7 s dt clamp), duplicate
  times, 20,000 times in one record, records of 0 and 10^4 times in one call, gaps of 1e-9, 1e-6 and 1e-2 s between a
  factor's t_end and the next factor's first sample, and timestamps at t0 = 1.7e9 s.
- A window 5 km from the origin; slots after one and three drop_victim calls, after save on a handle whose sample
  store holds 1,500 rows per factor and restore onto a fresh one, after mirror_frame merged a non-keyframe's samples
  into the factor of the frame that replaced it, and a slot reset from N = 16 to N = 3.
- Near-singular Sigma(T): a one-sample factor (frame -2), a two-sample factor whose last sample ends 1e-6 s before
  t_end and a 400-sample factor (both smoothed), each clear of the 1e-10 pivot rule (test_trajectory_shapes_windows
  prints the margins).
- Every case in one call, shuffled, with 1 and 15 warps present, each record the bits of its single-record call.

Bars.  Forward states 1e-12 relative to 1 + |x| (test_gpu_batch_window_trajectory's).  Smoothed states
max(1e-11, 64 kappa(Sigma(T)) 2^-53), kappa in the Jacobi scaling (chol_oracle.scaled_condition): the smoother solves
with Sigma(T), so its rounding grows with kappa; only the two-sample factor ending 1e-6 s before t_end (kappa ~ 1e6)
lifts the bar above 1e-11.  Covariances BAR_FP64 from test_gpu_batch_window_covariance, against the oracles fed each
slot's joint frame covariance from pvio_b200_batch_window_covariance (which test_gpu_batch_window_covariance_shapes
holds to cov_oracle): what is measured here is the propagation and the block each kernel reads."""
import functools

import numpy as np
import pytest

from oracle import chol_oracle
from oracle import trajectory_oracle as to
from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows, Edit, Imu
from pvio_b200.bundle_adjustor import BundleAdjustor
from synthetic import synth
from test_gpu_batch_window_covariance import BAR_FP64, _err, _feed, _tracks
import trajectory_mp_oracle as mpo
import trajectory_smoothing_oracle as tso

pytestmark = pytest.mark.gpu
MAX_FRAMES, MAX_WINDOWS, M = 16, 64, 40
COV_MAX_N = 11                                   # the largest inertial window cov_kernel's shared memory takes
IMU_WARP_SM = 8 * (2 * 81 + 4 * 9 + 2 * 9 + 2 * 9 + 5 * 9 + 4 + 3 + 3 + 3 + 2)    # sizeof(ImuWarpSm), imu.cuh
OFFS = (0.0, -1e-9, 1e-9, -5e-8, 5e-8, -2e-7, 2e-7)
FWD_BAR, SMOOTH_FLOOR = 1e-12, 1e-11


def patterns(N):
    """which factors hold samples, by name"""
    nf = N - 1
    return {"none": (), "first": (0,), "last": (nf - 1,), "all_but_first": tuple(range(1, nf)),
            "all_but_last": tuple(range(nf - 1)), "alternate": tuple(range(0, nf, 2)), "middle": (nf // 2,)}


SPECS = {f"N{N}": dict(N=N, seed=1100 + N) for N in range(1, 17)}
for _N in (7, 16):
    for _p, _h in patterns(_N).items():
        SPECS[f"N{_N}_{_p}"] = dict(N=_N, seed=1200 + _N, holds=_h)
SPECS.update({
    "N3_first": dict(N=3, seed=1103, holds=(0,)),                    # the window a N = 16 slot is reset to
    "mix": dict(N=8, seed=1301, hz=1000.0, counts=(1, 2, 3, 50, 250, 50, 2)),
    "long": dict(N=4, seed=1302, kf_dt=2.0),                          # 400 samples per factor
    "sing": dict(N=5, seed=1303, sing=True),
    "gaps": dict(N=5, seed=1304, gaps=(None, 1e-9, 1e-6, 1e-2)),
    "epoch": dict(N=6, seed=1305, t0=1.7e9),
    "offset": dict(N=6, seed=1306, offset=True),
})
MP_CASES = ("offset", "epoch", "long")


def noise(k, seed):
    """factor k's own noise: even k EuRoC's scaled by 1 + 0.37 k, odd k R diag(d) R^T per block (R a random rotation,
    d EuRoC's diagonal times U(0.5, 2))"""
    base = [np.eye(3) * synth.EUROC[c] for c in ("cov_g", "cov_a", "cov_bg", "cov_ba")]
    if k % 2 == 0:
        return tuple(b * (1.0 + 0.37 * k) for b in base)
    rng = np.random.default_rng(31 * seed + k)
    out = []
    for b in base:
        Q, _ = np.linalg.qr(rng.normal(size=(3, 3)))
        S = Q @ np.diag(b[0, 0] * rng.uniform(0.5, 2.0, 3)) @ Q.T
        out.append(0.5 * (S + S.T))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def window(name):
    """the case's generated window: w, st, N, factors [(samples or None, t_end)], noises [per factor or None]"""
    sp = SPECS[name]
    N = sp["N"]
    if sp.get("offset"):
        w, st, truth = synth.hard_base(True, "offset", N, M, sp["seed"])
        w, st, truth = synth.with_offset(w, st, truth)   # the samples are body-frame rates: nothing of theirs moves
    else:
        w, st, truth = synth.make_cfg3(N=max(N, 2), M=M, seed=sp["seed"], kf_dt=sp.get("kf_dt", 0.25),
                                       imu_hz=sp.get("hz", 200.0))
    holds = sp.get("holds", tuple(range(N - 1)))
    factors, noises = [], []
    for k in range(N - 1):
        s, t_end = truth.imu_factors[k][0].copy(), float(truth.imu_factors[k][1])
        if "counts" in sp:                            # from the 1 kHz stream
            c = sp["counts"][k]
            s = s[:c] if c <= 3 else (s[::5] if c == 50 else s)
        if sp.get("sing"):
            s = [np.vstack([s[0], np.r_[t_end - 1e-6, s[1, 1:]]]), s[:1], s, s[[0, 25]]][k]
        if sp.get("gaps") and sp["gaps"][k] is not None:
            t0 = s[0, 0] + sp["gaps"][k]              # the first sample moved to its frame's time + gap
            s = np.vstack([np.r_[t0, s[0, 1:]], s[s[:, 0] > t0]])
        s[:, 0] += sp.get("t0", 0.0)
        t_end += sp.get("t0", 0.0)
        factors.append((s if k in holds else None, t_end))
        noises.append(noise(k, sp["seed"]) if k in holds else None)
    return dict(w=w, st=st, N=N, factors=factors, noises=noises)


def times(name, every=None):
    """the case's query times (times_of)"""
    return times_of(window(name)["factors"], every)


def times_of(F, every=None):
    """query times over the factors F, sorted: their samples (every `every`-th; None: about six per factor) and t_end
    each with the offsets OFFS, sample midpoints, the gaps' middles, times before, after and over factors without
    samples, and every tenth time three times"""
    if not F:
        return np.array([-1.0, 0.0, 0.0, 0.5])
    ts = []
    for k, (s, t_end) in enumerate(F):
        if s is None:
            ts.append(t_end - 0.5e-3)
            continue
        for b in list(s[::every or max(1, len(s) // 6), 0]) + [t_end]:
            ts += [b + o for o in OFFS]
        ts += list(0.5 * (s[1:, 0] + s[:-1, 0])[::13])
        if k + 1 < len(F) and F[k + 1][0] is not None:
            g = F[k + 1][0][0, 0] - t_end
            ts += [t_end + 0.5 * g, t_end + 0.999 * g] if g > 0 else []
    held = [s for s, _ in F if s is not None]
    if held:
        ts += [held[0][0, 0] - 1e-3, F[-1][1] + 1e-3]
    ts = np.sort(np.array(ts))
    return np.sort(np.concatenate([ts, np.repeat(ts[::10], 2)]))


def smem_forward(warps, covs):
    """bw_trajectory_kernel's dynamic shared memory: per warp two ImuWarpSm, with covariances four 15 x 15"""
    return warps * (2 * IMU_WARP_SM + (4 * 225 * 8 if covs else 0))


def sigma_T(c, frames, k):
    """factor k's Sigma(T), its 15 x 15 increment covariance at frame k's biases"""
    s, t_end = c["factors"][k]
    x = frames[k]
    return to.delta(s, t_end, x[10:13], x[13:16], c["noises"][k])["cov"]


def smoother_pd(S):
    return tso.chol_pd(S[0:9, 0:9]) and tso.chol_pd(S[9:12, 9:12]) and tso.chol_pd(S[12:15, 12:15])


# ---------------------------------------------------------------------------------------------------------- device side
def _seat(bw, slot, name):
    c = window(name)
    w, st = c["w"], c["st"]
    if c["N"] == 1:                                   # frame 0 of a two-frame window, with its prior
        bw.reset(slot, w)
        bw.edit([Edit(slot).frame(np.concatenate([st.q[0], st.p[0], st.v[0], st.bg[0], st.ba[0]]), True)])
        x0 = np.concatenate([w.prior_q0, w.prior_p0, w.prior_v0, w.prior_bg0, w.prior_ba0], axis=1)
        bw.set_prior(slot, w.prior_S, w.prior_e, x0)
    else:
        _feed(bw, slot, w, st, _tracks(w, planes=False))
    recs = [Imu(slot, k + 1, s, t, n) for k, ((s, t), n) in enumerate(zip(c["factors"], c["noises"])) if s is not None]
    if recs:
        bw.set_imu(recs)


def call(ba, slots, tss, covs, smoothed):
    """one raw call with a covariance flag per record; outputs start as 7s.  Returns (rc, per record a dict)"""
    n = len(slots)
    recs, outs = (_lib.CWindowTrajectory * max(n, 1))(), []
    for r, s, t, cv in zip(recs, slots, tss, covs):
        t = np.ascontiguousarray(t, dtype=np.float64)
        k = len(t)
        o = dict(states=np.full((k, 16), 7.0), frame=np.full(k, 7, dtype=np.int32),
                 state_cov=np.full((k, 15, 15), 7.0) if cv else None, t=t)
        r.slot, r.n_times, r.status = int(s), k, 99
        _lib.set_ptrs(r, times=t if k else None, states=o["states"] if k else None, frame=o["frame"] if k else None,
                      state_cov=o["state_cov"] if (cv and k) else None)
        outs.append(o)
    fn = ba.lib.pvio_b200_batch_window_smoothed_trajectory if smoothed else ba.lib.pvio_b200_batch_window_trajectory
    rc = fn(ba.h, n, recs)
    for r, o in zip(recs, outs):
        o["status"] = int(r.status)
        del o["t"]
    return rc, outs


def same(a, b, what):
    for key in ("states", "frame", "state_cov", "status"):
        x, y = a.get(key), b.get(key)
        assert (x is None) == (y is None), (what, key)
        if x is not None:
            assert np.array_equal(np.asarray(x), np.asarray(y), equal_nan=True), (what, key)


def run4(ba, slot, ts, cov_ok=True):
    """forward and smoothed, without and (cov_ok) with covariances: {(smoothed, cov): output}"""
    out = {}
    for sm in (False, True):
        for cv in ((False, True) if cov_ok else (False,)):
            rc, o = call(ba, [slot], [ts], [cv], sm)
            assert rc == 0, (slot, sm, cv)
            out[(sm, cv)] = o[0]
    return out


def _subset(mask, lim):
    idx = np.flatnonzero(mask)
    if len(idx) <= lim:
        return idx
    return idx[np.unique(np.linspace(0, len(idx) - 1, lim).round().astype(int))]


def check(bw, slot, c, ts, outs, label, factors=None, noises=None, frames=None, lim=(60, 10, 16, 4)):
    """outs of run4 against the oracles at the slot's downloaded state; the frame index of every row exactly, states
    and covariances on a fixed subsample of at most lim = (forward states, smoothed states, forward covariances,
    smoothed covariances) rows"""
    F = c["factors"] if factors is None else factors
    nz = c["noises"] if noises is None else noises
    frames = bw.download([slot], 200)[0]["frames"] if frames is None else frames
    N = len(frames)
    fr = np.array([to.factor_of(t, F) for t in ts], dtype=np.int32)
    pd = {k: smoother_pd(sigma_T(dict(factors=F, noises=nz), frames, k)) for k in set(fr[fr >= 0].tolist())}
    frs = np.array([f if f < 0 or pd[f] else -2 for f in fr], dtype=np.int32)
    kap = {k: chol_oracle.scaled_condition(sigma_T(dict(factors=F, noises=nz), frames, k)) if pd[k] else np.nan for k in pd}
    joint = None
    if (False, True) in outs:
        cv = bw.covariance([slot], [list(range(N))], [[]])[0]
        assert outs[(False, True)]["status"] == cv["status"] == outs[(True, True)]["status"], label
        joint = cv["cov"] if cv["status"] == _lib.OK else None
    for (sm, cv), o in outs.items():
        want = frs if sm else fr
        assert np.array_equal(o["frame"], want), (label, sm, cv)
        off = want < 0
        assert np.all(o["states"][off] == 0.0), (label, sm, cv)
        if cv:
            assert np.isnan(o["state_cov"][off]).all(), (label, sm, cv)
            sc = o["state_cov"]
            assert np.array_equal(sc, np.transpose(sc, (0, 2, 1)), equal_nan=True), (label, sm)
        if not cv:
            assert np.array_equal(o["states"], outs[(sm, True)]["states"] if (sm, True) in outs else o["states"])
    on = fr >= 0
    # forward states and covariances
    i = _subset(on, lim[0])
    if len(i):
        Sig = None if joint is None else np.array([joint[15 * f:15 * f + 15, 15 * f:15 * f + 15] for f in range(N)])
        _, st, _ = to.trajectory(ts[i], frames, F, nz)
        e = (np.abs(outs[(False, False)]["states"][i] - st) / (1.0 + np.abs(st))).max()
        msg = f"{label}: forward {on.sum()} rows, state error {e:.2e} (bar {FWD_BAR:.0e})"
        assert e < FWD_BAR, msg
        if Sig is not None:
            j = _subset(on, lim[2])
            _, _, cov = to.trajectory(ts[j], frames, F, nz, Sig)
            worst = max(_err(a, b) for a, b in zip(outs[(False, True)]["state_cov"][j], cov))
            msg += f", covariance error {worst:.2e} (bar {BAR_FP64[0]:.0e})"
            assert worst < BAR_FP64[0], msg
        print(msg)
    # smoothed states and covariances
    ons = frs >= 0
    i = _subset(ons, lim[1])
    if len(i):
        _, st, _ = tso.smoothed(ts[i], frames, F, nz)
        e = np.abs(outs[(True, False)]["states"][i] - st) / (1.0 + np.abs(st))
        bars = np.array([max(SMOOTH_FLOOR, 64 * kap[f] * 2.0 ** -53) for f in frs[i]])
        rows = e.max(axis=1)
        msg = (f"{label}: smoothed {ons.sum()} rows, kappa(Sigma(T)) <= {max(kap[f] for f in frs[i]):.1e}, "
               f"state error {rows.max():.2e} (bar {bars.min():.1e} .. {bars.max():.1e})")
        assert np.all(rows < bars), msg
        if joint is not None:
            j = _subset(ons, lim[3])
            _, _, cov = tso.smoothed(ts[j], frames, F, nz, joint)
            worst = max(_err(a, b) for a, b in zip(outs[(True, True)]["state_cov"][j], cov))
            msg += f", covariance error {worst:.2e} (bar {BAR_FP64[0]:.0e})"
            assert worst < BAR_FP64[0], msg
        print(msg)


@pytest.fixture(scope="module")
def seq():
    ba = BundleAdjustor(max_windows=MAX_WINDOWS, max_frames=MAX_FRAMES, max_landmarks=64, max_obs=1500)
    bw = BatchWindows(ba)
    slot = {name: j for j, name in enumerate(SPECS)}
    for name, j in slot.items():
        _seat(bw, j, name)
    yield ba, bw, slot
    ba.close()


def _free(slot, k=0):
    return len(slot) + k                              # slots past the cases', for the histories


@pytest.mark.parametrize("name", [n for n in SPECS if SPECS[n]["N"] <= COV_MAX_N])
def test_with_covariances_against_the_oracles(seq, name):
    ba, bw, slot = seq
    c = window(name)
    ts = times(name, every=1 if name in ("N7", "mix", "gaps") else None)
    check(bw, slot[name], c, ts, run4(ba, slot[name], ts), name)


@pytest.mark.parametrize("name", [n for n in SPECS if SPECS[n]["N"] > COV_MAX_N])
def test_large_windows_without_covariances_and_refused_with_them(seq, name):
    ba, bw, slot = seq
    c = window(name)
    s = slot[name]
    ts = times(name)
    check(bw, s, c, ts, run4(ba, s, ts, cov_ok=False), name)
    before, d0 = bw.save([s]), bw.download([s], 200)
    held = any(f[0] is not None for f in c["factors"])
    for sm in (False, True):
        rc, o = call(ba, [slot["N3"], s], [times("N3"), ts], [True, True], sm)
        if not held:                                  # no covariance system to solve: NaN rows, as at any N
            assert rc == 0 and np.all(o[1]["frame"] == -1) and np.isnan(o[1]["state_cov"]).all(), (name, sm)
            assert o[1]["status"] == _lib.OK
            continue
        assert rc == _lib.EINVAL, (name, sm)
        for r in o:
            assert np.all(r["states"] == 7.0) and np.all(r["frame"] == 7) and np.all(r["state_cov"] == 7.0)
            assert r["status"] == 99
    assert bw.save([s]) == before
    d1 = bw.download([s], 200)
    for key in d0[0]:
        assert np.array_equal(d0[0][key], d1[0][key]), key


def test_fifty_digit_judge(seq):
    ba, bw, slot = seq
    for name in MP_CASES:
        c = window(name)
        frames = bw.download([slot[name]], 200)[0]["frames"]
        F = c["factors"]
        ts = times(name)
        fr = np.array([to.factor_of(t, F) for t in ts])
        i = _subset(fr >= 0, 30)
        rc, o = call(ba, [slot[name]], [ts], [False], False)
        assert rc == 0 and o[0]["status"] == _lib.OK, name
        dev = o[0]["states"][i]
        _, ora, _ = to.trajectory(ts[i], frames, F, c["noises"])
        ref = np.array([mpo.state(frames[fr[r]], F[fr[r]][0], ts[r]) for r in i])
        ed = (np.abs(dev - ref) / (1.0 + np.abs(ref))).max()
        eo = (np.abs(ora - ref) / (1.0 + np.abs(ref))).max()
        print(f"{name}: {len(i)} times against 50 digits: device {ed:.2e}, trajectory_oracle {eo:.2e} (bar {FWD_BAR:.0e})")
        assert ed < FWD_BAR and eo < FWD_BAR, name


def test_large_records_and_splits(seq):
    ba, bw, slot = seq
    for name, cv in (("N16", False), ("N11", True)):
        c = window(name)
        F = [f for f in c["factors"] if f[0] is not None]
        ts = np.sort(np.random.default_rng(5).uniform(F[0][0][0, 0] - 0.01, F[-1][1] + 0.01, 20000))
        for sm in (False, True):
            whole = call(ba, [slot[name]], [ts], [cv], sm)[1][0]
            parts = [call(ba, [slot[name]], [p], [cv], sm)[1][0] for p in np.array_split(ts, 5)]
            for key in ("states", "frame") + (("state_cov",) if cv else ()):
                assert np.array_equal(whole[key], np.concatenate([p[key] for p in parts]), equal_nan=True), (name, sm, key)
        outs = run4(ba, slot[name], ts, cov_ok=cv)
        check(bw, slot[name], c, ts, outs, f"{name} x 20000")
    # records of 0 and 10^4 times in one call
    names = ["N9", "N5", "mix", "N2"]
    tss = []
    for j, n in enumerate(names):                     # over each window's own span, 0.01 s either side
        F = [f for f in window(n)["factors"] if f[0] is not None]
        lo, hi = F[0][0][0, 0] - 0.01, F[-1][1] + 0.01
        tss.append(np.sort(np.random.default_rng(j).uniform(lo, hi, 10000)) if j % 2 else np.zeros(0))
    for sm in (False, True):
        for cv in (False, True):
            rc, many = call(ba, [slot[n] for n in names], tss, [cv] * 4, sm)
            assert rc == 0
            for n, t, m in zip(names, tss, many):
                same(call(ba, [slot[n]], [t], [cv], sm)[1][0], m, (n, sm, cv))


def test_sample_store_growth_changes_no_output(seq):
    ba, bw, slot = seq
    A = [slot["mix"], slot["long"], slot["N11"]]
    before = {s: run4(ba, s, times(n)) for s, n in zip(A, ("mix", "long", "N11"))}
    B = _free(slot)
    c, F = _seat_long(bw, B)
    long, t_end = F[0]
    for s_, n in zip(A, ("mix", "long", "N11")):
        after = run4(ba, s_, times(n))
        for key in after:
            same(before[s_][key], after[key], (n, key))
    ts = np.sort(np.concatenate([long[::50, 0], [t_end, long[-1, 0] + 5e-5]]))
    check(bw, B, c, ts, run4(ba, B, ts), "1500-sample factor", factors=F, lim=(20, 3, 6, 2))


LONG = 1500                                       # samples of _seat_long's first factor, past any case's


def _seat_long(bw, slot):
    """the N3 window in `slot` with its first factor's 50 samples respread as LONG over the same span: a handle holding
    it has LONG rows per factor in its sample store (ensure_imu_store grows the store to the longest factor it is
    given).  Returns (case, factors)"""
    _seat(bw, slot, "N3")
    c = window("N3")
    s, t_end = c["factors"][0]
    long = np.repeat(s, 40, axis=0)[:LONG]
    long[:, 0] = np.linspace(s[0, 0], t_end - 1e-4, len(long))
    bw.set_imu([Imu(slot, 1, long, t_end, c["noises"][0])])
    return c, [(long, t_end), c["factors"][1]]


def _twin(bw, slot, twin, w, factors, noises):
    """a fresh slot fed the slot's current frames and IMU records, and the given factors' samples"""
    d = bw.download([slot], 200)[0]["frames"]
    recs = bw.imu_records([slot])[0]
    bw.reset(twin, w)
    for f in range(len(d)):
        bw.edit([Edit(twin).frame(d[f], f == 0, recs[f - 1] if f > 0 else None)])
    imu = [Imu(twin, k + 1, s, t, n) for k, ((s, t), n) in enumerate(zip(factors, noises)) if s is not None]
    if imu:
        bw.set_imu(imu)
    return d


@pytest.mark.parametrize("drops", [1, 3])
def test_after_drop_victim(seq, drops):
    ba, bw, slot = seq
    name = "N10"
    c = window(name)
    s, tw = _free(slot, 1), _free(slot, 2)
    _seat(bw, s, name)
    for _ in range(drops):
        bw.drop_victim([s])
    F, nz = c["factors"][drops:], c["noises"][drops:]
    ts = times(name)
    outs = run4(ba, s, ts)
    d = _twin(bw, s, tw, c["w"], F, nz)
    check(bw, s, dict(factors=F, noises=nz), ts, outs, f"{name} after {drops} drop(s)", frames=d)
    for sm in (False, True):
        same(call(ba, [tw], [ts], [False], sm)[1][0], outs[(sm, False)], ("twin", drops, sm))


def test_save_on_a_large_store_and_restore_onto_a_fresh_handle(seq):
    ba, bw, slot = seq
    L = _free(slot, 4)
    _, FL = _seat_long(bw, L)                         # this handle's store holds LONG rows per factor
    names = ["mix", "long", "N7_alternate", "long1500"]
    slots = [slot[n] for n in names[:3]] + [L]
    tss = [times(n) for n in names[:3]] + [times_of(FL)]
    blobs = bw.save(slots)
    ba2 = BundleAdjustor(max_windows=4, max_frames=MAX_FRAMES, max_landmarks=64, max_obs=1500)
    try:
        bw2 = BatchWindows(ba2)                       # a fresh handle: an empty store, grown by the restore
        bw2.restore([3, 0, 1, 2], blobs)
        for n, s1, s2, ts in zip(names, slots, (3, 0, 1, 2), tss):
            a, b = run4(ba, s1, ts), run4(ba2, s2, ts)
            for key in a:
                same(a[key], b[key], (n, key))
    finally:
        ba2.close()


def test_after_a_merged_non_keyframe():
    """mirror_frame keeping its samples onto a slot whose newest frame is not a keyframe: the newest frame is replaced
    and factor N - 2 becomes the replaced frame's samples followed by the new frame's (merge list ++ samples), with
    t_end and noise of the new frame.  Against the oracles at the slot's state, and bit for bit against a fresh twin
    fed that window."""
    from test_gpu_batch_window_mirror import CAP, CX, CY, Seq, _advance, _start
    from pvio_b200.batch_window import Mirror
    mb = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=4096, max_obs=16384)
    try:
        bw = BatchWindows(mb)
        sq = Seq(0, 0, 1, 4, 1311)
        _start(bw, [sq])
        ft = _advance(bw, [sq])
        s1, t1, n1 = sq.imu()
        o = bw.mirror_frame([Mirror(sq.slot, sq.tracker, s1, t1, n1, CX, CY, True)], CAP)[0]
        kp = o["kp_track"][:len(ft[0]["keypoints"])]
        bw.set_keypoints(sq.slot, sq.tracker, sq.f + 1, {int(t): kj for kj, t in enumerate(kp) if t >= 0}, False,
                         o["skipped_frames"])
        assert len(bw.download([sq.slot], 4096)[0]["frames"]) == 2
        _advance(bw, [sq])
        s2, t2, _ = sq.imu()
        nz = noise(1, 1311)                          # the merged factor takes the new frame's noise
        bw.mirror_frame([Mirror(sq.slot, sq.tracker, s2, t2, nz, CX, CY, True)], CAP)
        F, NZ = [(np.concatenate([s1, s2]), t2)], [nz]
        ts = times_of(F, every=1)
        outs = run4(mb, sq.slot, ts)
        d = _twin(bw, sq.slot, 2, sq.run.w, F, NZ)
        assert len(d) == 2
        check(bw, sq.slot, dict(factors=F, noises=NZ), ts, outs, f"merged factor of {len(F[0][0])} samples", frames=d,
              lim=(40, 8, 12, 4))
        for sm in (False, True):
            same(call(mb, [2], [ts], [False], sm)[1][0], outs[(sm, False)], ("merged twin", sm))
    finally:
        mb.close()


def test_reset_from_sixteen_frames_to_three(seq):
    ba, bw, slot = seq
    s = _free(slot, 3)
    _seat(bw, s, "N16")
    _seat(bw, s, "N3_first")                          # factor 1 holds no samples now
    ts = np.concatenate([times("N3_first"), times("N16")])
    ts.sort()
    outs = run4(ba, s, ts)
    check(bw, s, window("N3_first"), ts, outs, "N16 -> N3")
    twin = run4(ba, slot["N3_first"], ts)
    for key in outs:
        same(outs[key], twin[key], key)


def test_one_call_many_slots(seq):
    ba, bw, slot = seq
    rng = np.random.default_rng(17)
    names = list(SPECS)
    rng.shuffle(names)
    names = names[:MAX_WINDOWS]
    tss = [times(n)[::1 + j % 3] for j, n in enumerate(names)]
    warps = [max(1, SPECS[n]["N"] - 1) for n in names]
    assert min(warps) == 1 and max(warps) == MAX_FRAMES - 1
    for cov in (False, True):
        covs = [cov and SPECS[n]["N"] <= COV_MAX_N for n in names]
        if cov:
            print(f"{len(names)} records, forward dynamic shared memory {smem_forward(max(warps), True)} B")
        for sm in (False, True):
            L = ba.kernel_launches
            rc, many = call(ba, [slot[n] for n in names], tss, covs, sm)
            assert rc == 0 and ba.kernel_launches - L == (4 if cov else 1), (cov, sm)
            for n, t, cv, m in zip(names, tss, covs, many):
                same(call(ba, [slot[n]], [t], [cv], sm)[1][0], m, (n, cov, sm))
