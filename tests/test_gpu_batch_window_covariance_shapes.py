"""pvio_b200_batch_window_covariance and pvio_b200_batch_window_landmarks(covariance) at every window size the handle
accepts, under every fixing pattern, on hard windows and after slot histories, against cov_oracle.covariance(refine=True)
(frame blocks, Var(rho)) and landmark_oracle.point_covariance (world points):

  every size     inertial cfg3 windows N = 1 ... 11 (N = 1 with its prior) on an fp64 handle of max_frames 12; visual cfg2
                 windows N = 1 ... 16 on an fp32 handle of max_frames 16, and N = 2, 9 and 16 on an fp64 handle of
                 max_frames 16 (a handle that also holds an inertial slot runs every window in fp64); N = 1 with its
                 frame fixed (OK, zero blocks) and with its frame free and unobserved (ENUMERIC, NaN, the other records
                 of the call unaffected);
  one call       every window of a handle in one call, shuffled, with its frames and tracks named in a permuted order:
                 bit for bit the records called one at a time, and those the matching blocks of the all-frames call;
  fixing         frame 0, the last frame, {0, N - 1}, every other frame, all but one, all frames, at visual N = 7, 13,
                 16 and inertial N = 5, 11.  A monocular window with one fixed frame has its scale free (J has an exact
                 null vector), so on visual windows "frame 0" fixes {0, 1} and "the last frame" {N - 2, N - 1};
  histories      a slot that held N = 16 (fp32) or N = 11 (fp64) reset to an N = 3 window, and an inertial slot taken
                 through three drop_victims (which takes windows with motion states only): the oracle, and bit for bit a
                 fresh twin slot fed the same window;
  hard windows   synth.hard_window at visual N = 8, 16 (far_depths, low_baseline, offset, general_w, cauchy_0.3) and
                 inertial N = 6, 11 (far_depths, offset, cauchy_0.01).  Left out: outliers (without a robust loss J^T J
                 does not depend on the residuals, so the kind only moves the state; the Cauchy kinds carry the same
                 outliers under the loss), rejected (its behind-camera landmarks are the post-pass's case,
                 test_gpu_batch_window.py; their rows are far_depths' rows with a sign), all (the union of the kinds
                 above), visual cauchy_0.01 and inertial general_w / cauchy_0.3 (the same linearisation branches as the
                 kinds run, on the other pipeline);
  refusals       an inertial N = 12 slot (its reduced system does not fit the shared memory of the factorisation):
                 EINVAL from covariance and landmarks(covariance=True), landmarks(covariance=False) still served, and no
                 slot's download or save blob changed.

Each case's bar follows from its conditioning: kappa, the condition number of the free-coordinate Schur complement in
the Jacobi scaling (chol_oracle.scaled_condition), times the pipeline's unit roundoff u (2^-53 fp64, 2^-24 fp32) times
C_BAR, floored at the bars of test_gpu_batch_window_covariance / test_gpu_batch_window_landmarks.  Frame blocks are
measured as |C - C_ref|_ij / sqrt(C_ref,ii C_ref,jj), Var(rho) relatively, point covariances as the frame blocks."""
import dataclasses

import numpy as np
import pytest

import landmark_oracle as lo
from oracle import ba_oracle, chol_oracle, cov_oracle
from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows, Edit, Planes
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from synthetic import synth
from test_gpu_batch_window_covariance import BAR_FP32, BAR_FP64, _err, _feed, _repack, _snap, _tracks
import test_gpu_batch_window_landmarks as tl

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"
C_BAR = 16                      # the bar is C_BAR kappa u, floored at the pipeline's bars below
FP64 = dict(name="fp64", u=2.0 ** -53, floor=(BAR_FP64[0], BAR_FP64[1], tl.BAR_FP64))
FP32 = dict(name="fp32", u=2.0 ** -24, floor=(BAR_FP32[0], BAR_FP32[1], tl.BAR_FP32))
M = 40                          # landmarks per generated window
T = 128                         # track stride of the downloads


def _handle(W, max_frames):
    return BundleAdjustor(max_windows=W, max_frames=max_frames, max_landmarks=64, max_obs=1024)


def _visual(N, seed, fixed=None):
    """cfg2 (frames 0 and 1 fixed unless `fixed` names the fixed frames), keypoints rounded to fp32 as the slots keep
    them, so that the reference sees the window the kernels see"""
    w, st = synth.make_cfg2(seed=seed, N=N, M=M)[:2]
    synth.f32_keypoints(w)
    if fixed is not None:
        w.frame_fixed = np.array([f in fixed for f in range(N)], dtype=np.uint8)
    return w, st, _tracks(w, planes=False)


def _inertial(N, seed, fixed=()):
    """cfg3 (the synthetic prior over frames 0 .. N - 2), keypoints rounded to fp32; N = 1: the N = 2 window's frame
    0 with its prior, and the tracks born there as one-observation tracks"""
    w, st = synth.make_cfg3(seed=seed, N=max(N, 2), M=M)[:2]
    synth.f32_keypoints(w)
    tr = _tracks(w, planes=False)
    if N == 1:
        tr = [dict(t, frames=[0], zs=t["zs"][:1]) for t in tr if t["frames"][0] == 0]
        w = dataclasses.replace(w, N=1, frame_fixed=w.frame_fixed[:1].copy(), n_imu=0, M=0, K=0)
    w.frame_fixed = np.array([f in fixed for f in range(N)], dtype=np.uint8)
    return w, st, tr


def _conditioning(wr, sr):
    """(kappa of the free-coordinate Schur complement in the Jacobi scaling, 1 without free frame coordinates;
    whether the free-coordinate system is positive definite, i.e. the status the reference predicts is OK)"""
    H = ba_oracle.normal_equations(wr, sr)[0]
    free = ba_oracle.free_mask(wr)
    try:
        np.linalg.cholesky(H[np.ix_(free, free)])
    except np.linalg.LinAlgError:
        return np.inf, False
    n = 15 * wr.N
    ff = np.flatnonzero(free[:n])
    fl = n + np.flatnonzero(free[n:])
    if len(ff) == 0:
        return 1.0, True
    Hfl = H[np.ix_(ff, fl)]
    S = H[np.ix_(ff, ff)] - Hfl @ (Hfl.T / np.diag(H)[fl][:, None])
    return chol_oracle.scaled_condition(S), True


def _case(bw, slot, w, model, fixed, pipe, label, prior=None):
    """the slot's covariance and landmarks(covariance) against the oracle at its downloaded state; returns
    (covariance record of all frames and tracks, landmarks record, ids) for further checks"""
    d = bw.download([slot], T)[0]
    imu = bw.imu_records([slot])[0] if w.use_inertial else None
    wr, sr, lms = _repack(w, d, model, imu, fixed, prior)
    N, ids = wr.N, [int(i) for i in d["ids"]]
    lm_of = {t: k for k, t in enumerate(lms)}
    tr = [lm_of.get(t) for t in ids]
    out = bw.covariance([slot], [list(range(N))], [ids])[0]
    lmk = bw.landmarks([slot], covariance=True)[0]
    assert np.array_equal(lmk["ids"], ids)
    assert np.array_equal(out["inv_depth_var"], lmk["inv_depth_var"], equal_nan=True)   # one arithmetic, bit for bit
    kappa, ok = _conditioning(wr, sr)
    if not ok:
        print(f"{label} [{pipe['name']}]: N {N}, singular: ENUMERIC")
        assert out["status"] == lmk["status"] == _lib.ENUMERIC
        assert np.isnan(out["cov"]).all() and np.isnan(out["inv_depth_var"]).all() and np.isnan(lmk["point_cov"]).all()
        return out, lmk, ids
    assert out["status"] == lmk["status"] == _lib.OK
    cov_ref, var_ref, Sig = cov_oracle.covariance(wr, sr, list(range(N)), tr, refine=True)
    pref = lo.point_covariance(wr, sr, tr, Sig=Sig)
    bar = [max(C_BAR * kappa * pipe["u"], f) for f in pipe["floor"]]
    C = out["cov"]
    e_cov = _err(C, cov_ref)                                  # rows / columns that are not free exactly 0
    var = out["inv_depth_var"]
    assert np.array_equal(np.isnan(var), np.isnan(var_ref))
    for m, t in zip(np.isnan(var), ids):                      # NaN exactly for the tracks with one observation
        assert m == (len(model[t]["frames"]) < 2)
    ok = ~np.isnan(var_ref)
    e_var = float(np.max(np.abs(var[ok] - var_ref[ok]) / var_ref[ok])) if ok.any() else 0.0
    e_pt = 0.0
    for P, R in zip(lmk["point_cov"], pref):
        assert np.isnan(P).all() == np.isnan(R).all()
        if not np.isnan(R).all():
            assert np.array_equal(P, P.T)
            s = np.sqrt(np.diag(R))
            e_pt = max(e_pt, float(np.max(np.abs(P - R) / np.outer(s, s))))
    assert np.array_equal(C, C.T) or np.allclose(C, C.T, rtol=0, atol=1e-12 * np.abs(C).max())
    nz = np.diag(C) > 0
    if nz.any():                                              # positive semi-definite in its own Jacobi scaling
        dc = np.sqrt(np.diag(C)[nz])
        Cs = C[np.ix_(nz, nz)] / np.outer(dc, dc)
        assert np.linalg.eigvalsh(0.5 * (Cs + Cs.T)).min() > -len(dc) * bar[0]
    print(f"{label} [{pipe['name']}]: N {N}, kappa {kappa:.3g}, frames {e_cov:.3g}, var {e_var:.3g}, "
          f"points {e_pt:.3g}, frames / (kappa u) {e_cov / (kappa * pipe['u']):.3g} (bars {bar[0]:.3g}, {bar[1]:.3g}, {bar[2]:.3g})")
    assert e_cov < bar[0] and e_var < bar[1] and e_pt < bar[2], (label, e_cov, e_var, e_pt, bar)
    return out, lmk, ids


def _one_call(bw, cases, seed):
    """every case's slot in one covariance call and one landmarks call, shuffled, frames and tracks in a permuted order:
    the records called one at a time bit for bit, and those the permuted blocks of the all-frames records"""
    rng = np.random.default_rng(seed)
    order = rng.permutation(len(cases))
    recs = []
    for k in order:
        slot, out, lmk, ids = cases[k]
        fr = [int(f) for f in rng.permutation(out["cov"].shape[0] // 15)]
        tk = [ids[j] for j in rng.permutation(len(ids))]
        recs.append((slot, fr, tk, out, ids))
    many = bw.covariance([r[0] for r in recs], [r[1] for r in recs], [r[2] for r in recs])
    lm_many = bw.landmarks([r[0] for r in recs], [r[2] for r in recs], covariance=True)
    for (slot, fr, tk, full, ids), m, lm in zip(recs, many, lm_many):
        one = bw.covariance([slot], [fr], [tk])[0]
        lm_one = bw.landmarks([slot], [tk], covariance=True)[0]
        assert m["status"] == one["status"] == full["status"]
        assert np.array_equal(m["cov"], one["cov"], equal_nan=True), slot
        assert np.array_equal(m["inv_depth_var"], one["inv_depth_var"], equal_nan=True), slot
        for key in ("ids", "point", "role", "point_cov", "inv_depth_var"):
            assert np.array_equal(lm[key], lm_one[key], equal_nan=True), (slot, key)
        cols = np.concatenate([15 * f + np.arange(15) for f in fr])
        assert np.array_equal(one["cov"], full["cov"][np.ix_(cols, cols)], equal_nan=True), slot
        pos = {t: j for j, t in enumerate(ids)}
        assert np.array_equal(one["inv_depth_var"], full["inv_depth_var"][[pos[t] for t in tk]], equal_nan=True)
        assert np.array_equal(lm_one["inv_depth_var"], one["inv_depth_var"], equal_nan=True)


def test_visual_windows_of_every_size_on_an_fp32_handle():
    """cfg2 at N = 1 ... 16 and an N = 1 window whose frame is free and unobserved, then all of them in one call.  The
    handle has an odd slot count: the second buffer set of the reduced systems, which the Schur sweep reads by bulk
    copies, must stay 16-byte aligned"""
    res = _handle(17, 16)
    bw = BatchWindows(res)
    wins = {}
    for N in range(1, 17):
        w, st, tr = _visual(N, 1000 + N)
        wins[N - 1] = (w, _feed(bw, N - 1, w, st, tr))
    w1, st1, tr1 = _visual(1, 1100, fixed=())                  # N = 1, its frame free and observed by nobody
    wins[16] = (w1, _feed(bw, 16, w1, st1, tr1))
    bw.solve(list(range(16)), max_iterations=3)
    cases = []
    for s, (w, m) in wins.items():
        out, lmk, ids = _case(bw, s, w, m, list(w.frame_fixed), FP32, f"visual N {w.N}" + (" free" if s == 16 else ""))
        cases.append((s, out, lmk, ids))
    assert cases[0][1]["status"] == _lib.OK and not cases[0][1]["cov"].any()       # the fixed frame: zero blocks
    assert cases[16][1]["status"] == _lib.ENUMERIC
    _one_call(bw, cases, 7)
    res.close()


def test_inertial_windows_of_every_size_and_the_n12_refusal():
    """cfg3 at N = 1 ... 11 on an fp64 handle of max_frames 12; then an N = 12 slot, fed and never solved, is refused by
    covariance and landmarks(covariance=True) with every slot unchanged, and its points are still served"""
    res = _handle(12, 12)
    bw = BatchWindows(res)
    wins = {}
    for N in range(1, 12):
        w, st, tr = _inertial(N, 1200 + N)
        wins[N - 1] = (w, _feed(bw, N - 1, w, st, tr))
    bw.solve(list(range(11)), max_iterations=2)
    cases = []
    for s, (w, m) in wins.items():
        out, lmk, ids = _case(bw, s, w, m, [0] * w.N, FP64, f"inertial N {w.N}")
        cases.append((s, out, lmk, ids))
    _one_call(bw, cases, 8)
    w12, st12, tr12 = _inertial(12, 1212)
    _feed(bw, 11, w12, st12, tr12)
    before = _snap(bw, list(range(12)))
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.covariance([11], [[0]], [[]])
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.covariance([3, 11], [[0], [0]], [[], []])
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.landmarks([11], covariance=True)
    pts = bw.landmarks([11, 3])
    assert pts[0]["status"] == _lib.OK and len(pts[0]["ids"]) == len(tr12)
    after = _snap(bw, list(range(12)))
    for x, y in zip(before[0], after[0]):
        for k in x:
            assert np.array_equal(x[k], y[k]), k
    assert before[1] == after[1]
    res.close()


def test_visual_windows_on_an_fp64_handle():
    """visual N = 2, 9, 16 next to an inertial N = 11 slot, so every window runs the fp64 pipeline (Ncap 16): solved in
    one call (launches shaped for an inertial N = 11 and a visual N = 16 window, each within the shared memory), then
    the inertial slot alone above the unnamed N = 16 slot (shaped for the named slot only)"""
    res = _handle(4, 16)
    bw = BatchWindows(res)
    wi, sti, tri = _inertial(11, 1311)
    mi = _feed(bw, 3, wi, sti, tri)
    wins = {}
    for s, N in enumerate((2, 9, 16)):
        w, st, tr = _visual(N, 1300 + N)
        wins[s] = (w, _feed(bw, s, w, st, tr))
    bw.solve([0, 1, 2, 3], max_iterations=2)
    bw.solve([3], max_iterations=1)                          # a solve that names only the inertial slot
    cases = [(s, *_case(bw, s, w, m, list(w.frame_fixed), FP64, f"visual N {w.N} on fp64")) for s, (w, m) in wins.items()]
    cases.append((3, *_case(bw, 3, wi, mi, [0] * wi.N, FP64, "inertial N 11 on Ncap 16")))
    _one_call(bw, cases, 9)
    res.close()


def _patterns(N, visual):
    one = (0, 1) if visual else (0,)
    last = (N - 2, N - 1) if visual else (N - 1,)
    return {"frame 0": one, "last frame": last, "first and last": (0, N - 1), "every other": tuple(range(0, N, 2)),
            "all but one": tuple(f for f in range(N) if f != N // 2), "all": tuple(range(N))}


@pytest.mark.parametrize("pipeline", ["visual", "inertial"])
def test_fixing_patterns(pipeline):
    """every fixing pattern; with every frame fixed the pose blocks are 0 and Var(rho) is 1 / H_ll (the inertial
    windows keep v, bg and ba free)"""
    visual = pipeline == "visual"
    sizes = (7, 13, 16) if visual else (5, 11)
    res = _handle(6 * len(sizes), 16 if visual else 12)
    bw = BatchWindows(res)
    runs, s = [], 0
    for N in sizes:
        for name, fixed in _patterns(N, visual).items():
            w, st, tr = _visual(N, 1400 + N, fixed) if visual else _inertial(N, 1400 + N, fixed)
            runs.append((s, name, w, _feed(bw, s, w, st, tr)))
            s += 1
    bw.solve(list(range(s)), max_iterations=2)
    for s, name, w, m in runs:
        out, lmk, ids = _case(bw, s, w, m, list(w.frame_fixed), FP32 if visual else FP64, f"{pipeline} N {w.N} {name}")
        if name == "all":
            C = out["cov"]
            for f in range(w.N):
                assert not C[15 * f:15 * f + 6].any() and not C[:, 15 * f:15 * f + 6].any()
            assert visual == (not C.any())
            d = bw.download([s], T)[0]
            wr, sr, lms = _repack(w, d, m, bw.imu_records([s])[0] if not visual else None, list(w.frame_fixed))
            H = ba_oracle.normal_equations(wr, sr)[0]
            pos = {t: j for j, t in enumerate(ids)}
            inv = np.array([1.0 / H[15 * wr.N + l, 15 * wr.N + l] for l in range(len(lms))])
            got = out["inv_depth_var"][[pos[t] for t in lms]]
            floor = (FP32 if visual else FP64)["floor"][1]
            assert np.max(np.abs(got - inv) / inv) < floor
    res.close()


def _drop_model(m):
    """the model of a slot after drop_victim: frame 0's observations leave, tracks re-anchor, frames shift down"""
    for t in list(m):
        if m[t]["frames"][0] == 0:
            m[t]["frames"].pop(0); m[t]["zs"].pop(0)
        if not m[t]["frames"]:
            del m[t]
            continue
        m[t]["frames"] = [f - 1 for f in m[t]["frames"]]


def _refeed(bw, slot, w, d, model, imu, prior):
    """a fresh slot fed the downloaded inertial window d: its frame states, the model's tracks in id order with the
    downloaded inverse depths, the IMU records imu and the prior (S, e) linearised at the frame states; returns its
    model"""
    bw.reset(slot, w)
    rho = dict(zip((int(i) for i in d["ids"]), d["inv_depth"]))
    tracks = [dict(old=t, frames=m["frames"], zs=m["zs"]) for t, m in sorted(model.items())]
    out = {}
    for f in range(len(d["frames"])):
        e = Edit(slot).frame(d["frames"][f], False, imu[f - 1] if f > 0 else None)
        born = []
        for t in tracks:
            if t["frames"][0] == f:
                e.new.append((f, t["zs"][0], rho[t["old"]]))
                born.append(t)
            elif f in t["frames"]:
                e.obs.append((t["id"], f, t["zs"][t["frames"].index(f)]))
        for t, i in zip(born, bw.edit([e])[0]):
            t["id"] = int(i)
            out[int(i)] = dict(frames=t["frames"], zs=t["zs"], role=model[t["old"]]["role"])
    bw.set_prior(slot, prior[0], prior[1], d["frames"])
    bw.set_planes([Planes(slot, np.concatenate([w.plane_normal, w.plane_distance[:, None]], axis=1))])
    return out


def _same(bw, a, b, N):
    """slots a and b give the same bits for every frame and track (their track ids may differ, their rows match)"""
    ra = bw.covariance([a], [list(range(N))], [bw.download([a], T)[0]["ids"]])[0]
    rb = bw.covariance([b], [list(range(N))], [bw.download([b], T)[0]["ids"]])[0]
    la, lb = bw.landmarks([a], covariance=True)[0], bw.landmarks([b], covariance=True)[0]
    assert ra["status"] == rb["status"] == _lib.OK
    assert np.array_equal(ra["cov"], rb["cov"]) and np.array_equal(ra["inv_depth_var"], rb["inv_depth_var"], equal_nan=True)
    for key in ("point", "role", "point_cov", "inv_depth_var"):
        assert np.array_equal(la[key], lb[key], equal_nan=True), key


@pytest.mark.parametrize("pipeline", ["visual", "inertial"])
def test_slot_histories(pipeline):
    """a slot reset from the largest window (solved) to N = 3 against a fresh twin: bit for bit at the fed state, and
    after both are solved in one call, their states to 1e-9 and each covariance against the oracle; inertial: a slot
    after three drop_victims against a fresh twin fed its window (states, tracks, IMU records and the prior the drops
    left), bit for bit.  Solved twins are not compared bit for bit: the solve sums its model costs (the IMU and prior
    terms of solve_kernel, the per-warp costs of the linearise sweep) with atomics, whose order varies, so two slots
    solved from the same window may end some ulps apart."""
    visual = pipeline == "visual"
    Nmax, pipe = (16, FP32) if visual else (11, FP64)
    make = _visual if visual else _inertial
    res = _handle(4, 16 if visual else 12)
    bw = BatchWindows(res)
    w, st, tr = make(Nmax, 1500)
    _feed(bw, 0, w, st, tr)
    bw.solve([0], max_iterations=2)
    w3, st3, tr3 = make(3, 1503)
    m0 = _feed(bw, 0, w3, st3, [dict(t) for t in tr3])
    m1 = _feed(bw, 1, w3, st3, [dict(t) for t in tr3])
    fixed = list(w3.frame_fixed)
    _case(bw, 0, w3, m0, fixed, pipe, f"{pipeline} N 3 after N {Nmax}")
    _case(bw, 1, w3, m1, fixed, pipe, f"{pipeline} N 3 fresh")
    _same(bw, 0, 1, 3)
    # solved in one call: the slot that held the larger window ends where the fresh one does, up to the ulps the
    # solve's atomic cost sums leave (a state left over from the larger window would move it far more)
    bw.solve([0, 1], max_iterations=2)
    d0, d1 = bw.download([0, 1], T)
    gap = max(float(np.max(np.abs(d0[k] - d1[k]) / (1.0 + np.abs(d1[k])))) for k in ("frames", "inv_depth"))
    print(f"{pipeline} N 3 solved after N {Nmax} / fresh: state gap {gap:.3g}")
    assert gap < 1e-9, gap
    _case(bw, 0, w3, m0, fixed, pipe, f"{pipeline} N 3 after N {Nmax}, solved")
    _case(bw, 1, w3, m1, fixed, pipe, f"{pipeline} N 3 fresh, solved")
    if not visual:
        w, st, tr = make(Nmax, 1510)
        m = _feed(bw, 2, w, st, tr)
        bw.solve([2], max_iterations=2)
        for k in range(3):
            S, e = bw.drop_victim([2], want=True, max_frames=12)
            _drop_model(m)
        N = Nmax - 3
        dk = 15 * N
        prior = (S[0, :dk * dk].reshape(dk, dk), e[0, :dk])
        d = bw.download([2], T)[0]
        imu = bw.imu_records([2])[0]
        m3 = _refeed(bw, 3, w, d, m, imu, prior)
        _case(bw, 2, w, m, [0] * N, pipe, f"inertial N {N} after three drops", prior=prior)
        _case(bw, 3, w, m3, [0] * N, pipe, f"inertial N {N} fed as the dropped slot", prior=prior)
        _same(bw, 2, 3, N)
    res.close()


@pytest.mark.parametrize("pipeline", ["visual", "inertial"])
def test_hard_windows(pipeline):
    visual = pipeline == "visual"
    kinds = ("far_depths", "low_baseline", "offset", "general_w", "cauchy_0.3") if visual else \
        ("far_depths", "offset", "cauchy_0.01")
    sizes = (8, 16) if visual else (6, 11)
    res = _handle(len(kinds) * len(sizes), 16 if visual else 12)
    bw = BatchWindows(res)
    runs = []
    for N in sizes:
        for kind in kinds:
            w, st = synth.hard_window(kind, inertial=not visual, N=N, M=M, seed=1600 + N)
            s = len(runs)
            runs.append((s, kind, w, _feed(bw, s, w, st, _tracks(w, planes=False))))
    bw.solve([r[0] for r in runs], max_iterations=3)
    for s, kind, w, m in runs:
        _case(bw, s, w, m, list(w.frame_fixed), FP32 if visual else FP64, f"{pipeline} N {w.N} {kind}")
    res.close()
