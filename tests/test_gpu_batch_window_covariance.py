"""pvio_b200_batch_window_covariance: the covariance of resident windows against cov_oracle.covariance at the slot's
downloaded state, the selection of frames and tracks, its structure, its numeric status, and that it changes no slot."""
import dataclasses

import numpy as np
import pytest

from oracle import cov_oracle
from pvio_b200 import _lib
from pvio_b200.batch_window import LANDMARK, SMALL_PLANE, BatchWindows, Edit, Planes
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.window import State
from synthetic import synth

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"
# |C - C_ref|_ij / sqrt(C_ref,ii C_ref,jj) of the frame blocks, and the relative error of the inverse-depth variances:
# inertial windows run the fp64 pipeline, visual-only ones fp32 Jacobians.  Set from the first H100 run (DESIGN 5b):
# worst seen 4.9e-7 / 2.2e-5 (fp64), 2.8e-6 / 8.9e-6 (fp32)
BAR_FP64, BAR_FP32 = (2e-6, 1e-4), (2e-3, 2e-3)


def _tracks(w, planes=True):
    out = []
    for l in range(w.M):
        ks = range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1])
        role = SMALL_PLANE if (planes and w.lm_anchor[l] == 0 and l % 5 == 0) else LANDMARK
        out.append(dict(frames=[int(w.lm_anchor[l])] + [int(w.obs_frame[k]) for k in ks],
                        zs=[w.lm_z_ref[l]] + [w.obs_z[k] for k in ks], lm=l, role=role))
    for t in range(w.n_ptracks if planes else 0):
        ks = list(range(w.pt_obs_begin[t], w.pt_obs_begin[t + 1]))
        if t % 6 == 0:
            ks = ks[:1]
        out.append(dict(frames=[int(w.pt_obs_frame[k]) for k in ks], zs=[w.pt_obs_z[k] for k in ks], lm=None,
                        role=int(w.pt_plane[t]), rho=0.2 + 0.01 * (t % 7)))
    return out


def _feed(bw, slot, w, st, tracks, skip_obs_frame=None):
    """the window fed frame by frame into a slot (and its prior and planes when inertial); returns id -> track"""
    bw.reset(slot, w)
    rec = _lib.PackedArgs(w, st).keep["imu"].reshape(-1, 288) if (w.use_inertial and w.N > 1) else None
    model = {}
    for f in range(w.N):
        e = Edit(slot).frame(np.concatenate([st.q[f], st.p[f], st.v[f], st.bg[f], st.ba[f]]), bool(w.frame_fixed[f]),
                             rec[f - 1] if (rec is not None and f > 0) else None)
        born = []
        for t in tracks:
            if f == skip_obs_frame and f in t["frames"]:
                continue
            if t["frames"][0] == f:
                e.new.append((f, t["zs"][0], st.rho[t["lm"]] if t["lm"] is not None else t["rho"]))
                born.append(t)
            elif f in t["frames"]:
                e.obs.append((t["id"], f, t["zs"][t["frames"].index(f)]))
        for t, i in zip(born, bw.edit([e])[0]):
            t["id"] = int(i)
            model[int(i)] = dict(frames=[g for g in t["frames"] if g != skip_obs_frame],
                                 zs=[z for g, z in zip(t["frames"], t["zs"]) if g != skip_obs_frame], role=t["role"])
    if w.use_inertial:
        x0 = np.concatenate([w.prior_q0, w.prior_p0, w.prior_v0, w.prior_bg0, w.prior_ba0], axis=1)
        bw.set_prior(slot, w.prior_S, w.prior_e, x0)
        p = Planes(slot, np.concatenate([w.plane_normal, w.plane_distance[:, None]], axis=1))
        for i, t in model.items():
            if t["role"] != LANDMARK:
                p.role(i, t["role"])
        bw.set_planes([p])
    return model


def _repack(w, d, model, imu, fixed, prior=None):
    """the slot's window as ba_oracle sees it: landmarks (role < 0, >= 2 observations) and plane tracks in id order,
    states and inverse depths from the download d, IMU records imu [N - 1, 288]; returns (win, state, landmark ids)"""
    row = {int(t): r for r, t in enumerate(d["ids"])}
    N = len(d["frames"])
    lms = [i for i in sorted(model) if model[i]["role"] < 0 and len(model[i]["frames"]) >= 2]
    pts = [i for i in sorted(model) if model[i]["role"] >= 0]
    wr = dataclasses.replace(w)
    wr.N, wr.frame_fixed = N, np.array(fixed, dtype=np.uint8)
    of, oz, begins = [], [], [0]
    for i in lms:
        of += model[i]["frames"][1:]; oz += model[i]["zs"][1:]; begins.append(len(of))
    wr.M, wr.K = len(lms), len(of)
    wr.lm_anchor = np.array([model[i]["frames"][0] for i in lms], dtype=np.int32)
    wr.lm_z_ref = np.array([model[i]["zs"][0] for i in lms]).reshape(-1, 2)
    wr.lm_obs_begin, wr.obs_frame = np.array(begins, dtype=np.int32), np.array(of, dtype=np.int32)
    wr.obs_z = np.array(oz).reshape(-1, 2)
    wr.lm_in_victim = np.zeros(len(lms), dtype=np.uint8)
    pf, pz, pb = [], [], [0]
    for i in pts:
        pf += model[i]["frames"]; pz += model[i]["zs"]; pb.append(len(pf))
    wr.n_ptracks = len(pts)
    wr.pt_plane = np.array([model[i]["role"] for i in pts], dtype=np.int32)
    wr.pt_obs_begin, wr.pt_obs_frame = np.array(pb, dtype=np.int32), np.array(pf, dtype=np.int32)
    wr.pt_obs_z = np.array(pz).reshape(-1, 2)
    fr = d["frames"]
    if w.use_inertial:
        wr.n_imu = N - 1
        wr.imu_frame_i, wr.imu_frame_j = np.arange(N - 1, dtype=np.int32), np.arange(1, N, dtype=np.int32)
        L = _lib
        wr.imu_dt = imu[:, L.IMU_DT].copy()
        wr.imu_dq, wr.imu_dp, wr.imu_dv = (imu[:, o:o + k].copy() for o, k in ((L.IMU_DQ, 4), (L.IMU_DP, 3), (L.IMU_DV, 3)))
        wr.imu_sqrt_inv_cov = imu[:, L.IMU_SQRT_INV_COV:L.IMU_SQRT_INV_COV + 225].reshape(-1, 15, 15).copy()
        for name, o in (("imu_dq_dbg", L.IMU_DQ_DBG), ("imu_dp_dbg", L.IMU_DP_DBG), ("imu_dp_dba", L.IMU_DP_DBA),
                        ("imu_dv_dbg", L.IMU_DV_DBG), ("imu_dv_dba", L.IMU_DV_DBA)):
            setattr(wr, name, imu[:, o:o + 9].reshape(-1, 3, 3).copy())
        wr.imu_bg0, wr.imu_ba0 = imu[:, L.IMU_BG0:L.IMU_BG0 + 3].copy(), imu[:, L.IMU_BA0:L.IMU_BA0 + 3].copy()
        if prior is not None:
            S, e = prior
            wr.n_prior, wr.prior_frames, wr.prior_S, wr.prior_e = N, np.arange(N, dtype=np.int32), S, e
            wr.prior_q0, wr.prior_p0, wr.prior_v0 = fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy()
            wr.prior_bg0, wr.prior_ba0 = fr[:, 10:13].copy(), fr[:, 13:16].copy()
    wr.validate()
    st = State(fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy(), fr[:, 10:13].copy(), fr[:, 13:16].copy(),
               np.array([d["inv_depth"][row[i]] for i in lms]))
    return wr, st, lms


def _err(C, R):
    d = np.sqrt(np.abs(np.diag(R)))
    den = np.outer(d, d)
    nz = den > 0
    assert np.all(C[~nz] == 0), "rows / columns that are not free must be 0"
    return float(np.max(np.abs(C - R)[nz] / den[nz])) if nz.any() else 0.0


def _check(bw, slot, w, model, fixed, bar, prior=None):
    d = bw.download([slot], 600)[0]
    imu = bw.imu_records([slot])[0] if w.use_inertial else None
    wr, sr, lms = _repack(w, d, model, imu, fixed, prior)
    N = wr.N
    ids = [int(i) for i in d["ids"]]
    out = bw.covariance([slot], [list(range(N))], [ids])[0]
    assert out["status"] == _lib.OK
    lm_of = {t: k for k, t in enumerate(lms)}
    cov_ref, var_ref, _ = cov_oracle.covariance(wr, sr, list(range(N)), [lm_of.get(t) for t in ids], refine=True)
    e_cov = _err(out["cov"], cov_ref)
    assert np.array_equal(np.isnan(out["inv_depth_var"]), np.isnan(var_ref))
    ok = ~np.isnan(var_ref)
    e_var = float(np.max(np.abs(out["inv_depth_var"][ok] - var_ref[ok]) / var_ref[ok]))
    print(f"slot {slot}: N {N}, frames error {e_cov:.3g}, inverse-depth variance error {e_var:.3g}")
    assert e_cov < bar[0] and e_var < bar[1], (e_cov, e_var)
    for m, t in zip(np.isnan(out["inv_depth_var"]), ids):            # NaN exactly for plane and one-observation tracks
        assert m == (model[t]["role"] >= 0 or len(model[t]["frames"]) < 2)
    C = out["cov"]
    assert np.array_equal(C, C.T) or np.allclose(C, C.T, rtol=0, atol=1e-12 * np.abs(C).max())
    assert np.linalg.eigvalsh(0.5 * (C + C.T)).min() > -1e-9 * np.abs(C).max()
    return out, d


def test_inertial_windows_match_the_oracle_before_and_after_a_drop():
    """cfg4 windows (first window with its gauge prior, plane tracks, role -2 tracks, one-observation plane tracks),
    solved in their slots; the covariance against the oracle, then again after drop_victim with the new prior."""
    res = BundleAdjustor(max_windows=3, max_frames=9, max_landmarks=600, max_obs=4000)
    bw = BatchWindows(res)
    wins = [synth.make_cfg4(seed=990 + i, N=(7, 9)[i], M=150)[:2] for i in range(2)]
    models = [_feed(bw, i + 1, w, st, _tracks(w)) for i, (w, st) in enumerate(wins)]
    bw.solve([1, 2], max_iterations=4)
    for i, (w, _) in enumerate(wins):
        _check(bw, i + 1, w, models[i], [0] * w.N, BAR_FP64)
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
        w1 = dataclasses.replace(w)
        _check(bw, i + 1, w1, m, [0] * (w.N - 1), BAR_FP64, prior=(S[i, :dk * dk].reshape(dk, dk), e[i, :dk]))
    res.close()


def _visual(bw, slot, seed=995, skip=None):
    w, st = synth.make_cfg2(seed=seed, N=6, M=120)[:2]
    return w, _feed(bw, slot, w, st, _tracks(w, planes=False), skip_obs_frame=skip)


def test_visual_windows_selection_structure_and_status():
    """cfg2 windows with two fixed frames on an fp32 handle: the oracle; naming {a, b} gives the single-frame calls'
    diagonal blocks bit for bit; fixed poses and v / bg / ba are 0; a twin slot gives the same bits; a slot with an
    unobserved free frame is ENUMERIC with NaN outputs while the other records of the call are unaffected."""
    res = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=600, max_obs=4000)
    bw = BatchWindows(res)
    w, m = _visual(bw, 0)
    _visual(bw, 1)
    assert w.frame_fixed.sum() == 2
    bw.solve([0, 1], max_iterations=3)
    out, d = _check(bw, 0, w, m, list(w.frame_fixed), BAR_FP32)
    C = out["cov"]
    for f in range(w.N):
        blk = C[15 * f:15 * f + 15, :]
        assert np.all(blk[6:] == 0) and np.all(C[:, 15 * f + 6:15 * f + 15] == 0)
        if w.frame_fixed[f]:
            assert np.all(blk == 0)
    ids = list(d["ids"])
    a, b = [f for f in range(w.N) if not w.frame_fixed[f]][:2]
    two = bw.covariance([0], [[a, b]], [ids[:5]])[0]
    one_a = bw.covariance([0], [[a]], [[]])[0]["cov"]
    one_b = bw.covariance([0], [[b]], [[]])[0]["cov"]
    assert np.array_equal(two["cov"][:15, :15], one_a) and np.array_equal(two["cov"][15:, 15:], one_b)
    r = bw.covariance([0, 1], [[a, b], [a, b]], [ids[:20], list(bw.download([1], 600)[0]["ids"][:20])])
    assert np.array_equal(r[0]["cov"], r[1]["cov"]) and np.array_equal(r[0]["inv_depth_var"], r[1]["inv_depth_var"])
    # a free frame nobody observes: the system is singular
    free = [f for f in range(w.N) if not w.frame_fixed[f]]
    _visual(bw, 3, skip=free[-1])
    r = bw.covariance([3, 0], [[0, 1], [a]], [[], ids[:4]])
    assert r[0]["status"] == _lib.ENUMERIC and np.isnan(r[0]["cov"]).all()
    assert r[1]["status"] == _lib.OK and np.array_equal(r[1]["cov"], one_a)
    res.close()


def _snap(bw, slots):
    return [bw.download(slots, 600), bw.save(slots)]


def test_no_side_effects_rejections_and_launch_count():
    """every slot's download and save blob are byte-identical after the call and after every rejection; the launch
    count is the same at 8 and 264 records"""
    W = 264
    res = BundleAdjustor(max_windows=W, max_frames=6, max_landmarks=200, max_obs=1200)
    bw = BatchWindows(res)
    w, st = synth.make_cfg2(seed=997, N=5, M=60)[:2]
    tr = _tracks(w, planes=False)
    for s in range(W):
        _feed(bw, s, w, st, [dict(t) for t in tr])
    bw.solve([0, 1, 2], max_iterations=2)
    ids = [int(i) for i in bw.download([0], 200)[0]["ids"]]
    before = _snap(bw, [0, 1, 2])
    bw.covariance([0, 1], [[1, 2], [3]], [ids[:10], ids[10:12]])
    bad = [([0, 0], [[1], [2]], [[], []]),                     # slot twice
           ([W], [[1]], [[]]),                                 # slot out of range
           ([0], [[5]], [[]]),                                 # frame out of range
           ([0], [[1, 1]], [[]]),                              # frame twice
           ([0], [[]], [[]]),                                  # asking for nothing
           ([0], [[1]], [[ids[0], ids[0]]]),                   # track twice
           ([0], [[1]], [[10 ** 6]])]                          # unknown track
    for args in bad:
        with pytest.raises(PvioB200Error, match=EINVAL):
            bw.covariance(*args)
    after = _snap(bw, [0, 1, 2])
    for x, y in zip(before[0], after[0]):
        for k in x:
            assert np.array_equal(x[k], y[k]), k
    assert before[1] == after[1]
    counts = []
    for n in (8, W):
        l0 = res.kernel_launches
        bw.covariance(list(range(n)), [[1]] * n, [ids[:3]] * n)
        counts.append(res.kernel_launches - l0)
    assert counts[0] == counts[1] == 4, counts
    res.close()
