"""Plane factors in the resident batched windows (pvio_b200_batch_window_set_planes): every track of a slot has a role --
a landmark (-1), a landmark kept out of the marginaliser's victim set (-2), or a plane track of plane p >= 0 -- and the
slot keeps its plane parameters; the solve sees exactly the window a re-pack of the same tracks in id order gives it."""
import ctypes as C
import dataclasses

import numpy as np
import pytest

from pvio_b200 import _lib
from pvio_b200.batch_window import LANDMARK, SMALL_PLANE, BatchWindows, Edit, Planes, _constants
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.window import State
from synthetic import synth
from synthetic.sequence import BatchPlayer, Chain, Run

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"
SUMMARY_KEYS = ("iterations", "accepted_steps", "termination", "initial_cost", "final_cost", "final_radius", "final_mu")


def _tracks(w):
    """the landmarks and plane tracks of a cfg4 window as one track list: frames, keypoints, initial inverse depth, role.
    Every 5th landmark anchored in frame 0 takes role -2; every 6th plane track keeps its first observation only."""
    out = []
    for l in range(w.M):
        ks = range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1])
        role = SMALL_PLANE if (w.lm_anchor[l] == 0 and l % 5 == 0) else LANDMARK
        out.append(dict(frames=[int(w.lm_anchor[l])] + [int(w.obs_frame[k]) for k in ks],
                        zs=[w.lm_z_ref[l]] + [w.obs_z[k] for k in ks], lm=l, role=role))
    for t in range(w.n_ptracks):
        ks = list(range(w.pt_obs_begin[t], w.pt_obs_begin[t + 1]))
        if t % 6 == 0:
            ks = ks[:1]
        out.append(dict(frames=[int(w.pt_obs_frame[k]) for k in ks], zs=[w.pt_obs_z[k] for k in ks], lm=None,
                        role=int(w.pt_plane[t]), rho=0.2 + 0.01 * (t % 7)))
    return out


def _feed(bw, slot, w, st, tracks, planes=True):
    """the window fed frame by frame into a resident slot, then its roles and planes in one set_planes; returns
    id -> track (the host model of the slot)"""
    bw.reset(slot, w)
    rec = _lib.PackedArgs(w, st).keep["imu"].reshape(-1, 288)
    model = {}
    for f in range(w.N):
        e = Edit(slot).frame(np.concatenate([st.q[f], st.p[f], st.v[f], st.bg[f], st.ba[f]]), False,
                             rec[f - 1] if f > 0 else None)
        born = []
        for t in tracks:
            if t["frames"][0] == f:
                e.new.append((f, t["zs"][0], st.rho[t["lm"]] if t["lm"] is not None else t["rho"]))
                born.append(t)
            elif f in t["frames"]:
                e.obs.append((t["id"], f, t["zs"][t["frames"].index(f)]))
        for t, i in zip(born, bw.edit([e])[0]):
            t["id"] = int(i)
            model[int(i)] = dict(frames=list(t["frames"]), zs=list(t["zs"]), role=t["role"])
    x0 = np.concatenate([w.prior_q0, w.prior_p0, w.prior_v0, w.prior_bg0, w.prior_ba0], axis=1)
    bw.set_prior(slot, w.prior_S, w.prior_e, x0)
    if planes:
        p = Planes(slot, np.concatenate([w.plane_normal, w.plane_distance[:, None]], axis=1))
        for i, t in model.items():
            if t["role"] != LANDMARK:
                p.role(i, t["role"])
        bw.set_planes([p])
    return model


def _repack(w, d, model, prior=None):
    """the window of a download as a gather packs it: landmarks (role < 0, >= 2 observations) and plane tracks in id
    order, lm_in_victim = anchored in frame 0 and not role -2; states and inverse depths from the download"""
    row = {int(t): r for r, t in enumerate(d["ids"])}
    assert sorted(model) == sorted(row)
    N = len(d["frames"])
    lms = [i for i in sorted(model) if model[i]["role"] < 0 and len(model[i]["frames"]) >= 2]
    pts = [i for i in sorted(model) if model[i]["role"] >= 0]
    wr = dataclasses.replace(w)
    wr.N, wr.frame_fixed = N, np.zeros(N, dtype=np.uint8)
    of, oz, begins = [], [], [0]
    for i in lms:
        of += model[i]["frames"][1:]; oz += model[i]["zs"][1:]; begins.append(len(of))
    wr.M, wr.K = len(lms), len(of)
    wr.lm_anchor = np.array([model[i]["frames"][0] for i in lms], dtype=np.int32)
    wr.lm_z_ref = np.array([model[i]["zs"][0] for i in lms]).reshape(-1, 2)
    wr.lm_obs_begin, wr.obs_frame = np.array(begins, dtype=np.int32), np.array(of, dtype=np.int32)
    wr.obs_z = np.array(oz).reshape(-1, 2)
    wr.lm_in_victim = np.array([model[i]["frames"][0] == 0 and model[i]["role"] != SMALL_PLANE for i in lms], dtype=np.uint8)
    pf, pz, pb = [], [], [0]
    for i in pts:
        pf += model[i]["frames"]; pz += model[i]["zs"]; pb.append(len(pf))
    wr.n_ptracks = len(pts)
    wr.pt_plane = np.array([model[i]["role"] for i in pts], dtype=np.int32)
    wr.pt_obs_begin, wr.pt_obs_frame = np.array(pb, dtype=np.int32), np.array(pf, dtype=np.int32)
    wr.pt_obs_z = np.array(pz).reshape(-1, 2)
    wr.n_imu = N - 1
    wr.imu_frame_i, wr.imu_frame_j = np.arange(N - 1, dtype=np.int32), np.arange(1, N, dtype=np.int32)
    for k in ('imu_dt', 'imu_dq', 'imu_dp', 'imu_dv', 'imu_sqrt_inv_cov', 'imu_dq_dbg', 'imu_dp_dbg', 'imu_dp_dba',
              'imu_dv_dbg', 'imu_dv_dba', 'imu_bg0', 'imu_ba0'):
        setattr(wr, k, getattr(w, k)[w.N - N:].copy())
    fr = d["frames"]
    if prior is not None:                            # the prior drop_victim left: S, e over frames 0 .. N - 1
        S, e = prior
        wr.n_prior, wr.prior_frames, wr.prior_S, wr.prior_e = N, np.arange(N, dtype=np.int32), S, e
        wr.prior_q0, wr.prior_p0, wr.prior_v0 = fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy()
        wr.prior_bg0, wr.prior_ba0 = fr[:, 10:13].copy(), fr[:, 13:16].copy()
    wr.validate()
    st = State(fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy(), fr[:, 10:13].copy(), fr[:, 13:16].copy(),
               np.array([d["inv_depth"][row[i]] for i in lms]))
    return wr, st, lms


def _packed_solve(pk, packs, iters):
    for i, (wr, sr, _) in enumerate(packs):
        pk.batch_set(i, wr, sr)
    pk.batch_upload(len(packs))
    pk.batch_solve(len(packs), max_iterations=iters)
    return pk.batch_download_state(len(packs), 9, 400)


def _compare(sm, after, packs, ref, exact):
    """resident (summaries, downloads) against the re-packed batch solve; returns the worst relative difference"""
    frames, rho, sm_ref = ref
    worst = 0.0
    for i, (wr, _, lms) in enumerate(packs):
        row = {int(t): r for r, t in enumerate(after[i]["ids"])}
        got = np.array([after[i]["inv_depth"][row[t]] for t in lms])
        fr = frames[i, :wr.N].reshape(wr.N, 16)
        for k in ("iterations", "accepted_steps", "termination"):
            assert sm[i][k] == sm_ref[i][k], (i, k)
        assert sm[i]["iterations"] > 0
        if exact:
            assert np.array_equal(after[i]["frames"], fr), i
            assert np.array_equal(got, rho[i, :wr.M]), i
            for k in SUMMARY_KEYS:
                assert sm[i][k] == sm_ref[i][k], (i, k)
        worst = max(worst, np.abs(after[i]["frames"] - fr).max(), np.max(np.abs(got - rho[i, :wr.M]) / np.abs(rho[i, :wr.M])),
                    abs(sm[i]["final_cost"] - sm_ref[i]["final_cost"]) / sm_ref[i]["final_cost"])
    assert worst < 2e-6, worst
    return worst


def _windows(n):
    return [synth.make_cfg4(seed=960 + i, N=(6, 8, 9)[i % 3], M=200)[:2] for i in range(n)]


def test_plane_windows_solve_as_the_repacked_batch():
    """3 inertial cfg4 windows with a prior, landmarks, 2 planes, role -2 tracks and plane tracks of 1 to N observations,
    in resident slots, solved there; then a drop and an edit that removes tracks of every role, solved again.  Each time
    against the same windows re-packed (batch_set_window, id order) and solved by batch_solve over the same n: equal
    iteration counts, accepted steps and terminations; states, inverse depths and costs bit for bit when two runs of the
    re-packed path agree bit for bit (otherwise within 2e-6, the bar of the resident keyframe cycle, since the re-packed
    path itself then differs in the last bits from run to run)."""
    n, iters = 3, 8
    wins = _windows(n)
    res = BundleAdjustor(max_windows=n, max_frames=9, max_landmarks=400, max_obs=3000)
    pk = BundleAdjustor(max_windows=n, max_frames=9, max_landmarks=400, max_obs=3000)
    bw = BatchWindows(res)
    trs = [_tracks(w) for w, _ in wins]
    models = [_feed(bw, i, w, st, tr) for i, ((w, st), tr) in enumerate(zip(wins, trs))]
    for m in models:
        roles = [t["role"] for t in m.values()]
        assert roles.count(SMALL_PLANE) > 3 and min(roles) == SMALL_PLANE and max(roles) == 1
        assert min(len(t["frames"]) for t in m.values() if t["role"] >= 0) == 1
    worst = []
    for rnd in range(2):
        before = bw.download(range(n), 400)
        packs = [_repack(w, d, m, prior) for (w, _), d, m, prior in zip(wins, before, models, priors if rnd else [None] * n)]
        assert all(p[0].n_ptracks > 20 for p in packs)
        sm = bw.solve(list(range(n)), max_iterations=iters)
        after = bw.download(range(n), 400)
        a, b = _packed_solve(pk, packs, iters), _packed_solve(pk, packs, iters)
        exact = np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
        worst.append(_compare(sm, after, packs, a, exact))
        for d in after:                                              # plane tracks take no part in the post-pass
            assert d["valid"].any()
        for i, m in enumerate(models):
            row = {int(t): r for r, t in enumerate(after[i]["ids"])}
            assert all(after[i]["valid"][row[t]] == 0 and after[i]["quality"][row[t]] == 0.0 for t in m if m[t]["role"] >= 0)
        if rnd == 1:
            break
        # the victim leaves (plane tracks and role -2 tracks are re-anchored like any track), then tracks of every role go
        S, e = bw.drop_victim(list(range(n)), want=True, max_frames=9)
        priors = []
        for i, ((w, _), m) in enumerate(zip(wins, models)):
            d = 15 * (w.N - 1)
            priors.append((S[i, :d * d].reshape(d, d).copy(), e[i, :d].copy()))
            for t in list(m):
                if m[t]["frames"][0] == 0:
                    m[t]["frames"].pop(0); m[t]["zs"].pop(0)
                if not m[t]["frames"]:
                    del m[t]
                    continue
                m[t]["frames"] = [f - 1 for f in m[t]["frames"]]
        edits = []
        for i, m in enumerate(models):
            gone = [[t for t in sorted(m) if m[t]["role"] == r][:3] for r in (LANDMARK, SMALL_PLANE, 0, 1)]
            ed = Edit(i)
            ed.remove = [t for g in gone for t in g]
            for t in ed.remove:
                del m[t]
            edits.append(ed)
        bw.edit(edits)
    print("resident plane windows vs re-packed batch: worst difference per round", worst)
    res.close()
    pk.close()


def _rel_prior(S, e, S1, e1, H1, tol, noise_abs=1e-7):
    hs = np.maximum(np.sqrt(np.abs(np.diag(H1))), 1e-3)
    L, L1 = S.T @ S, S1.T @ S1
    eL = np.max(np.abs(L - L1) / (tol * np.outer(hs, hs) + noise_abs))
    ev = np.max(np.abs(S.T @ e - S1.T @ e1)) / np.max(np.abs(S1.T @ e1))
    return eL, ev


def test_marginaliser_skips_plane_and_small_plane_tracks():
    """drop_victim(want=True) on a slot whose victim frame is seen by plane tracks and role -2 tracks gives the prior
    ba_marginalize gives the re-packed window, where those tracks have lm_in_victim = 0 (the bars of
    test_batch_marginalize_matches_single_window_and_oracle)."""
    w, st = synth.make_cfg4(seed=970, N=8, M=220)[:2]
    res = BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=400, max_obs=3000)
    one = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=400, max_obs=3000)
    bw = BatchWindows(res)
    model = _feed(bw, 1, w, st, _tracks(w))
    assert sum(t["role"] >= 0 and t["frames"][0] == 0 for t in model.values()) > 5
    assert sum(t["role"] == SMALL_PLANE and t["frames"][0] == 0 for t in model.values()) > 5
    bw.solve([1], max_iterations=4)
    d = bw.download([1], 400)[0]
    wr, sr, _ = _repack(w, d, model)
    assert wr.lm_in_victim.sum() < (wr.lm_anchor == 0).sum()
    S, e = bw.drop_victim([1], want=True, max_frames=9)
    dk = 15 * (w.N - 1)
    S, e = S[0, :dk * dk].reshape(dk, dk), e[0, :dk]
    S1, e1, H1, _ = one.marginalize_frame(wr, sr, 0, want_info=True)
    eL, ev = _rel_prior(S, e, S1, e1, H1, 1e-9)
    assert eL < 1.0 and ev < 1e-9, (eL, ev)
    # the same window with every track a landmark gives a different prior: the roles reach the marginaliser
    wl = dataclasses.replace(wr, lm_in_victim=(wr.lm_anchor == 0).astype(np.uint8))
    S2, e2 = one.marginalize_frame(wl, sr, 0)
    assert _rel_prior(S2, e2, S1, e1, H1, 1e-9)[0] > 1.0
    res.close()
    one.close()


def _plane_slot(bw, slot, seed=975):
    w, st = synth.make_cfg4(seed=seed, N=7, M=160)[:2]
    return w, _feed(bw, slot, w, st, _tracks(w))


def _agree(x, y, exact):
    """two downloads of one slot: bit for bit when exact, else the integers equal and the states within 2e-6"""
    for k in x:
        if exact or x[k].dtype.kind in "iu":
            assert np.array_equal(x[k], y[k]), k
        else:
            assert np.allclose(x[k], y[k], rtol=2e-6, atol=2e-6), (k, np.abs(x[k] - y[k]).max())


def _summaries_agree(x, y, exact):
    for k in SUMMARY_KEYS:
        if exact or k in ("iterations", "accepted_steps", "termination"):
            assert x[k] == y[k], k
        else:
            assert abs(x[k] - y[k]) <= 2e-6 * abs(y[k]), k


def test_capacity_growth_keeps_other_slots_plane_tables():
    """Slot 0 holds plane tracks; a set_planes on slot 1 then pushes the plane-track count past the handle's plane-table
    capacity.  Slot 0's next solve equals the same solve on two handles where no growth happened: bit for bit when those
    two agree bit for bit (the inertial latency-path solve may differ in the last bits from run to run, DESIGN 5b; then
    within 2e-6)."""
    hs = [BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=640, max_obs=3000) for _ in range(3)]
    bws = [BatchWindows(h) for h in hs]
    w, ma = _plane_slot(bws[0], 0)
    for bw in bws[1:]:
        _plane_slot(bw, 0)
    bwa = bws[0]
    bwa.reset(1, w)
    bwa.edit([Edit(1).frame(np.concatenate([[0, 0, 0, 1], np.zeros(12)]))])
    e = Edit(1)
    e.new = [(0, np.array([0.01 * (i % 40), 0.02 * (i // 40)]), 0.3) for i in range(300)]   # more than 256 plane tracks
    ids = bwa.edit([e])[0]
    p = Planes(1, [[0.0, 0.0, 1.0, -1.4]])
    for i in ids:
        p.role(int(i), 0)
    bwa.set_planes([p])
    sm = [bw.solve([0], max_iterations=6)[0] for bw in bws]
    ds = [bw.download([0], 640)[0] for bw in bws]
    exact = all(np.array_equal(ds[1][k], ds[2][k]) for k in ds[1]) and all(sm[1][k] == sm[2][k] for k in SUMMARY_KEYS)
    print("growth-free handles agree bit for bit:", exact)
    _agree(ds[0], ds[1], exact)
    _summaries_agree(sm[0], sm[1], exact)
    assert sm[0]["iterations"] > 0 and sum(t["role"] >= 0 for t in ma.values()) > 20
    for h in hs:
        h.close()


def _snap(bw, slots, stride=640):
    return [{k: v.copy() for k, v in d.items()} for d in bw.download(slots, stride)]


def _same(x, y):
    return all(all(np.array_equal(p[k], q[k]) for k in p) for p, q in zip(x, y))


def test_rejections_change_nothing():
    """Every rejection of set_planes -- and a reset that passes plane arrays -- leaves every slot's download unchanged,
    including a call whose first record is valid and whose second is not."""
    b = BundleAdjustor(max_windows=3, max_frames=9, max_landmarks=640, max_obs=3000)
    bw = BatchWindows(b)
    w, m0 = _plane_slot(bw, 0, 976)
    _, m1 = _plane_slot(bw, 1, 977)
    bw.solve([0, 1], max_iterations=2)
    dead = Edit(1)
    dead.remove = [min(m1)]
    bw.edit([dead])
    snap = _snap(bw, [0, 1])
    lm0 = [t for t in sorted(m0) if m0[t]["role"] == LANDMARK]
    pt0 = [t for t in sorted(m0) if m0[t]["role"] == 1]
    ok = Planes(0).role(lm0[0], SMALL_PLANE, 0.77)                    # valid on its own: would change an inverse depth
    P = lambda s, planes=None: Planes(s, planes)
    bad = [
        [P(2)],                                                      # slot not resident
        [P(0), P(0)],                                                # a slot named twice
        [P(0, np.zeros((5, 4)))],                                    # more than 4 planes
        [ok, P(1).role(10 ** 6, LANDMARK)],                          # unknown track
        [ok, P(1).role(min(m1), LANDMARK)],                          # a dead track
        [P(0).role(lm0[1], LANDMARK).role(lm0[1], SMALL_PLANE)],     # a track named twice
        [P(0).role(lm0[1], 2)],                                      # a role >= the plane count
        [P(0).role(lm0[1], -3)],
        [P(0, [[0, 0, 1, np.nan]])],                                 # non-finite plane parameters
        [P(0, [[0, 0, np.inf, 1.0]])],
        [ok, P(1).role(max(m1), LANDMARK, np.inf)],                  # an infinite inverse depth
        [P(0, [[0, 0, 1, -1.4]])],                                   # one plane left: plane 1's tracks keep it
        [P(0, [[0, 0, 1, -1.4]]).role(pt0[0], 0)],                   # ... not all of them reassigned
    ]
    for i, recs in enumerate(bad):
        with pytest.raises(PvioB200Error, match=EINVAL):
            bw.set_planes(recs)
        assert _same(_snap(bw, [0, 1]), snap), i
    raw = b.lib.pvio_b200_batch_window_set_planes
    rec = _lib.CWindowPlanes()
    rec.slot, rec.n_planes = 0, -2
    assert raw(b.h, 1, C.byref(rec)) == -2                           # plane count -2
    cw = _constants(w)
    cw.n_planes = 2
    assert b.lib.pvio_b200_batch_window_reset(b.h, 0, C.byref(cw)) == -2
    assert _same(_snap(bw, [0, 1]), snap)
    # reassigning every track of plane 1 while dropping to one plane is accepted, and a reset clears planes and roles
    fix = P(0, [[0, 0, 1, -1.4]])
    for t in pt0:
        fix.role(t, SMALL_PLANE)
    bw.set_planes([fix])
    bw.reset(1, w)
    bw.solve([0], max_iterations=2)
    b.close()


def test_launch_count_and_slots_without_planes():
    """set_planes launches as many kernels for n = 1 as for n = 64; a slot that never received set_planes downloads and
    solves as on handles where no slot has planes: bit for bit when two such handles agree bit for bit, else within 2e-6
    (the inertial latency-path solve, DESIGN 5b)."""
    counts = {}
    for n in (1, 64):
        b = BundleAdjustor(max_windows=n, max_frames=9, max_landmarks=400, max_obs=3000)
        bw = BatchWindows(b)
        w, st = synth.make_cfg4(seed=978, N=6, M=120)[:2]
        ms = [_feed(bw, s, w, st, _tracks(w), planes=False) for s in range(n)]
        recs = []
        for s, m in enumerate(ms):
            p = Planes(s, np.concatenate([w.plane_normal, w.plane_distance[:, None]], axis=1))
            for i, t in m.items():
                if t["role"] != LANDMARK:
                    p.role(i, t["role"])
            recs.append(p)
        l0 = b.kernel_launches
        bw.set_planes(recs)
        counts[n] = b.kernel_launches - l0
        b.close()
    assert counts[1] == counts[64], counts
    run = Run(F=12, N=6, M=200, seed=979)
    w, st = synth.make_cfg4(seed=980, N=6, M=150)[:2]
    outs = []
    for planes in (True, False, False):                              # slot 0 with planes; twice without
        h = BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=400, max_obs=3000)
        bw = BatchWindows(h)
        _feed(bw, 0, w, st, _tracks(w), planes=planes)
        player = BatchPlayer(h, [run], slots=[1], bw=bw)
        d0 = player.bw.download([1], 400)[0]
        sm = player.bw.solve([1], max_iterations=6)[0]
        player.advance([0])
        sm2 = player.bw.solve([1], max_iterations=6)[0]
        outs.append((d0, sm, sm2, player.bw.download([1], 400)[0]))
        h.close()
    x, y, y2 = outs
    exact = _same([y[0], y[3]], [y2[0], y2[3]]) and all(y[1][k] == y2[1][k] and y[2][k] == y2[2][k] for k in SUMMARY_KEYS)
    print("handles without planes agree bit for bit:", exact)
    assert _same([x[0]], [y[0]])                                     # the fed window is the same before any solve
    _agree(x[3], y[3], exact)
    _summaries_agree(x[1], y[1], exact)
    _summaries_agree(x[2], y[2], exact)


def test_keyframe_cycle_with_planes_follows_the_repacked_sequences():
    """4 inertial sequences with 2 planes (N = 6, 8, 9, 6) take 12 keyframes each on different cycles, with a replaced
    non-keyframe between keyframes and set_planes after every keyframe: landmarks cast onto planes, plane tracks
    revalidated into landmarks with a new inverse depth, a plane under 20 tracks whose tracks turn -2 and back (Run.role).
    Each against its sequence re-packed through ba_solve + ba_marginalize with the same roles (Chain.window): equal
    iteration counts, anchors, landmark sets and plane-track sets, states and inverse depths within 2e-6 (the bar of
    test_keyframe_cycle_follows_the_repacked_sequences)."""
    runs = [Run(F=20, N=6, M=220, seed=710, planes=2), Run(F=22, N=8, M=260, seed=712, planes=2),
            Run(F=23, N=9, M=260, seed=714, planes=2), Run(F=20, N=6, M=220, seed=711, planes=2)]
    T = 480
    bat = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=T, max_obs=4000)
    one = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=T, max_obs=4000)
    player = BatchPlayer(bat, runs)
    refs = [Chain(r) for r in runs]
    done, worst, t, kinds = [0] * 4, 0.0, 0, set()
    while min(done) < 12:
        js = [j for j in range(4) if done[j] < 12 and (j % 2 == 0 or t % 2 == 0)]
        t += 1
        sms = player.bw.solve(js, max_iterations=6)
        ds = player.refresh(js, T)
        for j, d, sm in zip(js, ds, sms):
            ref, k = refs[j], player.k[j]
            wr, sr, lm = ref.window(k)
            out, summ = one.solve(wr, sr, max_iterations=6, postpass=False)
            S, e = one.marginalize_frame(wr, out, index=0)
            ref.store(k, out, lm)
            ref.set_prior(k, S, e, out)
            assert sm["iterations"] == summ["iterations"] and sm["accepted_steps"] == summ["accepted_steps"], (j, k)
            row = {int(i): r for r, i in enumerate(d["ids"])}
            role = {i: player.roles[j][l] for l, i in player.ids[j].items()}
            rows = [row[player.ids[j][l]] for l in lm]
            assert np.array_equal(d["anchor"][rows], wr.lm_anchor), (j, k)
            lms = [r for r, i in enumerate(d["ids"]) if role[int(i)] < 0 and d["n_obs"][r] >= 2]
            assert sorted(lms) == sorted(rows), (j, k)                  # the same landmarks take part
            assert {l for l, i in player.ids[j].items() if role[i] >= 0} == set(ref.pt_ids), (j, k)
            assert [role[player.ids[j][l]] for l in ref.pt_ids] == list(wr.pt_plane), (j, k)
            kinds |= {r for r in role.values()}
            refv = np.concatenate([out.q, out.p, out.v, out.bg, out.ba], axis=1)
            worst = max(worst, np.abs(d["frames"] - refv).max(), np.max(np.abs(d["inv_depth"][rows] - out.rho) / np.abs(out.rho)))
        player.advance(js)
        for j in js:
            done[j] += 1
    bat.close()
    one.close()
    print("resident plane keyframe cycle vs re-packed sequences: worst state / inverse-depth difference", worst)
    assert kinds == {-2, -1, 0, 1}
    assert worst < 2e-6


def test_observation_growth_keeps_other_slots_plane_tables():
    """An edit that adds observations to plane tracks of slot 1 pushes the plane-observation count past the handle's
    capacity (pt_frame / pt_z grow); slot 0's next solve equals the same solve on handles without that growth (bit for
    bit when two of those agree bit for bit, else within 2e-6)."""
    hs = [BundleAdjustor(max_windows=2, max_frames=9, max_landmarks=640, max_obs=3000) for _ in range(3)]
    bws = [BatchWindows(h) for h in hs]
    w, _ = _plane_slot(bws[0], 0)
    for bw in bws[1:]:
        _plane_slot(bw, 0)
    bwa = bws[0]
    bwa.reset(1, w)
    x = lambda f: np.concatenate([[0, 0, 0, 1], [0.1 * f, 0, 0], np.zeros(9)])
    bwa.edit([Edit(1).frame(x(0))])
    e = Edit(1)
    e.new = [(0, np.array([0.01 * (i % 40), 0.02 * (i // 40)]), 0.3) for i in range(250)]   # under 256 plane tracks
    ids = bwa.edit([e])[0]
    p = Planes(1, [[0.0, 0.0, 1.0, -1.4]])
    for i in ids:
        p.role(int(i), 0)
    bwa.set_planes([p])
    for f in range(1, 9):                                            # 250 x 9 = 2250 plane observations > 2048
        ob = Edit(1).frame(x(f), False, np.zeros(288))
        ob.obs = [(int(i), f, np.array([0.01, 0.02 * f])) for i in ids]
        bwa.edit([ob])
    sm = [bw.solve([0], max_iterations=6)[0] for bw in bws]
    ds = [bw.download([0], 640)[0] for bw in bws]
    exact = all(np.array_equal(ds[1][k], ds[2][k]) for k in ds[1]) and all(sm[1][k] == sm[2][k] for k in SUMMARY_KEYS)
    print("growth-free handles agree bit for bit:", exact)
    _agree(ds[0], ds[1], exact)
    _summaries_agree(sm[0], sm[1], exact)
    for h in hs:
        h.close()
