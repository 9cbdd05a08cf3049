"""Resident batched windows (pvio_b200_batch_window_*): many sequences' sliding windows kept on the device, edited per
camera frame, solved, marginalised and re-laid out on the device."""
import dataclasses

import numpy as np
import pytest

from pvio_b200 import _lib
from pvio_b200.batch_window import BatchWindows, Edit
from pvio_b200.bundle_adjustor import BundleAdjustor, PvioB200Error
from pvio_b200.window import State
from synthetic import synth
from synthetic.sequence import BatchPlayer, Chain, Run

pytestmark = pytest.mark.gpu
EINVAL = f"error {_lib.EINVAL}"


def _feed_window(bw, slot, w, st):
    """A packed window fed frame by frame into a resident slot; returns landmark -> track id"""
    bw.reset(slot, w)
    ids = {}
    for f in range(w.N):
        e = Edit(slot).frame(np.concatenate([st.q[f], st.p[f], st.v[f], st.bg[f], st.ba[f]]), bool(w.frame_fixed[f]))
        e.landmarks = []
        for l in range(w.M):
            if int(w.lm_anchor[l]) == f:
                e.new.append((f, w.lm_z_ref[l], st.rho[l]))
                e.landmarks.append(l)
            for k in range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1]):
                if int(w.obs_frame[k]) == f:
                    e.obs.append((ids[l], f, w.obs_z[k]))
        for l, i in zip(e.landmarks, bw.edit([e])[0]):
            ids[l] = int(i)
    return ids


def _repack(w, d, ids):
    """the window of a download, in track-id order, with its states and inverse depths"""
    order = sorted(range(w.M), key=lambda l: ids[l])
    row = {int(i): r for r, i in enumerate(d["ids"])}
    wr = dataclasses.replace(w)
    anchors, zref, begins, of, oz = [], [], [0], [], []
    for l in order:
        anchors.append(w.lm_anchor[l]); zref.append(w.lm_z_ref[l])
        for k in range(w.lm_obs_begin[l], w.lm_obs_begin[l + 1]):
            of.append(w.obs_frame[k]); oz.append(w.obs_z[k])
        begins.append(len(of))
    wr.lm_anchor = np.array(anchors, dtype=np.int32); wr.lm_z_ref = np.array(zref).reshape(-1, 2)
    wr.lm_obs_begin = np.array(begins, dtype=np.int32); wr.obs_frame = np.array(of, dtype=np.int32)
    wr.obs_z = np.array(oz).reshape(-1, 2); wr.lm_in_victim = (wr.lm_anchor == 0).astype(np.uint8)
    fr = d["frames"]
    st = State(fr[:, 0:4].copy(), fr[:, 4:7].copy(), fr[:, 7:10].copy(), fr[:, 10:13].copy(), fr[:, 13:16].copy(),
               np.array([d["inv_depth"][row[ids[l]]] for l in order]))
    return wr, st, order


def test_visual_windows_solve_bit_identically_to_the_repacked_batch():
    """Visual-only windows played into resident slots [0, n) and solved there equal the same windows re-packed (states
    and inverse depths from the resident download) and solved by batch_solve over the same n, bit for bit."""
    n = 5
    wins = [synth.make_cfg2(N=6 + (i % 3), M=90 + 10 * i, seed=900 + i, staggered=True)[:2] for i in range(n)]
    res = BundleAdjustor(max_windows=n, max_frames=8, max_landmarks=160, max_obs=1200)
    pk = BundleAdjustor(max_windows=n, max_frames=8, max_landmarks=160, max_obs=1200)
    bw = BatchWindows(res)
    idss = [_feed_window(bw, i, w, st) for i, (w, st) in enumerate(wins)]
    before = bw.download(range(n), 160)
    packs = [_repack(w, d, ids) for (w, _), d, ids in zip(wins, before, idss)]
    sm = bw.solve(list(range(n)), max_iterations=8)
    after = bw.download(range(n), 160)
    for i, (wr, sr, _) in enumerate(packs):
        pk.batch_set(i, wr, sr)
    pk.batch_upload(n)
    pk.batch_solve(n, max_iterations=8)
    frames, rho, sm_ref = pk.batch_download_state(n, 8, 160)
    for i, ((w, _), (wr, sr, order)) in enumerate(zip(wins, packs)):
        assert np.array_equal(after[i]["frames"], frames[i, :w.N].reshape(w.N, 16)), i
        row = {int(t): r for r, t in enumerate(after[i]["ids"])}
        got = np.array([after[i]["inv_depth"][row[idss[i][l]]] for l in order])
        assert np.array_equal(got, rho[i, :w.M]), i
        for k in ("iterations", "accepted_steps", "termination", "initial_cost", "final_cost", "final_radius", "final_mu"):
            assert sm[i][k] == sm_ref[i][k], (i, k)
        assert sm[i]["iterations"] > 0
    res.close()
    pk.close()


def _check_cycle_step(player, one, ref, j, d, sm, worst):
    k = player.k[j]
    wr, sr, lm = ref.window(k)
    out, summ = one.solve(wr, sr, max_iterations=6, postpass=False)
    S, e = one.marginalize_frame(wr, out, index=0)
    ref.store(k, out, lm)
    ref.set_prior(k, S, e, out)
    assert sm["iterations"] == summ["iterations"] and sm["accepted_steps"] == summ["accepted_steps"], (j, k)
    row = {int(t): r for r, t in enumerate(d["ids"])}
    rows = [row[player.ids[j][l]] for l in lm]
    assert np.array_equal(d["anchor"][rows], wr.lm_anchor), (j, k)
    assert np.all(d["n_obs"][rows] >= 2)
    assert int(np.sum(d["n_obs"] >= 2)) == wr.M, (j, k)              # the same tracks take part
    refv = np.concatenate([out.q, out.p, out.v, out.bg, out.ba], axis=1)
    return max(worst, np.abs(d["frames"] - refv).max(), np.max(np.abs(d["inv_depth"][rows] - out.rho) / np.abs(out.rho)))


def test_keyframe_cycle_follows_the_repacked_sequences():
    """4 inertial sequences (N = 6, 8, 9, 6) take 12 keyframes each on different cycles (odd slots every other camera
    frame), with a replaced non-keyframe between keyframes; each against its sequence re-packed through ba_solve +
    ba_marginalize (the bars of test_batched_keyframe_cycle_follows_the_repacked_sequences)."""
    runs = [Run(F=20, N=6, M=220, seed=710), Run(F=22, N=8, M=260, seed=712), Run(F=23, N=9, M=260, seed=714),
            Run(F=20, N=6, M=220, seed=711)]
    bat = BundleAdjustor(max_windows=4, max_frames=9, max_landmarks=320, max_obs=3000)
    one = BundleAdjustor(max_windows=1, max_frames=9, max_landmarks=320, max_obs=3000)
    player = BatchPlayer(bat, runs)
    refs = [Chain(r) for r in runs]
    done, worst, t = [0] * 4, 0.0, 0
    while min(done) < 12:
        js = [j for j in range(4) if done[j] < 12 and (j % 2 == 0 or t % 2 == 0)]
        t += 1
        sms = player.bw.solve(js, max_iterations=6)
        ds = player.refresh(js, 320)
        for j, d, sm in zip(js, ds, sms):
            worst = _check_cycle_step(player, one, refs[j], j, d, sm, worst)
        player.advance(js)
        for j in js:
            done[j] += 1
    bat.close()
    one.close()
    print("resident batched keyframe cycle vs re-packed sequences: worst state / inverse-depth difference", worst)
    assert worst < 2e-6


def test_reanchored_inverse_depths_match_the_chain():
    """After a drop, a track anchored in the victim holds the inverse depth Chain._reanchor gives at the same states."""
    run = Run(F=12, N=6, M=220, seed=715)
    b = BundleAdjustor(max_windows=2, max_frames=6, max_landmarks=320, max_obs=3000)
    player = BatchPlayer(b, [run], slots=[1])
    player.bw.solve([1], max_iterations=4)
    d0 = player.refresh([0], 320)[0]
    chain = Chain(run)
    fr = d0["frames"]
    chain.q[:6], chain.p[:6] = fr[:, 0:4], fr[:, 4:7]
    row0 = {int(t): r for r, t in enumerate(d0["ids"])}
    moving = []
    for l, i in player.ids[0].items():
        chain.rho[l] = d0["inv_depth"][row0[i]]
        chain.anchor[l] = d0["anchor"][row0[i]]
        fl = [f for f in run.tracks[l][0] if f < 6]
        if d0["anchor"][row0[i]] == 0 and len(fl) >= 2:
            moving.append((l, i, fl[1]))
    assert len(moving) > 20
    player.bw.drop_victim([1])
    d1 = player.bw.download([1], 320)[0]
    row1 = {int(t): r for r, t in enumerate(d1["ids"])}
    worst = 0.0
    for l, i, nxt in moving:
        chain._reanchor(l, nxt)
        got = d1["inv_depth"][row1[i]]
        worst = max(worst, abs(got - chain.rho[l]) / abs(chain.rho[l]))
        assert d1["anchor"][row1[i]] == nxt - 1
    assert worst < 1e-12, worst
    b.close()


def test_postpass_flags_match_ba_solve():
    """A window with far and behind-camera landmarks (synth.hard_window "rejected"): valid equals ba_solve's flags for
    the re-packed window bit for bit, quality agrees with ba_solve's and with bo.landmark_postpass at the downloaded
    final state, and tracks that did not take part in the solve read 0 / 0; a solve without post-pass clears them."""
    from oracle import ba_oracle as bo
    w, st = synth.hard_window("rejected", inertial=False, N=6, M=100, seed=890)[:2]
    res = BundleAdjustor(max_windows=2, max_frames=8, max_landmarks=256, max_obs=2000)
    one = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=256, max_obs=2000)
    bw = BatchWindows(res)
    ids = _feed_window(bw, 1, w, st)
    e = Edit(1)                                                      # a one-observation track: takes no part
    e.new.append((w.N - 1, np.array([0.01, 0.02]), 0.5))
    lonely = int(bw.edit([e])[0][0])
    d0 = bw.download([1], 256)[0]
    wr, sr, order = _repack(w, d0, ids)
    bw.solve([1], max_iterations=6)
    d = bw.download([1], 256)[0]
    _, _, valid, quality = _solve_with_flags(one, wr, sr)
    row = {int(t): r for r, t in enumerate(d["ids"])}
    rows = [row[ids[l]] for l in order]
    assert np.array_equal(d["valid"][rows], valid)
    assert (~valid.astype(bool)).sum() >= 3 and valid.any()
    assert np.allclose(d["quality"][rows], quality, rtol=1e-9, atol=0.0)
    _, fin, _ = _repack(w, d, ids)
    ov, oq = bo.landmark_postpass(wr, fin)
    assert np.array_equal(d["valid"][rows].astype(bool), ov)
    assert np.allclose(d["quality"][rows][ov], oq[ov], rtol=1e-6, atol=0.0)
    assert np.all(d["quality"][rows][~ov] == 0.0)
    assert d["valid"][row[lonely]] == 0 and d["quality"][row[lonely]] == 0.0
    bw.solve([1], max_iterations=2, postpass=False)
    d = bw.download([1], 256)[0]
    assert not d["valid"].any() and not d["quality"].any()
    res.close()
    one.close()


def _solve_with_flags(one, w, st):
    import ctypes as C
    from pvio_b200 import _lib
    pa = _lib.PackedArgs(w, st)
    opt = _lib.COptions(6, 1e6, 1, 1, 0.0)
    sm = _lib.CSummary()
    valid = np.zeros(max(w.M, 1), dtype=np.uint8)
    quality = np.zeros(max(w.M, 1))
    one._ck(one.lib.pvio_b200_ba_solve(one.h, C.byref(pa.cw), C.byref(pa.cs), C.byref(opt), C.byref(sm),
                                       _lib.ptr(valid), _lib.ptr(quality)))
    return None, sm, valid[:w.M], quality[:w.M]


def _snap(bw, slots, stride=320):
    return [{k: v.copy() for k, v in d.items()} for d in bw.download(slots, stride)]


def _same(a, b):
    return all(all(np.array_equal(x[k], y[k]) for k in x) for x, y in zip(a, b))


def test_isolation_and_rejections_change_nothing():
    runs = [Run(F=14, N=6, M=200, seed=720 + i) for i in range(3)]
    b = BundleAdjustor(max_windows=3, max_frames=6, max_landmarks=320, max_obs=3000)
    player = BatchPlayer(b, runs)
    bw = player.bw
    bw.solve([0, 1, 2], max_iterations=3)
    snap = _snap(bw, [0, 1, 2])
    bw.solve([1], max_iterations=4)                                  # slots 0 and 2 are not named: untouched
    s1 = _snap(bw, [0, 1, 2])
    assert _same([s1[0], s1[2]], [snap[0], snap[2]]) and not _same([s1[1]], [snap[1]])
    bw.drop_victim([2])
    s2 = _snap(bw, [0, 1, 2])
    assert _same(s2[:2], s1[:2]) and not _same([s2[2]], [s1[2]])
    snap = s2
    some = int(snap[0]["ids"][0])
    bad = [
        lambda: bw.solve([0, 0]),                                    # a slot named twice
        lambda: bw.solve([3]),                                       # out of range
        lambda: bw.edit([Edit(0), Edit(0)]),
        lambda: bw.edit([_with(Edit(1), remove=[10 ** 6])]),         # unknown track
        lambda: bw.edit([Edit(0), _with(Edit(1), obs=[(some, 0, np.zeros(2))])]),   # 'some' is slot 0's: unknown / order
        lambda: bw.edit([_with(Edit(2), obs=[(int(snap[2]["ids"][-1]), 0, np.zeros(2))])]),   # out of frame order
        lambda: bw.edit([Edit(0).frame(np.zeros(16), False, np.zeros(288))]),        # a 7th frame in a 6-frame window
        lambda: bw.edit([_with(Edit(1), new=[(0, np.zeros(2), 1.0)] * 400)]),      # more live tracks than max_landmarks
        lambda: bw.drop_victim([0, 2, 0]),
        lambda: b.batch_solve(1),                                    # existing calls refuse resident slots
        lambda: b.batch_upload(3),
        lambda: b.batch_marginalize(2),
    ]
    for i, call in enumerate(bad):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
        assert _same(_snap(bw, [0, 1, 2]), snap), i
    # a single-window call packs into slot 0: slot 0 stops being resident, the others stay
    w, st, _ = synth.make_cfg2(N=5, M=40, seed=7)
    b.gn_step(w, st)
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.download([0], 320)
    assert _same(_snap(bw, [1, 2]), snap[1:])
    bw.solve([1, 2], max_iterations=2)
    b.close()


def _with(e, remove=(), obs=(), new=()):
    e.remove, e.obs, e.new = list(remove), list(obs), list(new)
    return e


def test_long_sequence_reuses_dead_track_storage():
    """One slot creates many more tracks than max_landmarks over 60 keyframes while its live tracks stay under it."""
    b = BundleAdjustor(max_windows=1, max_frames=5, max_landmarks=64, max_obs=400)
    w, st, _ = synth.make_cfg2(N=5, M=10, seed=940)
    bw = BatchWindows(b)
    w = dataclasses.replace(w, use_inertial=False)
    bw.reset(0, w)
    rng = np.random.default_rng(3)
    for f in range(5):
        bw.edit([Edit(0).frame(np.concatenate([[0, 0, 0, 1], [0.1 * f, 0, 0], np.zeros(9)]), f < 2)])
    live, last = [], -1
    for k in range(60):                              # per keyframe: 20 tracks start, the 20 oldest are pruned
        e = Edit(0)
        e.new = [(4, rng.normal(size=2) * 0.1, 0.3) for _ in range(20)]
        if len(live) >= 40:
            e.remove, live = live[:20], live[20:]
        ids = bw.edit([e])[0]
        assert np.all(ids > last)
        last = int(ids.max())
        live += [int(i) for i in ids]
    d = bw.download([0], 64)[0]
    assert last + 1 == 1200 and len(d["ids"]) == len(live) <= 64
    assert np.array_equal(d["ids"], np.array(sorted(live)))
    b.close()


def test_long_inertial_sequence_reuses_storage_through_drops():
    """60 keyframes of one inertial sequence (solve, drop, replaced non-keyframe, new frame): it creates far more tracks
    than max_landmarks, its live tracks stay under it, ids keep increasing."""
    run = Run(F=67, N=6, M=1000, seed=760)
    b = BundleAdjustor(max_windows=1, max_frames=6, max_landmarks=480, max_obs=4000)   # at most 411 live (host model)
    player = BatchPlayer(b, [run])
    last = -1
    for k in range(60):
        player.bw.solve([0], max_iterations=2)
        d = player.refresh([0], 480)[0]
        assert np.all(np.diff(d["ids"]) > 0) and len(d["ids"]) <= 480
        player.advance([0])
        last = max(last, max(player.ids[0].values()))
    assert last >= 3 * 480
    b.close()


def test_more_rejections_change_nothing():
    """max_obs, more than 96 landmark chunks, a drop of a visual-only window, a drop with 15 (N - 1) > 165, and any call
    on a slot whose residency a packing call ended: rejected, nothing changes."""
    b = BundleAdjustor(max_windows=3, max_frames=16, max_landmarks=3600, max_obs=3500)
    bw = BatchWindows(b)
    wv, _, _ = synth.make_cfg2(N=5, M=10, seed=950)
    wi, _, _ = synth.make_cfg3(N=6, M=20, seed=951)
    bw.reset(0, wv)
    bw.reset(1, wi)
    bw.reset(2, wv)
    x = lambda f: np.concatenate([[0, 0, 0, 1], [0.1 * f, 0, 0], np.zeros(9)])
    for f in range(16):
        bw.edit([Edit(0).frame(x(f), f < 2), Edit(1).frame(x(f), False, np.zeros(288) if f else None), Edit(2).frame(x(f), False)])
    e = Edit(0)                                                      # 15 anchors x 7 chunks of 32 landmarks
    e.new = [(a, np.array([0.01 * (i % 50), 0.02]), 0.2) for a in range(15) for i in range(224)]
    ids = bw.edit([e])[0]
    ok = Edit(0)                                                     # 15 x 6 = 90 chunks of 2-observation landmarks
    ok.obs = [(int(ids[a * 224 + i]), a + 1, np.zeros(2)) for a in range(15) for i in range(192)]
    bw.edit([ok])
    snap = _snap(bw, [0, 1, 2], 3600)
    more = Edit(0)                                                   # 105 chunks
    more.obs = [(int(ids[a * 224 + i]), a + 1, np.zeros(2)) for a in range(15) for i in range(192, 224)]
    with pytest.raises(PvioB200Error, match=EINVAL):
        bw.edit([more])
    assert _same(_snap(bw, [0, 1, 2], 3600), snap)
    t2 = bw.edit([_with(Edit(2), new=[(0, np.zeros(2), 1.0)] * 1800)])[0]
    snap = _snap(bw, [0, 1, 2], 3600)
    obs = Edit(2)                                                    # 1800 observations, then 3600 > max_obs
    obs.obs = [(int(t), 1, np.zeros(2)) for t in t2]
    bw.edit([obs])
    snap = _snap(bw, [0, 1, 2], 3600)
    obs2 = Edit(2)
    obs2.obs = [(int(t), 2, np.zeros(2)) for t in t2]
    for call in (lambda: bw.edit([obs2]),                            # more than max_obs observations
                 lambda: bw.drop_victim([2]),                        # a visual-only window
                 lambda: bw.drop_victim([1]),                        # 16 frames: 15 (N - 1) = 225 > 165
                 lambda: bw.drop_victim([0, 1])):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
        assert _same(_snap(bw, [0, 1, 2], 3600), snap)
    b.batch_set(2, *synth.make_cfg2(N=5, M=40, seed=952)[:2])         # set_window ends slot 2's residency
    for call in (lambda: bw.download([2], 320), lambda: bw.edit([Edit(2)]), lambda: bw.solve([2])):
        with pytest.raises(PvioB200Error, match=EINVAL):
            call()
    assert _same(_snap(bw, [0, 1], 3600), snap[:2])
    b.close()


def test_downloads_of_the_packed_path_refuse_resident_slots():
    """A slot once packed with unsorted anchors, then made resident with more landmarks than that pack: the packed path's
    downloads refuse it (their landmark permutation belongs to the old pack) and the resident download serves it."""
    b = BundleAdjustor(max_windows=2, max_frames=8, max_landmarks=160, max_obs=1200)
    w, st, _ = synth.make_cfg2(N=6, M=30, seed=953, staggered=True)
    perm = np.arange(w.M)[::-1].copy()
    ws = dataclasses.replace(w, lm_anchor=w.lm_anchor[perm])
    begins = np.concatenate([[0], np.cumsum(np.diff(w.lm_obs_begin)[perm])]).astype(np.int32)
    of = np.concatenate([w.obs_frame[w.lm_obs_begin[l]:w.lm_obs_begin[l + 1]] for l in perm])
    oz = np.concatenate([w.obs_z[w.lm_obs_begin[l]:w.lm_obs_begin[l + 1]] for l in perm])
    ws = dataclasses.replace(ws, lm_z_ref=w.lm_z_ref[perm], lm_obs_begin=begins, obs_frame=of, obs_z=oz,
                             lm_in_victim=np.asarray(w.lm_in_victim)[perm] if len(w.lm_in_victim) == w.M else w.lm_in_victim)
    b.batch_set(0, ws, dataclasses.replace(st, rho=st.rho[perm]))
    b.batch_upload(1)
    b.batch_solve(1, max_iterations=2)
    big, bst, _ = synth.make_cfg2(N=6, M=120, seed=954, staggered=True)
    bw = BatchWindows(b)
    _feed_window(bw, 0, big, bst)
    with pytest.raises(PvioB200Error, match=EINVAL):
        b.batch_download_state(1, 8, 160)
    with pytest.raises(PvioB200Error, match=EINVAL):
        b.batch_download(1, 15 * 8 + 160)
    bw.solve([0], max_iterations=3)
    d = bw.download([0], 160)[0]
    assert len(d["ids"]) == 120 and np.all(np.isfinite(d["inv_depth"]))
    b.close()


def test_launch_count_does_not_depend_on_n():
    counts = {}
    for n in (2, 64):
        run = Run(F=10, N=6, M=120, seed=750)
        b = BundleAdjustor(max_windows=n, max_frames=6, max_landmarks=160, max_obs=1200)
        player = BatchPlayer(b, [run] * n)
        js = list(range(n))
        player.refresh(js, 160)
        c = []
        l0 = b.kernel_launches
        player.bw.solve(js, max_iterations=3)
        c.append(b.kernel_launches - l0)
        l0 = b.kernel_launches
        player.bw.drop_victim(js)
        c.append(b.kernel_launches - l0)
        player.refresh(js, 160)
        l0 = b.kernel_launches
        player.bw.edit([player.frame_edit(j, 6, 5) for j in js])
        c.append(b.kernel_launches - l0)
        counts[n] = c
        b.close()
    assert counts[2] == counts[64], counts
