"""The host model behind synthetic.sequence.BatchPlayer (no device): the windows it builds through the edits and drops of
pvio_b200_batch_window_* against Chain.window, and its non-keyframe replacement against erase_frame + put_frame."""
import numpy as np

from synthetic.sequence import BatchPlayer, Chain, ModelWindows, Run


def _tracks(model):
    """landmark -> [(window frame, keypoint)] of every live track"""
    return {t['l']: [(f, tuple(z)) for f, z in zip(t['frames'], t['zs'])] for t in model.tracks.values()}


def test_keyframe_only_model_matches_chain_windows():
    runs = [Run(F=16, N=6, M=200, seed=780), Run(F=17, N=8, M=220, seed=781)]
    player = BatchPlayer(None, runs, bw=ModelWindows())
    chains = [Chain(r) for r in runs]
    for k in range(8):
        for j, (r, c) in enumerate(zip(runs, chains)):
            view = player.model.m[j].view()
            w, _, lm = c.window(k)
            assert sorted(view) == sorted(lm), (j, k)
            for i, l in enumerate(lm):
                anchor, zref, of, oz = view[l]
                b0, b1 = w.lm_obs_begin[i], w.lm_obs_begin[i + 1]
                assert anchor == w.lm_anchor[i] and np.array_equal(zref, w.lm_z_ref[i]), (j, k, l)
                assert of == list(w.obs_frame[b0:b1]) and np.array_equal(np.array(oz).reshape(-1, 2), w.obs_z[b0:b1])
            assert player.model.m[j].frames == list(range(k, k + r.N))
        player.advance([0, 1], nonkey=False)


def _erase_frame(tr, last):
    """map->erase_frame(last) restated: the frame's keypoints leave their tracks, empty tracks go"""
    out = {l: [(f, z) for f, z in obs if f != last] for l, obs in tr.items()}
    return {l: obs for l, obs in out.items() if obs}


def _put_frame(tr, run, f_abs, f_win):
    """the frame's keypoints join their tracks (a new track for a landmark without one)"""
    out = {l: list(obs) for l, obs in tr.items()}
    fr_all = run.tracks
    for l, (fr, zs) in enumerate(fr_all):
        if f_abs in fr:
            out.setdefault(l, []).append((f_win, tuple(zs[fr.index(f_abs)])))
    return out


def test_nonkeyframe_replacement_is_erase_frame_then_put_frame():
    run = Run(F=14, N=6, M=200, seed=782)
    direct = BatchPlayer(None, [run], bw=ModelWindows())
    replaced = BatchPlayer(None, [run], bw=ModelWindows())
    for k in range(7):
        before = _tracks(replaced.model.m[0])
        assert before == _tracks(direct.model.m[0]), k
        replaced.advance([0], nonkey=True)
        direct.advance([0], nonkey=False)
        # restated: drop frame 0, put the non-keyframe, erase it, put the keyframe
        tr = {l: [(f - 1, z) for f, z in obs if f != 0] for l, obs in before.items()}
        tr = {l: obs for l, obs in tr.items() if obs}
        f_abs = k + run.N
        tr = _put_frame(tr, run, f_abs, run.N - 1)
        tr = _erase_frame(tr, run.N - 1)
        tr = _put_frame(tr, run, f_abs, run.N - 1)
        assert _tracks(replaced.model.m[0]) == tr, k
        assert replaced.model.m[0].frames == direct.model.m[0].frames
    # the non-keyframes' new tracks died with them: the same live landmarks, later ids
    assert replaced.model.m[0].next_id > direct.model.m[0].next_id
