"""The host model behind synthetic.sequence.BatchPlayer with plane roles (no device): played through a plane run with role
switches (a landmark cast onto a plane, a plane track revalidated into a landmark, a plane under 20 tracks whose tracks
turn -2 and back), non-keyframe replacement and drops, it gives at every keyframe the window Chain.window gathers."""
import numpy as np

from synthetic.sequence import BatchPlayer, Chain, ModelWindows, Run


def test_plane_model_matches_chain_windows():
    runs = [Run(F=18, N=6, M=200, seed=783, planes=2), Run(F=19, N=8, M=220, seed=784, planes=2)]
    player = BatchPlayer(None, runs, bw=ModelWindows())
    chains = [Chain(r) for r in runs]
    switched, on_plane = [0, 0], [set(), set()]
    for k in range(10):
        for j, c in enumerate(chains):
            m = player.model.m[j]
            w, _, lm = c.window(k)
            view, victims = m.view(), m.victims()
            assert sorted(view) == sorted(lm), (j, k)
            for i, l in enumerate(lm):
                anchor, zref, of, oz = view[l]
                b0, b1 = w.lm_obs_begin[i], w.lm_obs_begin[i + 1]
                assert anchor == w.lm_anchor[i] and np.array_equal(zref, w.lm_z_ref[i]), (j, k, l)
                assert of == list(w.obs_frame[b0:b1]) and np.array_equal(np.array(oz).reshape(-1, 2), w.obs_z[b0:b1])
                assert victims[l] == w.lm_in_victim[i], (j, k, l)
            pv = m.plane_view()
            assert [t[0] for t in pv] == c.pt_ids, (j, k)                 # the same plane tracks, in id order
            assert [t[1] for t in pv] == list(w.pt_plane), (j, k)
            for t, (l, p, fr, zs) in enumerate(pv):
                b0, b1 = w.pt_obs_begin[t], w.pt_obs_begin[t + 1]
                assert fr == list(w.pt_obs_frame[b0:b1]) and np.array_equal(np.array(zs), w.pt_obs_z[b0:b1]), (j, k, l)
            roles = [t['role'] for t in m.tracks.values()]
            assert w.n_ptracks > 20 and (-2 in roles) == (4 <= k < 8), (j, k)
            if 4 <= k < 8:                                             # plane 1 under 20 tracks: its tracks are -2
                assert w.lm_in_victim.sum() < (w.lm_anchor == 0).sum(), (j, k)
            r = runs[j]
            if k == 3:
                switched[0] += sum(r.plane_of[t['l']] < 0 and t['role'] >= 0 for t in m.tracks.values())
            if k == 4:
                on_plane[j] = {t['l'] for t in m.tracks.values() if t['role'] >= 0}
            if k == 5:                                                 # revalidated: a landmark with its new inverse depth
                reval = [t['l'] for t in m.tracks.values() if t['l'] in on_plane[j] and t['role'] == -1]
                switched[1] += len(reval)
                assert all(c.rho[l] == r.revalidated_rho(l) for l in reval if l in lm), (j, k)
        player.advance([0, 1], nonkey=True)
    # every switch took place: landmarks cast onto planes, plane tracks revalidated into landmarks
    assert switched[0] and switched[1]
