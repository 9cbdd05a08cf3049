"""ba_solve on a window whose landmarks are not in anchor order: the solver packs them sorted by anchor, and every
per-landmark output (inverse depths, post-pass valid / quality) comes back in the caller's landmark order."""
import copy

import numpy as np
import pytest

from oracle import ba_oracle as bo
from pvio_b200.bundle_adjustor import BundleAdjustor
from synthetic import synth

pytestmark = pytest.mark.gpu


def _reordered(w, st, order):
    """the window with landmark order[i] as landmark i"""
    w, st = copy.deepcopy(w), copy.deepcopy(st)
    beg, of, oz = [0], [], []
    for l in order:
        b0, b1 = int(w.lm_obs_begin[l]), int(w.lm_obs_begin[l + 1])
        of += list(w.obs_frame[b0:b1])
        oz += list(w.obs_z[b0:b1])
        beg.append(len(of))
    w.lm_anchor, w.lm_z_ref, w.lm_in_victim = w.lm_anchor[order], w.lm_z_ref[order], w.lm_in_victim[order]
    w.lm_obs_begin = np.array(beg, dtype=np.int32)
    w.obs_frame, w.obs_z = np.array(of, dtype=np.int32), np.array(oz).reshape(-1, 2)
    st.rho = st.rho[order]
    w.validate()
    return w, st


def test_ba_solve_postpass_in_caller_landmark_order():
    """A window with landmarks anchored in 5 frames, behind-camera and far ones among them (synth.with_rejected_landmarks),
    in shuffled landmark order, against the same window stably sorted by anchor, which packs to the same device tables:
    its outputs are the sorted window's, landmark for landmark; valid and quality also equal the oracle's post-pass at
    the solved state (keypoints rounded to fp32, as the device keeps them)."""
    w, st, truth = synth.make_cfg2(N=7, M=90, staggered=True, seed=5)
    w, st = synth.with_rejected_landmarks(w, st, truth, seed=3)[:2]
    w = synth.f32_keypoints(w)
    wu, su = _reordered(w, st, np.random.default_rng(5).permutation(w.M))
    assert np.any(np.diff(wu.lm_anchor) < 0)
    rank = np.argsort(wu.lm_anchor, kind="stable")                  # sorted landmark i is shuffled landmark rank[i]
    ws, ss = _reordered(wu, su, rank)
    ba = BundleAdjustor(max_windows=1, max_frames=8, max_landmarks=256, max_obs=2000)
    out_u, sm_u = ba.solve(wu, su, max_iterations=6)
    out_s, sm_s = ba.solve(ws, ss, max_iterations=6)
    ba.close()
    assert sm_u["iterations"] == sm_s["iterations"] > 0
    assert np.array_equal(sm_u["valid"][rank], sm_s["valid"])
    assert (~sm_u["valid"]).any() and sm_u["valid"].any()
    assert np.allclose(sm_u["quality"][rank], sm_s["quality"], rtol=1e-9, atol=0.0)
    assert np.allclose(out_u.rho[rank], out_s.rho, rtol=1e-9, atol=0.0)
    ov, oq = bo.landmark_postpass(wu, out_u)
    assert np.array_equal(sm_u["valid"], ov)
    assert np.allclose(sm_u["quality"][ov], oq[ov], rtol=1e-6, atol=0.0)
    assert np.all(sm_u["quality"][~ov] == 0.0)
