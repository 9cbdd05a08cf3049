"""The two oracles of the marginaliser (oracle/ba_oracle.py and the C restatement oracle/ba_oracle.c) agree at every
window size the library accepts up to the reference's default (N = 11) and beyond (N = 12), for every victim index:
the index-specific code of bundle_adjustor.cpp (IMU factors into and out of the victim :416-450, the complement blocks
around it :547-581) is restated in both, and the GPU tests of other indices rely on them.  CPU only."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import c_oracle
from synthetic import synth
from test_gpu_batch_marginalize import NOISE_ABS, _n_noise, _n_pos

U = 2.0 ** -53


def victim_flags(w, index):
    """lm_in_victim for victim `index`: the landmarks anchored in it or observed by it"""
    f = np.zeros(w.M, dtype=np.uint8)
    for l in range(w.M):
        seen = w.obs_frame[int(w.lm_obs_begin[l]):int(w.lm_obs_begin[l + 1])]
        f[l] = int(w.lm_anchor[l]) == index or index in seen
    return f


def window(N, prior, index, seed=None):
    w, st, _ = synth.make_cfg3(N=N, M=120, seed=100 + N if seed is None else seed, prior=prior)
    w.lm_in_victim = victim_flags(w, index)
    return w, st


def gauge_noise(H):
    """Absolute allowance on S^T S (and on H) of a window without a prior.  Its absolute position and yaw are unobservable,
    so the marginalised H is singular up to rounding: the Schur complement cancels terms of size |H|, and the eigenvalues
    of the null space are rounding noise of size n u |H| on both sides of the 1e-8 clamp (|H| reaches 1e10 once a middle
    frame is the victim: up to 2e-5 absolute between the two oracles).  Two marginalisers agree there only to that
    noise; NOISE_ABS (measured at index 0) stays the floor."""
    return max(NOISE_ABS, 64 * len(H) * U * np.max(np.abs(np.linalg.eigvalsh(0.5 * (H + H.T)))))


def cases(sizes, indices):
    """(N, prior, index).  The 1e15 gauge prior only at index 0: it lives on frame 0's pose, which every later index
    leaves in the window, and then b on that pose is 1e30 x the rounding of the prior residual (4.8e13 in the C oracle
    against ~1e6 in NumPy); PVIO never gets there, as the gauge prior exists only before the first marginalisation, which
    removes frame 0.  No prior-less window of two frames: the victim's block, held only by one IMU factor and the shared
    landmarks, is so nearly singular that the complement is not determined to the gauge noise (the oracles differ by
    9e-7 absolute, three times gauge_noise)."""
    return [(N, p, i) for N in sizes for p in ("synthetic", "none", "gauge") for i in indices(N)
            if (p != "gauge" or i == 0) and (p != "none" or N > 2)]


CASES = cases((2, 3, 6, 11, 12), range)


@pytest.mark.parametrize("N,prior,index", CASES)
def test_numpy_and_c_oracles_marginalise_alike(N, prior, index):
    w, st = window(N, prior, index)
    S0, e0, H0, b0 = bo.marginalize(w, st, index=index)
    S, e, H, b = c_oracle.marginalize(w, st, index)
    hs = np.maximum(np.sqrt(np.abs(np.diag(H0))), 1e-3)
    noise = gauge_noise(H0) if prior == "none" else NOISE_ABS
    # measured: H 2.5e-11 (synthetic) / 7e-13 (gauge) scaled; b 6e-13 relative; S^T S 1.6e-9 scaled (synthetic),
    # 0.75 of the noise bar (none); S^T e 6e-13 relative
    eH = np.max(np.abs(H - H0) / (1e-9 * np.outer(hs, hs) + (noise if prior == "none" else 0.0)))
    eb = np.max(np.abs(b - b0)) / np.max(np.abs(b0))
    L, L0 = S.T @ S, S0.T @ S0
    eL = np.max(np.abs(L - L0) / (1e-8 * np.outer(hs, hs) + (0.0 if prior == "synthetic" else noise)))
    ev = np.max(np.abs(S.T @ e - S0.T @ e0)) / np.max(np.abs(S0.T @ e0))
    print(f"N={N} {prior} index {index}: H {eH:.2e}, b {eb:.2e}, S^T S {eL:.2e} (of the bars), S^T e {ev:.2e}")
    assert eH < 1.0 and eb < 1e-11 and eL < 1.0 and ev < 1e-11, (eH, eb, eL, ev)
    assert abs(_n_pos(S) - _n_pos(S0)) <= _n_noise(H0), (_n_pos(S), _n_pos(S0), _n_noise(H0))


@pytest.mark.parametrize("N", [3, 6, 11, 12])
def test_complement_at_a_middle_index_is_symmetric(N):
    """The reference mirrors the upper-right block of Hk into the lower-left at 0 < index < N - 1 (:572-577); the device
    does not.  The complement is symmetric to rounding, so the mirror changes nothing beyond it."""
    index = N // 2
    w, st = window(N, "synthetic", index)
    _, _, H, _ = c_oracle.marginalize(w, st, index)
    hs = np.maximum(np.sqrt(np.abs(np.diag(H))), 1e-3)
    asym = np.max(np.abs(H - H.T) / np.outer(hs, hs))
    print(f"N={N} index {index}: max |Hk - Hk^T| (scaled) {asym:.2e}")
    assert asym < 1e-10
