"""The whole marginaliser on the device (pvio_b200_ba_marginalize, pvio_b200_batch_marginalize) against bo.marginalize at
the window sizes and victim indices it accepts: N = 2 ... 12 (dk = 15 ... 165; N = 11 is the reference's default
sliding window, Config::sliding_window_size() = 10, marginalised at frame_num() = 11), victims at both ends and in the
middle (the IMU factors into and out of the victim and the complement blocks around it are index-specific code), and
the first size it rejects.  The bars are those of test_gpu_ba.py::test_marginalize_matches_oracle and
test_gpu_batch_marginalize.py; windows without a prior have a gauge null space, see gauge_noise."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from pvio_b200.bundle_adjustor import BundleAdjustor
from test_gpu_batch_marginalize import NOISE_ABS, _check_prior
from test_marginalize_oracle_shapes import cases, gauge_noise, window

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=1, max_frames=12, max_landmarks=128, max_obs=2000)
    yield b
    b.close()


def _noise(prior, H0):
    return gauge_noise(H0) if prior == "none" else NOISE_ABS


def _check_oracle(S, e, H, b, w, st, index, prior):
    """the bars of test_marginalize_matches_oracle: H scaled 1e-6, b 1e-6, the prior through _check_prior"""
    S0, e0, H0, b0 = bo.marginalize(w, st, index=index)
    hs = np.maximum(np.sqrt(np.abs(np.diag(H0))), 1e-3)
    noise = _noise(prior, H0)
    eH = np.max(np.abs(H - H0) / (1e-6 * np.outer(hs, hs) + (noise if prior == "none" else 0.0)))
    eb = np.max(np.abs(b - b0)) / np.max(np.abs(b0))
    assert eH < 1.0 and eb < 1e-6, (eH, eb)
    eL, ev = _check_prior(S, e, S0, e0, H0, 1e-6, noise)
    return eH, eb / 1e-6, eL, ev / 1e-6


SINGLE = cases((2, 3, 4, 7, 10, 11, 12), lambda N: sorted({0, 1, N // 2, N - 2, N - 1}))


@pytest.mark.parametrize("N,prior,index", SINGLE)
def test_marginalize_every_size_and_index_matches_oracle(ba, N, prior, index):
    w, st = window(N, prior, index)
    S, e, H, b = ba.marginalize_frame(w, st, index=index, want_info=True)
    r = _check_oracle(S, e, H, b, w, st, index, prior)
    print(f"N={N} {prior} index {index}: error / bar H {r[0]:.2e}, b {r[1]:.2e}, S^T S {r[2]:.2e}, S^T e {r[3]:.2e}")


def _batch_kinds(sizes):
    return [(N, p) for N in sizes for p in ("synthetic", "none", "gauge") if p != "none" or N > 2]


def test_batch_of_mixed_sizes_matches_single_windows_and_oracle():
    """80 windows of N in {2, 3, 7, 11, 12} in one pass of the dense kernels, at least half as many windows as an H100
    has SMs (the one-CTA-per-window vision sweep), every window of the eigen-solver's launch given the shared memory of
    dk = 165.  Each equals its own single-window prior and the oracle, and the windows below N = 12 keep their priors in
    a batch whose N = 12 windows are replaced by N = 11 ones.  That comparison is not bitwise: the vision sweep takes its
    launch shape from the batch's largest N (shared-memory layout of the direct blocks, whether the per-landmark sums
    stay in shared memory), so its sums round differently; on an H100 S differed in the last bits.  The eigen-solver's
    own independence of its launch is bitwise (test_gpu_marg_eig.py)."""
    W = 80
    b = BundleAdjustor(max_windows=W, max_frames=12, max_landmarks=128, max_obs=2000)
    kinds = _batch_kinds((2, 3, 7, 11, 12))
    wins = {k: window(k[0], k[1], 0, seed=300 + i) for i, k in enumerate(kinds)}
    singles = {k: b.marginalize_frame(*wins[k], 0, want_info=True) for k in kinds}

    def run(kind_of):
        for i in range(W):
            b.batch_set(i, *wins[kind_of(i)])
        b.batch_upload(W)
        return b.batch_marginalize(W, want=True)

    first = run(lambda i: kinds[i % len(kinds)])
    worst = [0.0] * 6
    for i in range(W):
        k = kinds[i % len(kinds)]
        (S, e), (S1, e1, H1, b1) = first[i], singles[k]
        assert S.shape == (15 * (k[0] - 1),) * 2
        worst[:2] = np.maximum(worst[:2], _check_prior(S, e, S1, e1, H1, 1e-9, _noise(k[1], H1)))
        worst[2:] = np.maximum(worst[2:], _check_oracle(S, e, H1, b1, *wins[k], 0, k[1]))
    print("batch of mixed sizes: worst vs single window S^T S %.2e, S^T e %.2e; vs oracle H %.2e, b %.2e, S^T S %.2e, "
          "S^T e %.2e (of the bars)" % tuple(worst))
    small = [k for k in kinds if k[0] != 12]
    second = run(lambda i: kinds[i % len(kinds)] if kinds[i % len(kinds)][0] != 12 else small[i % len(small)])
    for i in range(W):
        k = kinds[i % len(kinds)]
        if k[0] != 12:
            _check_prior(*second[i], *first[i], singles[k][2], 1e-9, _noise(k[1], singles[k][2]))
    b.close()


@pytest.mark.skipif(not __import__("torch").cuda.is_available() or __import__("torch").cuda.device_count() < 2,
                    reason="needs two CUDA devices")
def test_marginalize_on_a_second_device():
    """The eigen-solver's shared-memory opt-in is made for each handle's device: the same cfg3 N = 9 window marginalised
    through a handle on device 0 and then through one on device 1 gives the same prior."""
    from synthetic import synth
    w, st, _ = synth.make_cfg3(N=9, M=120, seed=640)
    out = []
    for dev in (0, 1):
        h = BundleAdjustor(device=dev, max_windows=1, max_frames=9, max_landmarks=128, max_obs=2000)
        out.append(h.marginalize_frame(w, st, 0, want_info=True))
        h.close()
    (S0, e0, _, _), (S1, e1, H1, _) = out
    _check_prior(S1, e1, S0, e0, H1, 1e-9)
