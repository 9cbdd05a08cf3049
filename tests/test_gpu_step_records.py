"""The batched GN step keeps the linearise sweep's per-landmark sums (H_ll = sum j.j, g_l = sum j.r) in shared memory
when one CTA owns a window, and reads the frame-major table as 8-byte keypoints plus 16-bit landmark indices.  Checked
here: bit-identical repeats at bench's batch sizes, the shared-memory sums against the per-block records of the
several-CTAs-per-window path, a landmark count whose shared layout does not fit (the records path again), and the
victim-only marginaliser sweep."""
import ctypes as C

import numpy as np
import pytest

from oracle import ba_oracle as bo
from synthetic import synth
from pvio_b200 import _lib as L
from pvio_b200.bundle_adjustor import BundleAdjustor

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _het_kinds():
    """bench.py's heterogeneous batch: 5 window kinds (sizes, anchors, visibility and fixed sets differ)"""
    kinds = [synth.make_cfg2(N=10, M=500, seed=41)[:2], synth.make_cfg2(N=10, M=420, staggered=True, seed=42)[:2],
             synth.make_cfg2(N=8, M=300, seed=43)[:2], synth.make_cfg2(N=9, M=350, staggered=True, seed=44)[:2],
             synth.make_cfg2(N=10, M=500, seed=45)[:2]]
    kinds[2][0].frame_fixed[:] = 0
    kinds[2][0].frame_fixed[0] = 1
    kinds[2][0].frame_fixed[5] = 1
    return kinds


@pytest.fixture(scope="module")
def big():
    b = BundleAdjustor(max_windows=4096, max_frames=10, max_landmarks=512, max_obs=4608)
    yield b
    b.close()


def _two_steps(b, W, stride):
    out = []
    for _ in range(2):
        b.batch_gn_step(W, 1e-8, apply=False)
        out.append(b.batch_download(W, stride))
    return out


def test_repeated_steps_are_bit_identical(big):
    """Two GN steps of 4096 cfg2 windows, and of the heterogeneous 5-kind batch, give the same dx and costs bit for bit."""
    W, stride = 4096, 15 * 10 + 512
    w, st, _ = synth.make_cfg2()
    big.batch_set(0, w, st)
    big.batch_replicate(W)
    big.batch_upload(W)
    (dx0, c0), (dx1, c1) = _two_steps(big, W, stride)
    assert np.array_equal(dx0, dx1) and np.array_equal(c0, c1)
    ref = bo.gn_step(w, st, schur=True)["dx"]
    n = 15 * w.N + w.M
    assert _rel(dx0[W - 1, :n], ref) < 1e-5

    kinds = _het_kinds()
    pas = [L.PackedArgs(w_, s_) for w_, s_ in kinds]
    for i in range(W):
        big.lib.pvio_b200_batch_set_window(big.h, i, C.byref(pas[i % 5].cw), C.byref(pas[i % 5].cs))
    big.batch_upload(W)
    (dx0, c0), (dx1, c1) = _two_steps(big, W, stride)
    assert np.array_equal(dx0, dx1) and np.array_equal(c0, c1)


def test_shared_sums_match_the_record_path(big):
    """The same windows through the batched path (one CTA per window, sums in shared memory) and one at a time through the
    latency path (16 CTAs per window, per-block records summed by lm_finish_kernel).  The two paths cut the table rows
    into different pieces, so the fp32 direct-block sums and the Cauchy log-sums round differently: dx differs by up to
    2.3e-6 relative on these windows (an H100, also before the shared-memory sums).  Both stay within the oracle bars
    of test_gpu_ba (1e-5 on dx, 2e-6 on the cost)."""
    kinds = _het_kinds()
    W, stride = 80, 15 * 10 + 512          # 80 windows: more than half the SM count, the batched path
    for i in range(W):
        big.batch_set(i, *kinds[i % 5])
    big.batch_upload(W)
    big.batch_gn_step(W, 1e-8, apply=False)
    dx_b, c_b = big.batch_download(W, stride)
    for j, (w, st) in enumerate(kinds):
        big.batch_set(0, w, st)
        big.batch_upload(1)
        big.batch_gn_step(1, 1e-8, apply=False)
        dx_1, c_1 = big.batch_download(1, stride)
        n = 15 * w.N + w.M
        assert _rel(dx_b[j, :n], dx_1[0, :n]) < 1e-5, j
        assert abs(c_b[j, 0] - c_1[0, 0]) <= 2e-6 * c_1[0, 0], j
        ref = bo.gn_step(w, st, schur=True)["dx"]
        assert _rel(dx_b[j, :n], ref) < 1e-5, j


@pytest.mark.parametrize("N,M", [(6, 1200), (4, 3000)])
def test_large_landmark_count_falls_back_to_records(N, M):
    """M = 1200: the shared sums would cost a resident CTA per SM; M = 3000: they would not fit at all.  Both take the
    per-block records and still match the oracle in a batch that fills the GPU."""
    w, st, _ = synth.make_cfg2(N=N, M=M, seed=77)
    W = 80
    b = BundleAdjustor(max_windows=W, max_frames=N, max_landmarks=M, max_obs=(N - 1) * M + 64 * N)
    try:
        b.batch_set(0, w, st)
        b.batch_replicate(W)
        b.batch_upload(W)
        b.batch_gn_step(W, 1e-8, apply=False)
        dx, _ = b.batch_download(W, 15 * N + M)
    finally:
        b.close()
    ref = bo.gn_step(w, st, schur=True)["dx"]
    assert _rel(dx[0], ref) < 1e-5
    assert _rel(dx[W - 1], ref) < 1e-5


def test_victim_only_sweep_matches_single_window():
    """The batched marginaliser (one CTA per window: the shared sums of the victim-only fp64 sweep) against the
    single-window marginaliser (the records path) on the same windows."""
    W = 80
    kinds = [synth.make_cfg3(N=6, M=120, seed=660 + i, prior=p)[:2] for i, p in enumerate(('synthetic', 'gauge', 'none'))]
    b = BundleAdjustor(max_windows=W, max_frames=6, max_landmarks=160, max_obs=1200)
    try:
        singles = [b.marginalize_frame(w, st, 0, want_info=True) for w, st in kinds]
        for i in range(W):
            b.batch_set(i, *kinds[i % 3])
        b.batch_upload(W)
        out = b.batch_marginalize(W, want=True)
    finally:
        b.close()
    for i in range(3):
        S, e = out[i]
        S1, e1, H1, _ = singles[i]
        L1, Lb = S1.T @ S1, S.T @ S
        hs = np.maximum(np.sqrt(np.abs(np.diag(H1))), 1e-3)
        assert np.max(np.abs(Lb - L1) / (1e-9 * np.outer(hs, hs) + 1e-7)) < 1.0, i
        assert np.max(np.abs(S.T @ e - S1.T @ e1)) <= 1e-9 * np.max(np.abs(S1.T @ e1)), i
