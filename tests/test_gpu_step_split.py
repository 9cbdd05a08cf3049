"""batch_gn_step may run the batch as contiguous sub-batches on two streams (api.cu: run_gn_step_split).  Every window
runs the same kernels with the same arguments either way, so dx and the costs must be bit-identical with the split
forced off and forced on: at bench.py's 4096 cfg2 windows, on its five-kind heterogeneous batch, and at a window
count that no sub-batch count divides.  The stage times of last_kernel_ms stay defined for the whole batch."""
import ctypes as C

import numpy as np
import pytest

from synthetic import synth
from pvio_b200 import _lib as L
from pvio_b200.bundle_adjustor import BundleAdjustor

pytestmark = pytest.mark.gpu

W = 4096


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
    b = BundleAdjustor(max_windows=W, max_frames=10, max_landmarks=512, max_obs=4608)
    yield b
    b.close()


def _cfg2(ba, n):
    w, st, _ = synth.make_cfg2()
    ba.batch_set(0, w, st)
    ba.batch_replicate(n)
    ba.batch_upload(n)
    return 15 * w.N + w.M


def _hetero(ba, n):
    pas = [L.PackedArgs(w, s) for w, s in _het_kinds()]
    for i in range(n):
        p = pas[i % len(pas)]
        ba.lib.pvio_b200_batch_set_window(ba.h, i, C.byref(p.cw), C.byref(p.cs))
    ba.batch_upload(n)
    return 15 * 10 + 500


def _step(ba, n, stride, parts):
    assert ba.lib.pvio_b200_internal_set_step_split(ba.h, parts) == 0
    l0 = ba.kernel_launches
    ba.batch_gn_step(n, 1e-8, apply=False)
    launches = ba.kernel_launches - l0
    dx, costs = ba.batch_download(n, stride)
    assert ba.lib.pvio_b200_internal_set_step_split(ba.h, 0) == 0
    return dx, costs, launches


def _same(a, b):
    assert a[0].shape == b[0].shape and a[1].shape == b[1].shape
    assert np.array_equal(a[0], b[0]), f"dx differs in {np.count_nonzero(a[0] != b[0])} entries"
    assert np.array_equal(a[1], b[1]), f"costs differ in {np.count_nonzero(a[1] != b[1])} entries"


def test_split_bit_identical_cfg2(big):
    stride = _cfg2(big, W)
    ref = _step(big, W, stride, 1)
    assert ref[2] == 5
    assert np.all(np.isfinite(ref[0])) and np.any(ref[0] != 0)
    for parts in (2, 3, 4):
        got = _step(big, W, stride, parts)
        assert got[2] == 5 * parts            # the split did run: 5 launches per sub-batch
        _same(got, ref)
    _same(_step(big, W, stride, 0), ref)       # the library's own choice


def test_split_bit_identical_hetero(big):
    stride = _hetero(big, W)
    ref = _step(big, W, stride, 1)
    for parts in (2, 3, 4):
        got = _step(big, W, stride, parts)
        assert got[2] == 5 * parts
        _same(got, ref)
    _same(_step(big, W, stride, 0), ref)


def test_split_bit_identical_odd_count(big):
    n = 4093                                   # prime: no sub-batch count divides it
    stride = _cfg2(big, n)
    ref = _step(big, n, stride, 1)
    for parts in (2, 3, 4):
        got = _step(big, n, stride, parts)
        assert got[2] == 5 * parts
        _same(got, ref)


def test_split_small_batch_keeps_one_part(big):
    """a batch too small for every part to keep the whole batch's launch shapes is not split, even when forced"""
    n = 200                                    # less than one window per SM in each of two parts (132 SMs)
    stride = _cfg2(big, n)
    ref = _step(big, n, stride, 1)
    got = _step(big, n, stride, 4)
    assert got[2] == 5
    _same(got, ref)


def test_split_stage_times_cover_the_whole_batch(big):
    _cfg2(big, W)
    for parts in (1, 2):
        assert big.lib.pvio_b200_internal_set_step_split(big.h, parts) == 0
        big.batch_gn_step(W, 1e-8, apply=False)
        big.sync()
        big.last_kernel_ms(-1)
        for _ in range(3):
            big.batch_gn_step(W, 1e-8, apply=False)
        stage, lin, schur = big.last_kernel_ms(1), big.last_kernel_ms(2), big.last_kernel_ms(3)
        assert lin > 0 and schur > 0
        assert abs(lin + schur - stage) <= 1e-3 * stage + 1e-3
    assert big.lib.pvio_b200_internal_set_step_split(big.h, 0) == 0
