"""The batched linearise sweep (one CTA per window, per-landmark sums in shared memory) evaluates two rows of the
frame-major table per lane and iteration and emits their contributions in row order.  Checked here on the row layouts
that path meets: segments of 1, 2 and 3 rows, a partial last row, odd pieces, warps whose row ranges start on an odd
row, and a staggered window with free anchors -- against the several-CTAs-per-window path (one row per iteration,
per-block records summed by lm_finish_kernel) and the oracle, with bit-identical repeats.  Segments of 63, 64, 65 and
96 rows (the most a window holds: 96 chunks of 32 landmarks) need more landmarks than the shared-sum layout holds, so
they take the one-row records path, in pieces of <= 64 rows; checked against the oracle as well.  The victim-only
marginaliser sweep (fp64, one row) is checked on the short-segment shapes."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from synthetic import synth
from pvio_b200.bundle_adjustor import BundleAdjustor

pytestmark = pytest.mark.gpu

kLinWarps = 4         # warps of a linearise CTA (api.cu); warp w owns rows [rows w / 4, rows (w + 1) / 4) of its window


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def _segment_rows(w):
    """rows of each (target, anchor) segment of the window's frame-major table: 32 blocks per row"""
    anchors = np.asarray(w.lm_anchor)
    ob = np.asarray(w.lm_obs_begin)
    frames = np.asarray(w.obs_frame)
    counts = {}
    for l in range(w.M):
        for t in frames[ob[l]:ob[l + 1]]:
            if t != anchors[l]:
                counts[(int(t), int(anchors[l]))] = counts.get((int(t), int(anchors[l])), 0) + 1
    return [(c + 31) // 32 for c in counts.values()]


def _warp_starts(w):
    rows = sum(_segment_rows(w))
    return [rows * k // kLinWarps for k in range(kLinWarps)]


def _window(N, M, staggered=False, seed=901, free_anchors=False):
    w, st, _ = synth.make_cfg2(N=N, M=M, staggered=staggered, seed=seed)
    if free_anchors:                    # frames 0 and 5 fixed (gauge and scale): the anchors 1 .. 4 of the staggered landmarks are free
        w.frame_fixed[:] = 0
        w.frame_fixed[0] = 1
        w.frame_fixed[5] = 1
    return w, st


SHORT = [
    # (N, M, staggered, free anchors): segments of 1 row (warp 0 owns no row), 2 and 3 rows; a partial last row
    (4, 32, False, False),
    (4, 64, False, False),
    (5, 96, False, False),
    (4, 33, False, False),
    (8, 300, False, False),
    (9, 350, True, True),
]


@pytest.fixture(scope="module")
def ba():
    b = BundleAdjustor(max_windows=80, max_frames=10, max_landmarks=512, max_obs=4608)
    yield b
    b.close()


def test_short_segment_shapes_cover_odd_rows():
    """the shapes below do what the test is for: odd piece lengths and odd warp starts"""
    rows = set()
    starts = []
    for N, M, stg, fa in SHORT:
        w, _ = _window(N, M, stg, free_anchors=fa)
        rows.update(_segment_rows(w))
        starts += _warp_starts(w)
    assert {1, 2, 3} <= rows
    assert any(s % 2 for s in starts)
    w, _ = _window(9, 350, True, free_anchors=True)
    assert any(a > 0 and not w.frame_fixed[a] for a in np.asarray(w.lm_anchor))


@pytest.mark.parametrize("N,M,staggered,free_anchors", SHORT)
def test_row_pairs_match_records_path_and_oracle(ba, N, M, staggered, free_anchors):
    """80 copies of the window through the batched path (two rows in flight) against the same window alone (16 CTAs per
    window, one row per iteration, per-block records) and the oracle, within the bars of test_gpu_step_records; two
    batched steps are bit-identical."""
    w, st = _window(N, M, staggered, free_anchors=free_anchors)
    W, stride = 80, 15 * 10 + 512
    n = 15 * N + M
    ba.batch_set(0, w, st)
    ba.batch_replicate(W)
    ba.batch_upload(W)
    ba.batch_gn_step(W, 1e-8, apply=False)
    dx_b, c_b = ba.batch_download(W, stride)
    ba.batch_gn_step(W, 1e-8, apply=False)
    dx_b2, c_b2 = ba.batch_download(W, stride)
    assert np.array_equal(dx_b, dx_b2) and np.array_equal(c_b, c_b2)
    assert np.array_equal(dx_b[0], dx_b[W - 1]) and c_b[0, 0] == c_b[W - 1, 0]

    ba.batch_set(0, w, st)
    ba.batch_upload(1)
    ba.batch_gn_step(1, 1e-8, apply=False)
    dx_1, c_1 = ba.batch_download(1, stride)
    assert _rel(dx_b[0, :n], dx_1[0, :n]) < 1e-5
    assert abs(c_b[0, 0] - c_1[0, 0]) <= 2e-6 * c_1[0, 0]
    ref = bo.gn_step(w, st, schur=True)["dx"]
    assert _rel(dx_b[0, :n], ref) < 1e-5


@pytest.mark.parametrize("seg_rows", [63, 64, 65, 96])
def test_long_segments_take_the_records_path(seg_rows):
    """N = 3: two segments (1, 0), (2, 0) of seg_rows rows each (pieces of <= 64 rows); batched and single-window steps
    against the oracle."""
    N, M = 3, 32 * seg_rows - 5
    w, st = _window(N, M, seed=905)
    assert set(_segment_rows(w)) == {seg_rows}
    W, stride = 80, 15 * N + M
    b = BundleAdjustor(max_windows=W, max_frames=N, max_landmarks=M, max_obs=(N - 1) * M + 64 * N)
    try:
        b.batch_set(0, w, st)
        b.batch_replicate(W)
        b.batch_upload(W)
        b.batch_gn_step(W, 1e-8, apply=False)
        dx_b, _ = b.batch_download(W, stride)
        b.batch_upload(1)
        b.batch_gn_step(1, 1e-8, apply=False)
        dx_1, _ = b.batch_download(1, stride)
    finally:
        b.close()
    ref = bo.gn_step(w, st, schur=True)["dx"]
    assert _rel(dx_b[0], ref) < 1e-5
    assert _rel(dx_b[W - 1], ref) < 1e-5
    assert _rel(dx_1[0], ref) < 1e-5


def test_victim_only_sweep_matches_single_window():
    """The batched marginaliser (victim-only fp64 sweep with the shared sums) against the single-window marginaliser (the
    records path) on windows of 1-, 2- and 3-row segments."""
    W = 80
    kinds = [synth.make_cfg3(N=N, M=M, seed=940 + i, prior=p)[:2]
             for i, (N, M, p) in enumerate([(4, 32, 'synthetic'), (5, 64, 'gauge'), (6, 96, 'none')])]
    b = BundleAdjustor(max_windows=W, max_frames=6, max_landmarks=128, max_obs=1200)
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
