"""The windows of test_gpu_step_shapes have exactly the shapes their cases are named for: frame, landmark and
observation counts, fixed frames, the chunks api.cu's pack_window cuts (96 at the 3,072-landmark limit, 97 for the
window it must reject) and the rows of 32 of the frame-major table.  And the oracle step of each is finite."""
import numpy as np
import pytest

from test_gpu_step_shapes import (CASES, HET, MAX_CHUNKS, MU, MU_GAUGE, SHAPE_FREE, SHAPE_M, SMALL, case, chunk_count,
                                  n_free, segment_rows, window)

# name -> (N, M, K, fixed frames, chunks, segment rows)
EXPECT = {f"M{m}": (4, m, 3 * m, (0, 1), -(-m // 32), 3 * -(-m // 32)) for m in SHAPE_M}
EXPECT.update({
    "N2": (2, 64, 64, (0,), 2, 2),
    "N3": (3, 64, 128, (0, 1), 2, 4),
    "M3073": (4, 3073, 3 * 3073, (0, 1), 97, 3 * 97),
    "cap65": (4, 65, 195, (0, 1), 3, 9),
    "cap66": (4, 66, 198, (0, 1), 3, 9),
    "cap67": (4, 67, 201, (0, 1), 3, 9),
    "lm3000": (4, 3000, 9000, (0, 1), 94, 3 * 94),
    "cfg2": (10, 500, 4500, (0, 1), 16, 9 * 16),
    "small0": (6, 80, 400, (0, 1), 3, 15),
    "small2": (8, 100, 700, (0, 5), 4, 28),
})


def _staggered(N, M):
    """cfg2b: landmark l anchored in frame l mod 5 and seen in every later frame"""
    per = [len(range(a, M, 5)) for a in range(5)]
    K = sum(n * (N - 1 - a) for a, n in enumerate(per))
    chunks = sum(-(-n // 32) for n in per)
    rows = sum(-(-n // 32) * (N - 1 - a) for a, n in enumerate(per))
    return K, chunks, rows


for name, fx in [("N16", (0, 1)), ("free15_16", (7,))] + [(f"free{k}", f) for k, f in SHAPE_FREE.items()]:
    M = 96 if name.startswith("free") and name != "free15_16" else 240
    EXPECT[name] = (16, M) + (_staggered(16, M)[0], fx) + _staggered(16, M)[1:]


@pytest.mark.parametrize("name", sorted(EXPECT))
def test_window_has_its_named_shape(name):
    w, st = window(name)
    N, M, K, fixed, chunks, rows = EXPECT[name]
    w.validate()
    assert (w.N, w.M, w.K) == (N, M, K)
    assert tuple(np.nonzero(w.frame_fixed)[0]) == tuple(fixed)
    assert n_free(w) == N - len(fixed)
    assert chunk_count(w) == chunks
    assert segment_rows(w) == rows
    assert st.rho.shape == (M,) and np.all(st.rho > 0)


def test_free_frame_sets():
    for k, fx in SHAPE_FREE.items():
        w, _ = window(f"free{k}")
        assert n_free(w) == k
    # non-contiguous constant frames: a free frame between fixed ones, fixed ones between free ones
    assert np.nonzero(window("free1")[0].frame_fixed == 0)[0].tolist() == [9]
    assert np.nonzero(window("free14")[0].frame_fixed)[0].tolist() == [3, 11]
    assert n_free(window("free15_16")[0]) == 15


def test_chunk_limit():
    assert chunk_count(window("M3072")[0]) == MAX_CHUNKS
    assert chunk_count(window("M3073")[0]) == MAX_CHUNKS + 1


@pytest.mark.parametrize("name", sorted(set(CASES) - {"M3073"}))
def test_oracle_step_is_finite(name):
    w, st, ref, mu = case(name)
    assert mu == (MU_GAUGE if name in ("M0", "M1", "N2", "free15", "free16", "free15_16") else MU)
    assert np.all(np.isfinite(ref["dx"])) and np.isfinite(ref["cost"])
    assert np.all(ref["dx"][~ref["free"]] == 0.0)
    if w.M == 0:
        assert ref["cost"] == 0.0 and np.all(ref["dx"] == 0.0)
    else:
        assert ref["cost"] > 0.0
    if n_free(w) > 0 and w.M > 0:
        assert np.any(ref["dx"][:15 * w.N] != 0.0)


def test_kind_lists():
    assert len(set(HET)) == 4 and len(set(SMALL)) == 3
    assert all(not window(n)[0].use_inertial for n in HET + SMALL)
    assert window("inertial")[0].use_inertial and window("plane")[0].n_ptracks > 0
