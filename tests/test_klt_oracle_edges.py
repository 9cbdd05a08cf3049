"""The LK tracker's edges on the CPU: the NumPy oracle (oracle/klt_oracle.py) pinned against cv2 at frame edges, odd and
small frame sizes (down to frames narrower than the 21-px window) and other LK parameters; the REFLECT_101 fold of the
kernels (csrc/klt_border.cuh), compiled into a host program, against cv2.borderInterpolate.  The edge cases built here
are the inputs of the GPU tests in test_gpu_klt_edges.py."""
import os
import shutil
import subprocess

import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")
from oracle import klt_oracle as ko
from synthetic import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN = 21

# (width, height): odd at every level, a 22-px level (176 at level 3), either side of the drop rule (86 / 84), 160 x 120
# (drops 20 x 15), frames narrower than the window
SIZES = [(753, 481), (751, 479), (176, 176), (86, 86), (84, 84), (178, 90), (160, 120), (64, 48), (20, 24), (12, 12)]
# cv2.buildOpticalFlowPyramid(img, (21, 21), 3)[0] + 1
LEVELS = {(753, 481): 4, (751, 479): 4, (176, 176): 4, (86, 86): 3, (84, 84): 2, (178, 90): 3, (160, 120): 3,
          (64, 48): 2, (20, 24): 1, (12, 12): 1}
PARAMS = ([("max_level", v) for v in (0, 1, 2, 4, 7)] + [("max_iter", v) for v in (0, 1, 5, 100, 150)] +
          [("eps", v) for v in (0.0, 1e-3, 0.5, 25.0)])


def edge_case(size, seed=1200):
    """A frame pair textured to its edge (make_klt_pair's texture and warp) with points that reach every border branch
    of the tracker.  Returns prev, next, pts [n, 2], init [n, 2] and the index arrays of each kind of point:
      grid     make_klt_pair's interior grid (empty on frames under 70 px);
      edge     x or y at 0, 0.5, 3, 9.5, 10, 10.5, w - 11, w - 10.5, w - 1, w - 0.5 (the other coordinate mid-frame),
               and the four corners;
      outside  x or y at -5, w + 3, w + 70 and w + 75 (at level 3 of 176 x 176 the last one's 24-px patch reaches index
               cols + 21, which one fold sends below 0);
      flat     the centre of a 40 x 40 flat patch (frames of at least 80 x 80).
    Of the grid and edge points' guesses a tenth start 6 px off, a twentieth 40 px off and one off the frame at (900, 50);
    the others start at the point."""
    w, h = size
    prev, nxt, grid, _ = synth.make_klt_pair(seed=seed, size=size, n_points=40, max_shift=4.0)
    prev, nxt = prev.copy(), nxt.copy()
    vx = [0.0, 0.5, 3.0, 9.5, 10.0, 10.5, w - 11.0, w - 10.5, w - 1.0, w - 0.5]
    vy = [0.0, 0.5, 3.0, 9.5, 10.0, 10.5, h - 11.0, h - 10.5, h - 1.0, h - 0.5]
    edge = [(x, h / 2 + 0.3) for x in vx] + [(w / 2 + 0.3, y) for y in vy] + [(0.0, 0.0), (w - 1.0, 0.0), (0.0, h - 1.0),
                                                                               (w - 1.0, h - 1.0)]
    outside = [(x, h / 2 + 0.3) for x in (-5.0, w + 3.0, w + 70.0, w + 75.0)] + \
              [(w / 2 + 0.3, y) for y in (-5.0, h + 3.0, h + 70.0, h + 75.0)]
    flat = []
    if w >= 80 and h >= 80:
        cx, cy = w // 2 - 20, h // 2 - 20
        prev[cy:cy + 40, cx:cx + 40] = 128
        nxt[cy:cy + 40, cx:cx + 40] = 128
        flat = [(cx + 20.0, cy + 20.0)]
        keep = (np.abs(grid[:, 0] - (cx + 20)) > 45) | (np.abs(grid[:, 1] - (cy + 20)) > 45)
        grid = grid[keep]                     # grid windows stay off the flat patch
    parts = [grid.reshape(-1, 2), np.array(edge, np.float32).reshape(-1, 2), np.array(outside, np.float32).reshape(-1, 2),
             np.array(flat, np.float32).reshape(-1, 2)]
    pts = np.concatenate(parts).astype(np.float32)
    init = pts.copy()
    r = np.random.default_rng(seed + 1)
    cand = np.arange(len(grid) + len(edge))                 # guesses of grid and edge points: a tenth 6 px off, a
    n6, n40 = max(len(cand) // 10, 2), max(len(cand) // 20, 2)        # twentieth 40 px off, one off the frame
    pick = r.choice(cand, n6 + n40 + 1, replace=False)
    init[pick[:n6]] += r.choice([-6.0, 6.0], (n6, 2)).astype(np.float32)
    init[pick[n6:n6 + n40]] += r.choice([-40.0, 40.0], (n40, 2)).astype(np.float32)
    init[pick[-1]] = (900.0, 50.0)
    off = np.cumsum([0] + [len(p) for p in parts])
    kinds = {k: np.arange(off[i], off[i + 1]) for i, k in enumerate(("grid", "edge", "outside", "flat"))}
    return prev, nxt, pts, init, kinds


def cv_lk(prev, nxt, pts, init, max_level=3, max_iter=30, eps=0.01):
    p1, st, err = cv2.calcOpticalFlowPyrLK(prev, nxt, pts.reshape(-1, 1, 2).copy(), init.reshape(-1, 1, 2).copy(),
                                           winSize=(WIN, WIN), maxLevel=max_level,
                                           criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, max_iter, eps),
                                           flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
    return p1.reshape(-1, 2), st.ravel(), err.ravel()


def assert_lk_parity(got, want, what=""):
    """status bit for bit; positions and error within 1e-2 px on the tracked points"""
    (p, st, err), (pw, stw, errw) = got[:3], want[:3]
    assert np.array_equal(st, stw), (what, np.nonzero(st != stw)[0])
    ok = stw == 1
    if ok.any():
        assert np.max(np.abs(p[ok] - pw[ok])) < 1e-2, what
        assert np.max(np.abs(err[ok] - errw[ok])) < 1e-2, what


def crosses_edge(pts, ok, size, level):
    """the points of `ok` whose 21 x 21 window (plus the bilinear neighbour) at `level` reaches outside that level"""
    w, h = size
    for _ in range(level):
        w, h = (w + 1) // 2, (h + 1) // 2
    q = pts[ok] / np.float32(1 << level) - np.float32((WIN - 1) / 2)
    i = np.floor(q).astype(int)
    return (i[:, 0] < 0) | (i[:, 1] < 0) | (i[:, 0] + WIN >= w) | (i[:, 1] + WIN >= h)


# ---- the fold ------------------------------------------------------------------------------------------------------
def _host_fold_table(tmp_path):
    """reflect101 / reflect101_once of csrc/klt_border.cuh compiled into a host program: one line 'n i r r1' per index
    for n in 1..64, i in [-2n - 30, 3n + 30]"""
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cxx = nvcc if os.path.exists(nvcc) else shutil.which("c++") or shutil.which("g++")
    if cxx is None:
        pytest.skip("no C++ compiler")
    src = tmp_path / "fold.cpp"
    src.write_text('#include <cstdio>\n#include "klt_border.cuh"\nint main() {\n'
                   '  for (int n = 1; n <= 64; ++n)\n    for (int i = -2 * n - 30; i <= 3 * n + 30; ++i)\n'
                   '      std::printf("%d %d %d %d\\n", n, i, pvio::reflect101(i, n), pvio::reflect101_once(i, n));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / "fold"
    subprocess.run([cxx, "-x", "c++", "-std=c++17", "-I", os.path.join(ROOT, "pvio_b200", "csrc"), str(src), "-o", str(exe)],
                   check=True, capture_output=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    return np.array([list(map(int, l.split())) for l in out.splitlines()])


def test_reflect101_fold_equals_cv2_border_interpolate(tmp_path):
    """Every n in 1..64: the LK window's two-fold reflect101 is cv2's BORDER_REFLECT_101 on [-3 (n - 1), 3 (n - 1)], which
    holds every index the window reads (-22 .. n + 21) once n >= 12, the smallest frame the tracker takes; pyrDown's
    one-fold variant is on [-(n - 1), 2 (n - 1)]; both fail outside, as a one-fold helper did for n + 21 on a 22-px level."""
    t = _host_fold_table(tmp_path)
    assert len(t) == sum(5 * n + 61 for n in range(1, 65))
    n, i = t[:, 0], t[:, 1]
    want = np.array([cv2.borderInterpolate(int(a), int(b), cv2.BORDER_REFLECT_101) for b, a in t[:, :2]])
    two = (np.abs(i) <= 3 * (n - 1))
    assert np.array_equal(t[two, 2], want[two]), t[two][t[two, 2] != want[two]][:10]
    one = (i >= -(n - 1)) & (i <= 2 * (n - 1))
    assert np.array_equal(t[one, 3], want[one])
    lk = (n >= 12) & (i >= -22) & (i <= n + 21)
    assert lk.sum() == sum(n_ + 44 for n_ in range(12, 65)) and two[lk].all()
    assert cv2.borderInterpolate(43, 22, cv2.BORDER_REFLECT_101) == 1
    assert t[(n == 22) & (i == 43), 2] == 1 and t[(n == 22) & (i == 43), 3] == -1


def test_pyrdown_taps_stay_within_one_fold():
    """pyrDown's taps 2x - 2 .. 2x + 2 on a level of sw >= 43 px (the smallest a pyramid level is built from) lie in
    [-(sw - 1), 2 (sw - 1)], where reflect101_once is exact; and the oracle's pyrDown equals cv2's at odd sizes."""
    for sw in range(43, 200):
        dw = (sw + 1) // 2
        assert -2 >= -(sw - 1) and 2 * (dw - 1) + 2 <= 2 * (sw - 1)
    for w, h in [(753, 481), (751, 479), (377, 241), (189, 121), (95, 61), (45, 43), (43, 44)]:
        img = synth.make_klt_pair(seed=w, size=(w, h), n_points=1)[0]
        assert np.array_equal(ko.pyr_down(img), cv2.pyrDown(img)), (w, h)


# ---- pyramid depth ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
def test_pyramid_depth_matches_cv2(size):
    """buildOpticalFlowPyramid halves first and drops the new level when it is not larger than the window."""
    img = np.zeros((size[1], size[0]), np.uint8)
    assert len(ko.build_pyramid(img, 3)) == LEVELS[size]
    for L in (0, 1, 2, 3, 4, 7):
        n_cv = cv2.buildOpticalFlowPyramid(img, (WIN, WIN), L, withDerivatives=False)[0] + 1
        assert len(ko.build_pyramid(img, L)) == n_cv, (size, L)


# ---- LK parity -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("size", SIZES)
def test_oracle_matches_cv2_on_edge_points(size):
    prev, nxt, pts, init, _ = edge_case(size)
    assert_lk_parity(ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init), cv_lk(prev, nxt, pts, init), size)


@pytest.mark.parametrize("name,value", PARAMS)
def test_oracle_matches_cv2_at_other_parameters(name, value):
    """max_level 0..7, max_iter 0..150 and eps 0..25 (OpenCV clamps max_iter to 100 and eps to 10)."""
    prev, nxt, pts, init, _ = edge_case((176, 176))
    kw = {"max_level": 3, "max_iter": 30, "eps": 0.01, name: value}
    assert_lk_parity(ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init, **kw), cv_lk(prev, nxt, pts, init, **kw), kw)


def test_edge_cases_reach_their_branches():
    """The edge cases lose points for every reason the tracker has, track points whose windows cross the frame edge at
    levels 0 and 3, and track points on frames narrower than the window."""
    reasons = set()
    for size in [(753, 481), (176, 176), (86, 86), (160, 120), (12, 12)]:
        prev, nxt, pts, init, kinds = edge_case(size)
        _, st, _, why = ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init, return_reasons=True)
        reasons |= set(why[st == 0].tolist())
        if kinds["flat"].size:
            assert why[kinds["flat"]][0] == ko.LOST_MIN_EIG
        ok = st == 1
        assert crosses_edge(pts, ok, size, 0).any(), size
        if LEVELS[size] == 4:
            assert crosses_edge(pts, ok, size, 3).any(), size
        if size == (12, 12):
            assert ok.sum() >= 4
    assert {ko.LOST_OUTSIDE, ko.LOST_MIN_EIG, ko.LOST_ITERATING} <= reasons, reasons
    # the guess off the frame is lost while iterating
    prev, nxt, pts, init, kinds = edge_case((753, 481))
    far = np.nonzero((init[:, 0] == 900.0) & (init[:, 1] == 50.0))[0]
    _, st, _, why = ko.calc_optical_flow_pyr_lk(prev, nxt, pts, init, return_reasons=True)
    assert len(far) == 1 and why[far[0]] == ko.LOST_ITERATING
