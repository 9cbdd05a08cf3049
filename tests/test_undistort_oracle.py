"""Lens undistortion without a GPU: oracle/undistort_oracle.py against cv2 (cv::undistort with Mat_<float> K and D, as
EurocDatasetReader::read_image; ImageUndistorter's equidistant float map through cv::convertMaps and cv::remap), and
the library's host-side map builder pvio_b200_undistort_map against the oracle, bit for bit, with its rejections."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import undistort_oracle as uo
from pvio_b200 import _lib
from pvio_b200.undistort import EQUIDISTANT, RADTAN, undistort_map
from pvio_b200._lib import EINVAL

cv2 = pytest.importorskip("cv2")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# (K = fx, fy, cx, cy), (k1, k2, p1, p2), width, height
RADTAN_LENSES = {
    "euroc": ((458.654, 457.296, 367.215, 248.375), (-0.28340811, 0.07395907, 0.00019359, 1.76187114e-05), 752, 480),
    "strong_barrel": ((300.0, 310.0, 320.5, 240.2), (-0.45, 0.2, 0.0, 0.0), 640, 480),
    "tangential": ((400.0, 405.0, 330.0, 250.0), (-0.1, 0.01, 0.02, -0.015), 640, 480),
    "small_97x61": ((60.0, 61.0, 48.0, 30.0), (-0.2, 0.05, 0.001, 0.002), 97, 61),
    "wide_4200": ((2000.0, 2000.0, 2100.0, 20.0), (-0.1, 0.02, 0.0005, 0.0003), 4200, 40),     # 1-row stripes
}
# TUM-VI's camera 0 (tum_dataset_reader.cpp:74-78) and a stronger fisheye at another size
EQUIDISTANT_LENSES = {
    "tumvi": ((190.97847715128717, 190.9733070521226, 254.93170605935475, 256.8974428996504),
              (0.0034003170790442797, 0.001766278153469831, -0.00266312569781606, 0.0003299517423931039), 512, 512),
    "fisheye_130x90": ((70.0, 72.0, 64.3, 44.9), (0.05, -0.02, 0.01, -0.003), 130, 90),
}


def _cv_k(K, D):
    fx, fy, cx, cy = K
    return (np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32), np.array(D, np.float32))


def _frames(w, h, seed):
    r = np.random.default_rng(seed)
    noise = r.integers(0, 256, (h, w), dtype=np.uint8)
    sat = noise.copy()
    sat[: h // 3, : w // 3] = 255
    sat[h // 2:, w // 2:] = 0
    return noise, sat


@pytest.mark.parametrize("name", sorted(RADTAN_LENSES))
def test_radtan_map_equals_cv2(name):
    K, D, w, h = RADTAN_LENSES[name]
    m1, m2 = uo.radtan_map(w, h, K, D)
    c1, c2 = cv2.initUndistortRectifyMap(*_cv_k(K, D), None, _cv_k(K, D)[0], (w, h), cv2.CV_16SC2)
    assert np.array_equal(m1, c1) and np.array_equal(m2, c2)


@pytest.mark.parametrize("name", sorted(RADTAN_LENSES))
def test_radtan_remap_equals_cv2_undistort(name):
    K, D, w, h = RADTAN_LENSES[name]
    m1, m2 = uo.radtan_map(w, h, K, D)
    for img in _frames(w, h, 11):
        assert np.array_equal(uo.remap(img, m1, m2), cv2.undistort(img, *_cv_k(K, D)))


@pytest.mark.parametrize("name", sorted(EQUIDISTANT_LENSES))
def test_equidistant_maps_convert_as_cv2(name):
    K, D, w, h = EQUIDISTANT_LENSES[name]
    mx, my = uo.equidistant_float_map(w, h, K, D)
    m1, m2 = uo.convert_maps(mx, my)
    c1, c2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    assert np.array_equal(m1, c1) and np.array_equal(m2, c2)
    for img in _frames(w, h, 12):
        want = cv2.remap(img, c1, c2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
        assert np.array_equal(uo.remap(img, m1, m2), want)


def test_remap_taps_outside_the_frame():
    """a map whose taps lie partly and wholly outside the frame: those taps read 0"""
    r = np.random.default_rng(13)
    img = r.integers(0, 256, (61, 97), dtype=np.uint8)
    mx = r.uniform(-40, 140, (61, 97)).astype(np.float32)
    my = r.uniform(-40, 100, (61, 97)).astype(np.float32)
    m1, m2 = uo.convert_maps(mx, my)
    c1, c2 = cv2.convertMaps(mx, my, cv2.CV_16SC2)
    assert np.array_equal(m1, c1) and np.array_equal(m2, c2)
    want = cv2.remap(img, c1, c2, cv2.INTER_LINEAR, borderMode=cv2.BORDER_CONSTANT, borderValue=0)
    assert np.array_equal(uo.remap(img, m1, m2), want)


@pytest.mark.parametrize("name", sorted(RADTAN_LENSES) + sorted(EQUIDISTANT_LENSES))
def test_library_map_equals_oracle(name):
    model = RADTAN if name in RADTAN_LENSES else EQUIDISTANT
    K, D, w, h = RADTAN_LENSES[name] if model == RADTAN else EQUIDISTANT_LENSES[name]
    m1, m2 = undistort_map(model, w, h, K, D)
    o1, o2 = uo.undistort_map(model, w, h, K, D)
    assert np.array_equal(m1, o1) and np.array_equal(m2, o2)


def _rc(model, w, h, K, D, m1=True, m2=True):
    lib = _lib.load()
    p = np.ascontiguousarray(K, dtype=np.float64)
    c = np.ascontiguousarray(D, dtype=np.float64)
    a = np.zeros((max(h, 1), max(w, 1), 2), np.int16)
    b = np.zeros((max(h, 1), max(w, 1)), np.uint16)
    return lib.pvio_b200_undistort_map(model, w, h, _lib.ptr(p), _lib.ptr(c),
                                       _lib.ptr(a) if m1 else None, _lib.ptr(b) if m2 else None)


def test_library_map_rejections():
    K, D, w, h = RADTAN_LENSES["small_97x61"]
    assert _rc(RADTAN, w, h, K, D) == 0 and _rc(EQUIDISTANT, w, h, K, D) == 0
    for model in (0, 3, -1):
        assert _rc(model, w, h, K, D) == EINVAL
    for model in (RADTAN, EQUIDISTANT):
        assert _rc(model, 7, h, K, D) == EINVAL
        assert _rc(model, w, 7, K, D) == EINVAL
        assert _rc(model, 32768, 8, K, D) == EINVAL
        for k in range(4):
            for bad in (math.nan, math.inf, -math.inf):
                Kb = list(K)
                Kb[k] = bad
                assert _rc(model, w, h, Kb, D) == EINVAL
                Db = list(D)
                Db[k] = bad
                assert _rc(model, w, h, K, Db) == EINVAL
        for k in range(2):
            for bad in (0.0, -1.0):
                Kb = list(K)
                Kb[k] = bad
                assert _rc(model, w, h, Kb, D) == EINVAL
        assert _rc(model, w, h, K, D, m1=False) == EINVAL
        assert _rc(model, w, h, K, D, m2=False) == EINVAL
    # map coordinates that are not finite: radtan's fx rounds to 0 in float32; the fisheye polynomial overflows
    assert _rc(RADTAN, w, h, (1e-300, 61.0, 48.0, 30.0), D) == EINVAL
    assert _rc(EQUIDISTANT, w, h, K, (1e308, 1e308, 0.0, 0.0)) == EINVAL


def test_struct_layouts_match_header():
    assert C.sizeof(_lib.CLens) == 80
    assert _lib.CLens.model.offset == 4 and _lib.CLens.width.offset == 8 and _lib.CLens.fx.offset == 16
    assert _lib.CLens.cy.offset == 40 and _lib.CLens.coeffs.offset == 48
    assert C.sizeof(_lib.CUndistortRequest) == 32
    assert _lib.CUndistortRequest.stride.offset == 12 and _lib.CUndistortRequest.src.offset == 16
    assert _lib.CUndistortRequest.dst.offset == 24


def test_struct_layouts_as_the_c_compiler_sees_them(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not installed")
    src = tmp_path / "layout.c"
    src.write_text(
        '#include <stddef.h>\n#include <stdio.h>\n#include "pvio_b200.h"\n'
        'int main(void) { printf("%zu %zu %zu %zu %zu %zu\\n", sizeof(pvio_b200_lens), offsetof(pvio_b200_lens, fx),\n'
        '  offsetof(pvio_b200_lens, coeffs), sizeof(pvio_b200_undistort_request),\n'
        '  offsetof(pvio_b200_undistort_request, src), offsetof(pvio_b200_undistort_request, dst)); return 0; }\n')
    exe = tmp_path / "layout"
    r = subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    out = subprocess.run([str(exe)], capture_output=True, text=True, timeout=60).stdout.split()
    assert [int(v) for v in out] == [80, _lib.CLens.fx.offset, _lib.CLens.coeffs.offset, 32,
                                     _lib.CUndistortRequest.src.offset, _lib.CUndistortRequest.dst.offset]
