"""Lens distortion removal of PVIO's dataset readers over the C-ABI: cv::undistort with K, D as Mat_<float>
(EurocDatasetReader::read_image, pvio-pc/src/euroc_dataset_reader.cpp:70-74) and ImageUndistorter's equidistant remap
(pvio-extra/include/pvio/extra/image_undistorter.h:28-95), bit for bit.  A lens is set once per sequence slot of the
batched tracker; the batched tracker and detector then take that slot's raw frames (klt.batch_track_keypoints and
detect.batch_detect_keypoints are unchanged)."""
import numpy as np

from . import _lib

NONE, RADTAN, EQUIDISTANT = 0, _lib.LENS_RADTAN, _lib.LENS_EQUIDISTANT


def undistort_map(model, width, height, K, coeffs):
    """Host only: the map of one lens (pvio_b200_undistort_map).  K = (fx, fy, cx, cy), coeffs [4] (radtan: k1 k2 p1 p2;
    equidistant: k1 k2 k3 k4).  Returns OpenCV's CV_16SC2 pair (m1 int16 [h, w, 2], m2 uint16 [h, w]); raises
    ValueError on a rejected lens."""
    lib = _lib.load()
    p = np.ascontiguousarray(K, dtype=np.float64).reshape(4)
    c = np.ascontiguousarray(coeffs, dtype=np.float64).reshape(4)
    m1 = np.zeros((height, width, 2), np.int16)
    m2 = np.zeros((height, width), np.uint16)
    rc = lib.pvio_b200_undistort_map(int(model), int(width), int(height), _lib.ptr(p), _lib.ptr(c), _lib.ptr(m1),
                                     _lib.ptr(m2))
    if rc != 0:
        raise ValueError(f"pvio_b200_undistort_map rejected the lens ({rc})")
    return m1, m2


def pack_lenses(lenses):
    """the pvio_b200_lens array of set_lens"""
    arr = (_lib.CLens * max(len(lenses), 1))()
    for i, d in enumerate(lenses):
        r = arr[i]
        r.slot, r.model = int(d["slot"]), int(d.get("model", NONE))
        r.width, r.height = int(d.get("width", 0)), int(d.get("height", 0))
        r.fx, r.fy, r.cx, r.cy = (float(v) for v in d.get("K", (0.0, 0.0, 0.0, 0.0)))
        r.coeffs[:] = [float(v) for v in d.get("coeffs", (0.0, 0.0, 0.0, 0.0))]
    return arr


def set_lens(ba, lenses):
    """pvio_b200_batch_set_lens: lenses is a list of dicts with slot, model (NONE clears the slot's lens, RADTAN,
    EQUIDISTANT), width, height (the raw frame's shape), K = (fx, fy, cx, cy) and coeffs [4].  Drops each named slot's
    cached frames."""
    ba._ck(ba.lib.pvio_b200_batch_set_lens(ba.h, len(lenses), pack_lenses(lenses)))


def batch_undistort(ba, requests):
    """pvio_b200_batch_undistort: requests is a list of dicts with slot (a slot with a lens) and image (the raw uint8
    [h, w] frame).  Returns the undistorted frames, uint8 [h, w] each."""
    n = len(requests)
    arr = (_lib.CUndistortRequest * max(n, 1))()
    keep, outs = [], []
    for i, d in enumerate(requests):
        img = np.ascontiguousarray(d["image"], dtype=np.uint8)
        h, w = img.shape
        out = np.zeros((h, w), np.uint8)
        r = arr[i]
        r.slot, r.width, r.height, r.stride = int(d["slot"]), w, h, w
        _lib.set_ptrs(r, src=img, dst=out)
        keep.append(img)
        outs.append(out)
    ba._ck(ba.lib.pvio_b200_batch_undistort(ba.h, n, arr))
    del keep
    return outs
