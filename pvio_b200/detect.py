"""Host mirror of OpenCvImage::detect_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:54-86) over the C-ABI:
Harris-GFTT on the device, PVIO's Poisson-disk filter against the frame's existing keypoints, 20-pixel border."""
import ctypes as C

import numpy as np

from . import _lib


def detect_keypoints(ba, image, keypoints=(), keypoint_distance=25.0, clahe_clip=0.0, clahe_tiles=(8, 8), frame_id=0,
                     shape=None, want_gftt=False, max_out=2048):
    """ba: a BundleAdjustor (owns the device handle).  image: uint8 [h, w] (None if frame_id is in the KLT pyramid
    cache; `shape` then names the frame size).  keypoints: the frame's existing keypoints [n, 2] (pixels).
    Returns the NEW keypoints [m, 2] in the reference's order (and the GFTT corners before the filter if want_gftt)."""
    img = None if image is None else np.ascontiguousarray(image, dtype=np.uint8)
    h, w = img.shape if img is not None else shape
    ex = np.ascontiguousarray(keypoints, dtype=np.float64).reshape(-1, 2)
    out = np.zeros((max_out, 2))
    gftt = np.zeros((1000, 2), dtype=np.float32)
    n, ng = C.c_int(), C.c_int()
    ba._ck(ba.lib.pvio_b200_detect_keypoints(ba.h, int(frame_id), _lib.ptr(img), w, h, w, float(clahe_clip), clahe_tiles[0],
                                             clahe_tiles[1], _lib.ptr(ex) if len(ex) else None, len(ex),
                                             float(keypoint_distance), max_out, _lib.ptr(out), C.byref(n), _lib.ptr(gftt),
                                             C.byref(ng)))
    return (out[:n.value].copy(), gftt[:ng.value].copy()) if want_gftt else out[:n.value].copy()


def pack_requests(requests, want_gftt=False):
    """The pvio_b200_detect_request array of a batched call (see batch_detect_keypoints) and its output arrays: returns
    (CDetectRequest array, outputs [(keypoints, n_out, gftt, n_gftt)] per request, the arrays that must stay alive)."""
    n = len(requests)
    cr = (_lib.CDetectRequest * max(n, 1))()
    outs, keep = [], []
    for i, d in enumerate(requests):
        img = None if d.get("image") is None else np.ascontiguousarray(d["image"], dtype=np.uint8)
        h, w = img.shape if img is not None else d["shape"]
        ex = np.ascontiguousarray(d.get("keypoints", ()), dtype=np.float64).reshape(-1, 2)
        max_out = int(d.get("max_out", 2048))
        out = np.zeros((max(max_out, 1), 2))
        cnt = np.zeros(2, dtype=np.int32)                  # n_out, n_gftt
        gftt = np.zeros((1000, 2), dtype=np.float32) if want_gftt else None
        c = cr[i]
        c.slot, c.width, c.height, c.stride = int(d["slot"]), w, h, w
        c.frame_id = int(d.get("frame_id", 0))
        c.n_existing = len(ex)
        c.max_out = max_out
        c.keypoint_distance = float(d.get("keypoint_distance", 25.0))
        _lib.set_ptrs(c, image=img, existing=ex if len(ex) else None, keypoints_out=out, n_out=cnt[:1], gftt_out=gftt,
                      n_gftt=cnt[1:])
        keep += [img, ex, out, cnt, gftt]
        outs.append((out, cnt, gftt))
    return cr, outs, keep


def batch_detect_keypoints(ba, requests, clahe_clip=0.0, clahe_tiles=(8, 8), want_gftt=False):
    """OpenCvImage::detect_keypoints (opencv_image.cpp:54-86) for many frames in one C-ABI call
    (pvio_b200_batch_detect_keypoints).  requests: one dict per frame with slot (a sequence slot of
    klt.batch_track_keypoints), frame_id (its id in that slot; 0 or not cached: `image` is uploaded), image (uint8 [h, w],
    raw when clahe_clip > 0; None when frame_id is cached in the slot, `shape` (h, w) then names the size), keypoints
    (the frame's existing keypoints [n, 2]), keypoint_distance (default 25) and max_out (default 2048).
    Returns per request the new keypoints [m, 2] in the reference's order (and the GFTT corners if want_gftt), each as
    detect.detect_keypoints gives it."""
    cr, outs, keep = pack_requests(requests, want_gftt)
    ba._ck(ba.lib.pvio_b200_batch_detect_keypoints(ba.h, len(requests), cr, float(clahe_clip), int(clahe_tiles[0]),
                                                   int(clahe_tiles[1])))
    del keep
    res = []
    for out, cnt, gftt in outs:
        kp = out[:cnt[0]].copy()
        res.append((kp, gftt[:cnt[1]].copy()) if want_gftt else kp)
    return res
