"""Host mirror of OpenCvImage::track_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:88-136)
over the C-ABI: pyramidal LK on the GPU (pvio_b200_klt_track) followed by the reference's 20-px
border rejection (:106) and the F-matrix RANSAC of :121-129 (pvio_b200_find_fundamental_mask;
track_keypoints(..., ransac=True) is the whole OpenCvImage::track_keypoints)."""
import numpy as np

from . import _lib


def clahe(ba, img, clip_limit=6.0, tiles=(8, 8)):
    """cv::createCLAHE(clip_limit, tiles)->apply on the device (opencv_image.cpp:138-143); bit-exact with OpenCV."""
    img = np.ascontiguousarray(img, dtype=np.uint8)
    h, w = img.shape
    out = np.zeros_like(img)
    ba._ck(ba.lib.pvio_b200_clahe(ba.h, _lib.ptr(img), w, h, w, float(clip_limit), tiles[0], tiles[1], _lib.ptr(out)))
    return out


def track_keypoints(ba, prev_img, next_img, curr_keypoints, next_keypoints=None, max_level=3, max_iter=30,
                    eps=0.01, border=20, raw=False, clahe_clip=0.0, clahe_tiles=(8, 8), prev_id=0, next_id=0, shape=None):
    """ba: a BundleAdjustor (owns the device handle).  Images: uint8 [h, w].  Keypoints in pixels.
    clahe_clip > 0: the images are the RAW frames and CLAHE runs on the device first (OpenCvImage::preprocess).
    prev_id / next_id != 0: frame ids for the device-side pyramid cache (pvio_b200_klt_track_cached): a frame whose id
    is cached is not uploaded again (prev_img may then be None); the border test also runs on the device.
    Returns (next_keypoints float32 [n,2], status uint8 [n], err float32 [n])."""
    if prev_id or next_id:
        return _track_cached(ba, prev_img, next_img, curr_keypoints, next_keypoints, max_level, max_iter, eps,
                             0 if raw else border, clahe_clip, clahe_tiles, prev_id, next_id, shape)
    prev_img = np.ascontiguousarray(prev_img, dtype=np.uint8)
    next_img = np.ascontiguousarray(next_img, dtype=np.uint8)
    h, w = prev_img.shape
    cur = np.ascontiguousarray(curr_keypoints, dtype=np.float32).reshape(-1, 2)
    nxt = cur.copy() if next_keypoints is None or len(next_keypoints) == 0 else \
        np.array(next_keypoints, dtype=np.float32, copy=True).reshape(-1, 2)
    n = len(cur)
    status = np.zeros(max(n, 1), dtype=np.uint8)
    err = np.zeros(max(n, 1), dtype=np.float32)
    if clahe_clip > 0:
        rc = ba.lib.pvio_b200_klt_track_raw(ba.h, _lib.ptr(prev_img), _lib.ptr(next_img), w, h, w, _lib.ptr(cur),
                                            _lib.ptr(nxt), _lib.ptr(status), _lib.ptr(err), n, max_level, max_iter, eps,
                                            float(clahe_clip), clahe_tiles[0], clahe_tiles[1], None, None)
    else:
        rc = ba.lib.pvio_b200_klt_track(ba.h, _lib.ptr(prev_img), _lib.ptr(next_img), w, h, w, _lib.ptr(cur), _lib.ptr(nxt),
                                        _lib.ptr(status), _lib.ptr(err), n, max_level, max_iter, eps)
    ba._ck(rc)
    status, err = status[:n], err[:n]
    if not raw:
        out = (nxt[:, 0] < border) | (nxt[:, 0] >= w - border) | (nxt[:, 1] < border) | (nxt[:, 1] >= h - border)
        status = np.where(out, 0, status).astype(np.uint8)      # opencv_image.cpp:106-108
    return nxt, status, err


def _track_cached(ba, prev_img, next_img, curr_keypoints, next_keypoints, max_level, max_iter, eps, border, clahe_clip,
                  clahe_tiles, prev_id, next_id, shape):
    imgs = [None if im is None else np.ascontiguousarray(im, dtype=np.uint8) for im in (prev_img, next_img)]
    ref = imgs[1] if imgs[1] is not None else imgs[0]
    h, w = ref.shape if ref is not None else shape        # both frames cached: the caller names the frame size
    cur = np.ascontiguousarray(curr_keypoints, dtype=np.float32).reshape(-1, 2)
    nxt = cur.copy() if next_keypoints is None or len(next_keypoints) == 0 else \
        np.array(next_keypoints, dtype=np.float32, copy=True).reshape(-1, 2)
    n = len(cur)
    status = np.zeros(max(n, 1), dtype=np.uint8)
    err = np.zeros(max(n, 1), dtype=np.float32)
    p = _lib.ptr
    ba._ck(ba.lib.pvio_b200_klt_track_cached(ba.h, prev_id, p(imgs[0]), next_id, p(imgs[1]), w, h, w, p(cur), p(nxt),
                                             p(status), p(err), n, max_level, max_iter, eps, float(clahe_clip),
                                             clahe_tiles[0], clahe_tiles[1], int(border)))
    return nxt, status[:n], err[:n]


def find_fundamental_mask(ba, p, q, threshold=1.0, confidence=0.99, max_iters=1000, schedule=None, return_info=False):
    """cv::findFundamentalMat(p, q, FM_RANSAC, threshold, confidence, mask) on the device (opencv_image.cpp:123);
    schedule: int32 [S][7] injected sample indices, None = the samples OpenCV itself draws.
    Returns (mask uint8 [n], F [3,3]) (+ info dict: iterations, best_iteration, best_model, method)."""
    p = np.ascontiguousarray(p, dtype=np.float32).reshape(-1, 2)
    q = np.ascontiguousarray(q, dtype=np.float32).reshape(-1, 2)
    n = len(p)
    mask = np.zeros(max(n, 1), dtype=np.uint8)
    F = np.zeros(9)
    info = np.zeros(4, dtype=np.int32)
    sch = None if schedule is None else np.ascontiguousarray(schedule, dtype=np.int32).reshape(-1, 7)
    ba._ck(ba.lib.pvio_b200_find_fundamental_mask(ba.h, n, _lib.ptr(p), _lib.ptr(q), float(threshold), float(confidence),
                                                  int(max_iters), _lib.ptr(sch), 0 if sch is None else len(sch),
                                                  _lib.ptr(mask), _lib.ptr(F), _lib.ptr(info)))
    out = (mask[:n], F.reshape(3, 3))
    if return_info:
        out += ({"iterations": int(info[0]), "best_iteration": int(info[1]), "best_model": int(info[2]),
                 "method": {0: None, 1: "ransac", 2: "lmeds", 3: "7point"}[int(info[3])]},)
    return out


def track_keypoints_ransac(ba, prev_img, next_img, curr_keypoints, next_keypoints=None, prev_id=1, next_id=2, max_level=3,
                           max_iter=30, eps=0.01, border=20, clahe_clip=0.0, clahe_tiles=(8, 8), shape=None,
                           ransac_threshold=1.0, ransac_confidence=0.99):
    """The whole OpenCvImage::track_keypoints (opencv_image.cpp:88-136) in one C-ABI call: LK on the cached pyramids,
    20-px border, F-matrix RANSAC over the survivors (>= 8).  Returns (next_keypoints float32 [n,2], status uint8 [n])."""
    imgs = [None if im is None else np.ascontiguousarray(im, dtype=np.uint8) for im in (prev_img, next_img)]
    ref = imgs[1] if imgs[1] is not None else imgs[0]
    h, w = ref.shape if ref is not None else shape
    cur = np.ascontiguousarray(curr_keypoints, dtype=np.float32).reshape(-1, 2)
    nxt = cur.copy() if next_keypoints is None or len(next_keypoints) == 0 else \
        np.array(next_keypoints, dtype=np.float32, copy=True).reshape(-1, 2)
    n = len(cur)
    status = np.zeros(max(n, 1), dtype=np.uint8)
    p = _lib.ptr
    ba._ck(ba.lib.pvio_b200_track_keypoints(ba.h, prev_id, p(imgs[0]), next_id, p(imgs[1]), w, h, w, p(cur), p(nxt),
                                            p(status), n, max_level, max_iter, eps, float(clahe_clip), clahe_tiles[0],
                                            clahe_tiles[1], int(border), float(ransac_threshold),
                                            float(ransac_confidence)))
    return nxt, status[:n]


def pack_pairs(pairs):
    """The pvio_b200_klt_pair array of a batched call (see batch_track_keypoints) and its output arrays: returns
    (CKltPair array, outputs [(next_pts, status, err, info)] per pair, the arrays that must stay alive for the call)."""
    n = len(pairs)
    cp = (_lib.CKltPair * max(n, 1))()
    outs, keep = [], []
    for i, d in enumerate(pairs):
        imgs = [None if d.get(k) is None else np.ascontiguousarray(d[k], dtype=np.uint8) for k in ("prev", "next")]
        ref = imgs[1] if imgs[1] is not None else imgs[0]
        h, w = ref.shape if ref is not None else d["shape"]
        cur = np.ascontiguousarray(d["pts"], dtype=np.float32).reshape(-1, 2)
        init = d.get("init")
        nxt = cur.copy() if init is None or len(init) == 0 else np.array(init, dtype=np.float32, copy=True).reshape(-1, 2)
        m = len(cur)
        status = np.zeros(max(m, 1), dtype=np.uint8)
        err = np.zeros(max(m, 1), dtype=np.float32)
        info = np.zeros(4, dtype=np.int32)
        c = cp[i]
        c.slot, c.width, c.height, c.stride = int(d["slot"]), w, h, w
        c.prev_id, c.next_id = int(d["prev_id"]), int(d["next_id"])
        c.n_points = m
        _lib.set_ptrs(c, prev=imgs[0], next=imgs[1], prev_pts=cur, next_pts=nxt, status=status, err=err, info=info)
        keep += [imgs, cur, nxt, status, err, info]
        outs.append((nxt, status[:m], err[:m], info))
    return cp, outs, keep


def batch_track_keypoints(ba, pairs, max_level=3, max_iter=30, eps=0.01, clahe_clip=0.0, clahe_tiles=(8, 8), border=20,
                          ransac_threshold=1.0, ransac_confidence=0.99):
    """OpenCvImage::track_keypoints (opencv_image.cpp:88-136) for many sequences in one C-ABI call
    (pvio_b200_batch_track_keypoints).  pairs: one dict per sequence with slot (its cache slot, distinct within the
    call), prev_id / next_id (frame ids within the sequence, != 0), prev / next (uint8 [h, w] frames, raw when
    clahe_clip > 0; None when the id is cached in the slot), pts (float32 [n, 2]), optionally init (the initial guess,
    default pts) and shape ((h, w), needed when both frames are None).
    Returns one (next_keypoints float32 [n, 2], status uint8 [n], err float32 [n], info int32 [4]) per pair; info as
    find_fundamental_mask's (iterations, best iteration, best model, method), {0, -1, -1, 0} when RANSAC did not run."""
    cp, outs, keep = pack_pairs(pairs)
    ba._ck(ba.lib.pvio_b200_batch_track_keypoints(ba.h, len(pairs), cp, int(max_level), int(max_iter), float(eps),
                                                  float(clahe_clip), int(clahe_tiles[0]), int(clahe_tiles[1]), int(border),
                                                  float(ransac_threshold), float(ransac_confidence)))
    del keep
    return outs
