"""The per-frame step of FeatureTracker::work (feature_tracker.cpp:77-99) for many sequences in one C-ABI call
(pvio_b200_batch_feature_track): track the previous frame's keypoints into the new frame, thin them by track length,
detect new ones.  Each sequence's keypoints stay in its slot on the device between calls."""
import math

import numpy as np

from . import _lib

MAX_CORNERS = 1000          # GFTTDetector::create(1000, ...): detections per frame, and untracked survivors


def min_capacity(width, height, keypoint_distance):
    """The smallest max_keypoints the call accepts for a width x height frame: cells + 2000, one keypoint per Poisson
    cell of side r / sqrt(2) after the thinning, plus at most 1000 untracked survivors and 1000 detections."""
    gs = keypoint_distance / math.sqrt(2.0)
    return (math.floor(width / gs) + 1) * (math.floor(height / gs) + 1) + 2 * MAX_CORNERS


def check_frames(frames, keypoint_distance):
    """The header's rejections that need no device: a slot named twice, a missing pixel array or frame id, a
    capacity below min_capacity.  Raises ValueError."""
    if not keypoint_distance > 0:
        raise ValueError("keypoint_distance must be > 0")
    seen = set()
    for d in frames:
        slot = int(d["slot"])
        if not 0 <= slot <= 65535:
            raise ValueError(f"slot {slot} out of range")
        if slot in seen:
            raise ValueError(f"slot {slot} appears twice")
        seen.add(slot)
        if d.get("image") is None or not int(d.get("frame_id", 0)):
            raise ValueError(f"slot {slot}: a frame needs its pixels and a frame id != 0")
        if int(d.get("map_frames", 0)) < 0:
            raise ValueError(f"slot {slot}: map_frames < 0")
        h, w = np.shape(d["image"])
        cap = int(d.get("max_keypoints", min_capacity(w, h, keypoint_distance)))
        if cap < min_capacity(w, h, keypoint_distance):
            raise ValueError(f"slot {slot}: max_keypoints {cap} below {min_capacity(w, h, keypoint_distance)}")


def pack_frames(frames, keypoint_distance):
    """The pvio_b200_feature_frame array of a call and its outputs: (array, outputs per frame, arrays to keep alive)."""
    n = len(frames)
    cf = (_lib.CFeatureFrame * max(n, 1))()
    outs, keep = [], []
    for i, d in enumerate(frames):
        img = np.ascontiguousarray(d["image"], dtype=np.uint8)
        h, w = img.shape
        cap = int(d.get("max_keypoints", min_capacity(w, h, keypoint_distance)))
        K = d["K"]
        q = d.get("predict_q")
        q = None if q is None else np.ascontiguousarray(q, dtype=np.float64).reshape(4)
        kp = np.zeros((max(cap, 1), 2))
        prev = np.zeros(max(cap, 1), dtype=np.int32)
        cnt = np.zeros(9, dtype=np.int32)              # n_keypoints, counts[4], info[4]
        c = cf[i]
        c.slot, c.width, c.height, c.stride = int(d["slot"]), w, h, w
        c.frame_id = int(d["frame_id"])
        c.fx, c.fy, c.cx, c.cy = (float(v) for v in K)
        c.map_frames, c.max_keypoints = int(d["map_frames"]), cap
        _lib.set_ptrs(c, image=img, predict_q=q, keypoints=kp, prev_index=prev, n_keypoints=cnt[:1], counts=cnt[1:5],
                      info=cnt[5:])
        keep += [img, q, kp, prev, cnt]
        outs.append((kp, prev, cnt))
    return cf, outs, keep


def batch_feature_track(ba, frames, keypoint_distance=20.0, max_level=3, max_iter=30, eps=0.01, clahe_clip=6.0,
                        clahe_tiles=(8, 8), border=20, ransac_threshold=1.0, ransac_confidence=0.99):
    """ba: a BundleAdjustor (owns the device handle).  frames: one dict per sequence with slot (a tracker slot,
    distinct within the call), frame_id (!= 0), image (uint8 [h, w], raw), K (fx, fy, cx, cy), map_frames (the map's
    frame count before this frame; 0 starts the sequence), optionally predict_q (x, y, z, w: delta_key_q of
    frame.cpp:98; None: no prediction) and max_keypoints (default min_capacity).
    Returns one dict per frame: keypoints (float64 [m, 2], normalised), prev_index (int32 [m], -1: new), counts
    (kept after LK and border, after F-RANSAC, after the thinning, detected) and info (as batch_track_keypoints')."""
    check_frames(frames, keypoint_distance)
    cf, outs, keep = pack_frames(frames, keypoint_distance)
    ba._ck(ba.lib.pvio_b200_batch_feature_track(ba.h, len(frames), cf, int(max_level), int(max_iter), float(eps),
                                                float(clahe_clip), int(clahe_tiles[0]), int(clahe_tiles[1]), int(border),
                                                float(ransac_threshold), float(ransac_confidence),
                                                float(keypoint_distance)))
    del keep
    res = []
    for kp, prev, cnt in outs:
        m = int(cnt[0])
        res.append({"keypoints": kp[:m].copy(), "prev_index": prev[:m].copy(), "counts": cnt[1:5].copy(),
                    "info": cnt[5:].copy()})
    return res
