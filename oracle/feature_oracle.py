"""TEST INFRASTRUCTURE ONLY.  CPU statement of the per-frame step of FeatureTracker::work (feature_tracker.cpp:77-99):
Frame::track_keypoints of the previous frame into the new one (frame.cpp:88-138) and Frame::detect_keypoints
(frame.cpp:72-86).
  * the guesses: apply_k(z) and apply_k(hnormalized(q [z; 1])) in float64 (numpy does not contract), q * v as Eigen's
    Quaternion::_transformVector;
  * LK, the border test and findFundamentalMat are the reference's own dependency, cv2 (opencv_image.cpp:88-136);
  * the thinning sorts with libstdc++'s std::sort itself (oracle/sort_helper.cpp, compiled on first use) and filters
    with detect_oracle.PoissonDiskFilter; keypoints detected in the previous frame have no track and skip it;
  * the detector is detect_oracle.detect_keypoints (cv2.goodFeaturesToTrack and the same filter)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import detect_oracle

_HERE = os.path.dirname(os.path.abspath(__file__))
_CSRC = os.path.join(os.path.dirname(_HERE), "pvio_b200", "csrc")
_lib = None


def sort_helper():
    """The compiled sort helper (std::sort and the restated introsort), built into a temporary directory."""
    global _lib
    if _lib is not None:
        return _lib
    src = os.path.join(_HERE, "sort_helper.cpp")
    hdr = os.path.join(_CSRC, "introsort.cuh")
    tag = hashlib.sha1(open(src, "rb").read() + open(hdr, "rb").read()).hexdigest()[:12]
    so = os.path.join(tempfile.gettempdir(), f"pvio_sort_helper_{os.getuid()}_{tag}.so")
    if not os.path.exists(so):
        tmp = so + f".{os.getpid()}"
        subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-DWITH_RESTATED", "-I", _CSRC, "-o", tmp, src],
                       check=True)
        os.replace(tmp, so)
    lib = C.CDLL(so)
    for name in ("std_sort_by_length", "restated_sort_by_length"):
        getattr(lib, name).argtypes = [C.c_int] + [C.POINTER(C.c_int32)] * 3
    _lib = lib
    return lib


def _sort(name, index, length):
    index = np.ascontiguousarray(index, dtype=np.int32)
    length = np.ascontiguousarray(length, dtype=np.int32)
    out = np.zeros(max(len(index), 1), dtype=np.int32)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))
    getattr(sort_helper(), name)(len(index), p(index), p(length), p(out))
    return out[:len(index)]


def std_sort_by_length(index, length):
    """The keypoint indices in the order std::sort leaves the (index, length) pairs, longer tracks first."""
    return _sort("std_sort_by_length", index, length)


def restated_sort_by_length(index, length):
    """The same through the restated introsort (pvio_b200/csrc/introsort.cuh) compiled for the host."""
    return _sort("restated_sort_by_length", index, length)


def apply_k(z, K):
    fx, fy, cx, cy = K
    z = np.asarray(z, dtype=np.float64).reshape(-1, 2)
    return np.stack([z[:, 0] * fx + cx, z[:, 1] * fy + cy], 1)


def remove_k(p, K):
    fx, fy, cx, cy = K
    p = np.asarray(p, dtype=np.float64).reshape(-1, 2)
    return np.stack([(p[:, 0] - cx) / fx, (p[:, 1] - cy) / fy], 1)


def qrot(q, v):
    """Eigen's q * v: uv = 2 (q.vec x v); v + w uv + q.vec x uv, evaluated left to right"""
    x, y, z, w = q
    v0, v1, v2 = v[:, 0], v[:, 1], v[:, 2]
    tx, ty, tz = 2.0 * (y * v2 - z * v1), 2.0 * (z * v0 - x * v2), 2.0 * (x * v1 - y * v0)
    return np.stack([v0 + w * tx + (y * tz - z * ty), v1 + w * ty + (z * tx - x * tz), v2 + w * tz + (x * ty - y * tx)], 1)


def guesses(z, K_prev, K_next, q):
    """frame.cpp:90-103: (LK input, initial guess) as float32 [n, 2]; q None: the guess is the input"""
    z = np.asarray(z, dtype=np.float64).reshape(-1, 2)
    prev = apply_k(z, K_prev).astype(np.float32)
    if q is None:
        return prev, prev.copy()
    y = qrot(q, np.concatenate([z, np.ones((len(z), 1))], 1))
    return prev, apply_k(np.stack([y[:, 0] / y[:, 2], y[:, 1] / y[:, 2]], 1), K_next).astype(np.float32)


def thin(next_pts, status, has_track, length, keypoint_distance):
    """frame.cpp:108-130: the status after the track-length-ordered Poisson-disk thinning"""
    status = np.asarray(status, dtype=bool).copy()
    idx = np.nonzero(status & np.asarray(has_track, dtype=bool))[0]
    order = std_sort_by_length(idx, np.asarray(length)[idx])
    f = detect_oracle.PoissonDiskFilter(keypoint_distance)
    for k in order:
        p = (float(next_pts[k][0]), float(next_pts[k][1]))
        if not f.insert(p):
            status[k] = False
    return status


def step(prev_eq, next_eq, z, prev_index, birth, prev_no, map_frames, K_prev, K_next, q, keypoint_distance):
    """One frame of a sequence: prev_eq / next_eq the equalised frames (prev_eq None: a new sequence), z the previous
    frame's keypoints (normalised), prev_index / birth theirs.  Returns (z, prev_index, birth, counts) of the new
    frame; births count in frame numbers, the new frame is prev_no + 1."""
    import cv2
    z = np.asarray(z, dtype=np.float64).reshape(-1, 2)
    h, w = next_eq.shape
    counts = [0, 0, 0, 0]
    new_z, new_prev, new_birth = [], [], []
    if prev_eq is not None and len(z):
        p0, p1 = guesses(z, K_prev, K_next, q)
        p1, st, _ = cv2.calcOpticalFlowPyrLK(prev_eq, next_eq, p0.reshape(-1, 1, 2), p1.reshape(-1, 1, 2).copy(),
                                             winSize=(21, 21), maxLevel=3,
                                             criteria=(cv2.TERM_CRITERIA_COUNT + cv2.TERM_CRITERIA_EPS, 30, 0.01),
                                             flags=cv2.OPTFLOW_USE_INITIAL_FLOW)
        p1 = p1.reshape(-1, 2)
        st = st.reshape(-1).astype(bool)
        st &= ~((p1[:, 0] < 20) | (p1[:, 0] >= w - 20) | (p1[:, 1] < 20) | (p1[:, 1] >= h - 20))
        counts[0] = int(st.sum())
        l = np.nonzero(st)[0]
        if len(l) >= 8:
            _, mask = cv2.findFundamentalMat(p0[l], p1[l], cv2.FM_RANSAC, 1.0, 0.99)
            st[l if mask is None else l[mask.reshape(-1) == 0]] = False      # no model: the mask is all zero
        counts[1] = int(st.sum())
        has_track = np.asarray(prev_index) != -1
        length = np.minimum(prev_no - np.asarray(birth) + 1, map_frames)
        st = thin(p1, st, has_track, length, keypoint_distance)
        counts[2] = int(st.sum())
        for k in np.nonzero(st)[0]:
            new_z.append(remove_k(p1[k].astype(np.float64), K_next)[0])
            new_prev.append(int(k))
            new_birth.append(int(birth[k]))
    existing = apply_k(np.array(new_z).reshape(-1, 2), K_next)
    det = detect_oracle.detect_keypoints(next_eq, existing, keypoint_distance)
    counts[3] = len(det)
    for p in det:
        new_z.append(remove_k(p, K_next)[0])
        new_prev.append(-1)
        new_birth.append(prev_no + 1)
    return np.array(new_z).reshape(-1, 2), np.array(new_prev, dtype=np.int32), np.array(new_birth, dtype=np.int32), counts
