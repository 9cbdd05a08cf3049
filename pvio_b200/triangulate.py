"""Host-side mirror of Track::triangulate (pvio/src/pvio/map/track.cpp:83-106) over the C ABI: a batch of tracks."""
import numpy as np

from . import _lib


def triangulate(ba, P, begin, obs_frame, obs_z):
    """P: [F][3][4] camera matrices; begin: [T+1]; obs_frame: [K]; obs_z: [K][2].
    Returns (points [T][3], valid [T] bool, score [T])."""
    P = np.ascontiguousarray(P, dtype=np.float64).reshape(-1, 12)
    begin = np.ascontiguousarray(begin, dtype=np.int32)
    fr = np.ascontiguousarray(obs_frame, dtype=np.int32)
    z = np.ascontiguousarray(obs_z, dtype=np.float64).reshape(-1, 2)
    n = len(begin) - 1
    pts, valid, score = np.zeros((n, 3)), np.zeros(n, dtype=np.uint8), np.zeros(n)
    ba._ck(ba.lib.pvio_b200_triangulate(ba.h, len(P), _lib.ptr(P), n, _lib.ptr(begin), _lib.ptr(fr), _lib.ptr(z),
                                        _lib.ptr(pts), _lib.ptr(valid), _lib.ptr(score)))
    return pts, valid.astype(bool), score
