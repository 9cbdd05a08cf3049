"""Host mirror of the two-view step of Initializer::init_sfm (pvio/src/pvio/core/initializer.cpp:102-161) over the
C-ABI (pvio_b200_batch_two_view): both RANSACs, both decompositions and the scored choice of pose on the device."""
import numpy as np

from . import _lib

STATUS = {_lib.TWO_VIEW_OK: "ok", _lib.TWO_VIEW_FEW_MATCHES: "few_matches", _lib.TWO_VIEW_LOW_PARALLAX: "low_parallax",
          _lib.TWO_VIEW_PURE_ROTATION: "pure_rotation", _lib.TWO_VIEW_FEW_TRIANGULATED: "few_triangulated"}


def batch_two_view(ba, problems, diagnostics=False):
    """problems: dicts with p1, p2 ([n][2] normalised keypoints of frames i and j), fx, fy, and optional min_matches
    (50), min_parallax (10), min_triangulation (20), seed (648), confidence (0.999), max_iteration (1000).
    Returns one dict per problem: status (a key of STATUS), parallax, H, E, h_inliers, h_iterations, h_best_it,
    e_inliers, e_iterations, e_best_it, e_best_model, candidate, triangulated, R, T, h_mask, e_mask, points,
    point_status; with diagnostics also h_schedule, e_schedule, h_counts, e_counts."""
    n = len(problems)
    recs, keep, outs = (_lib.CTwoView * max(n, 1))(), [], []
    for i, d in enumerate(problems):
        p1 = np.ascontiguousarray(d["p1"], dtype=np.float64).reshape(-1, 2)
        p2 = np.ascontiguousarray(d["p2"], dtype=np.float64).reshape(-1, 2)
        m, it = len(p1), int(d.get("max_iteration", 1000))
        o = dict(info=np.zeros(10, np.int32), parallax=np.zeros(1), H=np.zeros((3, 3)), E=np.zeros((3, 3)),
                 R=np.zeros((3, 3)), T=np.zeros(3), h_mask=np.zeros(m, np.uint8), e_mask=np.zeros(m, np.uint8),
                 points=np.zeros((m, 3)), point_status=np.zeros(m, np.uint8))
        if diagnostics:
            o.update(h_schedule=np.zeros((it, 4), np.int32), e_schedule=np.zeros((it, 5), np.int32),
                     h_counts=np.zeros(it, np.int32), e_counts=np.zeros((it, 11), np.int32))
        r = recs[i]
        r.n_matches, r.seed = m, int(d.get("seed", 648))
        r.fx, r.fy = float(d["fx"]), float(d["fy"])
        r.min_matches, r.min_triangulation = int(d.get("min_matches", 50)), int(d.get("min_triangulation", 20))
        r.min_parallax, r.confidence = float(d.get("min_parallax", 10.0)), float(d.get("confidence", 0.999))
        r.max_iteration = it
        _lib.set_ptrs(r, p1=p1, p2=p2, **o)
        keep += [p1, p2]
        outs.append(o)
    ba._ck(ba.lib.pvio_b200_batch_two_view(ba.h, n, recs))
    del keep
    res = []
    for o in outs:
        info = o.pop("info")
        names = ("status", "h_inliers", "h_iterations", "h_best_it", "e_inliers", "e_iterations", "e_best_it",
                 "e_best_model", "candidate", "triangulated")
        r = {k: int(v) for k, v in zip(names, info)}
        r["parallax"] = float(o.pop("parallax")[0])
        for k in ("h_mask", "e_mask", "point_status"):
            o[k] = o[k].astype(bool)
        r.update(o)
        res.append(r)
    return res


def two_view(ba, p1, p2, fx, fy, **kw):
    """init_sfm's two-view step for one sequence: a batch of one."""
    d = dict(kw, p1=p1, p2=p2, fx=fx, fy=fy)
    diagnostics = d.pop("diagnostics", False)
    return batch_two_view(ba, [d], diagnostics)[0]
