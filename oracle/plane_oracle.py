"""TEST INFRASTRUCTURE (CPU oracle) -- plane detection of PVIO, restated in NumPy fp64 from the algorithms:

- PlaneExtractor::work (pvio/src/pvio/core/plane_extractor.cpp:40-81): Ransac<3, PlaneState, PlaneSolver,
  PlaneEvaluator> with threshold 0.03 over the landmark points, then the inliers' centroid, covariance and the
  eigenvector of its smallest eigenvalue;
- Plane::update_parameter(true) (map/plane.cpp:64-114): the same over Track::try_triangulate of each track's window
  observations, threshold 0.05, no RANSAC below 50 points;
- PlaneSolver (plane_extractor.h): n = (p2 - p0) x (p1 - p0), Eigen's stableNormalize, d = p0 . n; PlaneEvaluator:
  |p . n - d|;
- the serial Ransac::solve loop itself (ransac.h:43-97, not a replay of precomputed counts), with the sample schedule of
  twoview_oracle.lotbox_schedule at seed 0;
- PlaneExtractor::enough_baseline and Track::compute_baseline (track.cpp:125-135).

Sums follow the reference's order: dot products ((x + y) + z), the centroid and covariance serially in point order.
The two deviations of the device (DESIGN 4.7g), followed here too: the refined normal's sign is fixed (d >= 0, and the
component of largest magnitude positive when d == 0), and a refit track whose triangulation fails is left out."""
import math

import numpy as np

from . import tri_oracle
from .twoview_oracle import lotbox_schedule

EXTRACT, REFIT = 0, 1
ACCEPTED, FEW_POINTS, REJECTED = 0, 1, 2
THRESHOLD = {EXTRACT: 0.03, REFIT: 0.05}
MIN_POINTS = {EXTRACT: 3, REFIT: 50}
CONFIDENCE, MAX_ITERATION, SEED, MIN_INLIERS = 0.999, 1000, 0, 31


def dot3(a, b):
    return (float(a[0]) * float(b[0]) + float(a[1]) * float(b[1])) + float(a[2]) * float(b[2])


def stable_normalize(v):
    """Eigen's stableNormalize: w = max |v_i|, z = |v / w|^2, v / (sqrt(z) w) when z > 0 (a zero vector stays zero)"""
    v = [float(x) for x in v]
    w = max(abs(x) for x in v)
    with np.errstate(divide="ignore", invalid="ignore"):
        u = [np.float64(x) / np.float64(w) for x in v]
    z = dot3(u, u)
    if z > 0:
        s = math.sqrt(z) * w
        v = [x / s for x in v]
    return np.array(v)


def plane_solve(p0, p1, p2):
    """PlaneSolver: (normal, distance)"""
    a, b = [float(p2[k]) - float(p0[k]) for k in range(3)], [float(p1[k]) - float(p0[k]) for k in range(3)]
    n = stable_normalize([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])
    return n, dot3(p0, n)


def inlier_mask(points, n, d, thr):
    return np.array([abs(dot3(p, n) - d) <= thr for p in points], dtype=bool)


def ransac(points, thr, schedule=None):
    """Ransac::solve, serially.  Returns a dict: normal, distance (the winner's raw model, NaN without one), inliers,
    mask, iterations (run), best_it (-1: none), counts (per iteration run), schedule."""
    n = len(points)
    res = dict(normal=np.full(3, np.nan), distance=np.nan, inliers=0, mask=np.zeros(n, dtype=bool), iterations=0,
               best_it=-1, counts=[], schedule=None)
    if n < 3:
        return res
    if schedule is None:
        schedule = lotbox_schedule(n, SEED, 3, MAX_ITERATION)
    res["schedule"] = schedule
    K = math.log(max(1 - CONFIDENCE, 1.0e-5))
    iter_max, it = MAX_ITERATION, 0
    while it < iter_max:
        i0, i1, i2 = schedule[it]
        nrm, d = plane_solve(points[i0], points[i1], points[i2])
        mask = inlier_mask(points, nrm, d, thr)
        c = int(mask.sum())
        res["counts"].append(c)
        if c > res["inliers"]:
            res.update(normal=nrm, distance=d, inliers=c, mask=mask, best_it=it)
            ratio = c / float(n)
            with np.errstate(divide="ignore"):
                N = K / math.log(1 - math.pow(ratio, 5)) if ratio < 1 else 0.0
            if N < iter_max:
                iter_max = int(math.ceil(N))
        it += 1
    res["iterations"] = it
    return res


def centroid(points, mask):
    """the inliers' centroid, summed serially in point order, then divided by the count"""
    c = [0.0, 0.0, 0.0]
    for p, m in zip(points, mask):
        if m:
            c = [c[k] + float(p[k]) for k in range(3)]
    cnt = float(int(np.sum(mask)))
    return np.array([x / cnt for x in c])


def covariance(points, mask, cog):
    C = [[0.0] * 3 for _ in range(3)]
    for p, m in zip(points, mask):
        if m:
            dx = [float(p[k]) - float(cog[k]) for k in range(3)]
            for i in range(3):
                for j in range(3):
                    C[i][j] = C[i][j] + dx[i] * dx[j]
    return np.array(C)


def sign_rule(n, cog):
    """the fixed sign of the refined normal: d = n . cog >= 0, and n's component of largest magnitude positive at d == 0"""
    d = dot3(n, cog)
    if d < 0 or (d == 0 and n[int(np.argmax(np.abs(n)))] < 0):
        n = -n
    return n


def refine(points, mask):
    """(normal, distance, reference point) of the inliers: the eigenvector of the covariance's smallest eigenvalue
    (numpy.linalg.eigh) under the sign rule, distance n . cog, reference point cog"""
    cog = centroid(points, mask)
    w, V = np.linalg.eigh(covariance(points, mask, cog))
    n = sign_rule(V[:, 0].copy(), cog)
    return n, dot3(n, cog), cog


def plane_ransac(points, mode):
    """one record of pvio_b200_batch_window_plane_ransac on its used points.  Returns the RANSAC dict plus status and
    plane [7] (normal, distance, reference point; NaN where the call leaves it undefined)."""
    points = np.asarray(points, dtype=np.float64).reshape(-1, 3)
    plane = np.full(7, np.nan)
    if len(points) < MIN_POINTS[mode]:
        r = ransac(points[:0], THRESHOLD[mode])
        r.update(status=FEW_POINTS, plane=plane)
        return r
    r = ransac(points, THRESHOLD[mode])
    if r["inliers"] >= MIN_INLIERS:
        n, d, cog = refine(points, r["mask"])
        plane[:3], plane[3], plane[4:] = n, d, cog
        r.update(status=ACCEPTED, plane=plane)
        return r
    if mode == REFIT:                     # plane.cpp:77 assigns the raw model whatever the count
        plane[:3], plane[3] = r["normal"], r["distance"]
    r.update(status=REJECTED, plane=plane)
    return r


def compute_baseline(positions):
    """Track::compute_baseline: the summed distances between the body positions of consecutive observing frames"""
    b = 0.0
    for a, c in zip(positions[:-1], positions[1:]):
        d = [float(a[k]) - float(c[k]) for k in range(3)]
        b += math.sqrt(dot3(d, d))
    return b


def enough_baseline(positions, inv_depth):
    """PlaneExtractor::enough_baseline"""
    b = compute_baseline(positions)
    return b > 0.5 or (inv_depth < 1 / 0.2 and b * inv_depth > 0.5)


def refit_point(cam_poses, zs):
    """Track::try_triangulate over the track's window views (camera poses (q, p) and keypoints): the point, or None when
    the triangulation fails or there are fewer than two views"""
    if len(zs) < 2:
        return None
    Ps = [tri_oracle.projection_matrix(q, p) for q, p in cam_poses]
    ok, p, _ = tri_oracle.triangulate_scored(Ps, [np.asarray(z, dtype=np.float64) for z in zs])
    return p if ok else None
