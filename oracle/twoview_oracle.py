"""TEST INFRASTRUCTURE (CPU oracle) -- the two-view step of Initializer::init_sfm
(pvio/src/pvio/core/initializer.cpp:102-161), restated in NumPy fp64 from the algorithms:

- the sample schedule of Ransac::solve (utility/ransac.h, utility/random.h): a LotBox over libstdc++'s
  std::default_random_engine (minstd_rand0) and std::uniform_int_distribution<size_t>;
- solve_homography_4pt (geometry/homography.cpp:99-166) and solve_essential_5pt (essential.cpp:114-288), with the
  symmetric transfer / epipolar errors of find_homography_matrix and find_essential_matrix (stereo.cpp:36-80);
- the serial Ransac::solve loop itself (not a replay of precomputed counts);
- decompose_homography (homography.cpp:22-91), decompose_essential in its SVD form (essential.cpp:259-274);
- triangulate_from_rt_scored over the 8 pose candidates (stereo.cpp:123-171) and init_sfm's gates.

Conventions shared with the device (pvio_b200/csrc/twoview.cu), where the reference leaves them to Eigen:
- null spaces from a Householder QR of the transposed system (fixes the sign of H and of the E basis);
- the real solutions of one 5-point problem in ascending order of their action-matrix eigenvalue;
- 3 x 3 SVDs by one-sided Jacobi, U's third column u0 x u1 for an essential matrix; its decomposition's translation
  has its component of largest magnitude positive, and R1 is the rotation of larger trace.
Eigenpairs come from LAPACK (numpy.linalg.eig), an independent route from the device's own QR iteration."""
import math

import numpy as np

from . import tri_oracle

MINSTD_M = 2147483647
STATUS_OK, STATUS_FEW_MATCHES, STATUS_LOW_PARALLAX, STATUS_PURE_ROTATION, STATUS_FEW_TRIANGULATED = range(5)


# ---- the sample schedule -------------------------------------------------------------------------------------------
class Minstd:
    """std::minstd_rand0 seeded through an unsigned int."""

    def __init__(self, seed):
        s = (int(seed) & 0xFFFFFFFF) % MINSTD_M
        self.x = s if s else 1

    def __call__(self):
        self.x = self.x * 16807 % MINSTD_M
        return self.x


def uniform_index(g, a, b):
    """std::uniform_int_distribution<size_t>(a, b)(g), a < b: libstdc++'s downscaling branch."""
    urngrange = MINSTD_M - 2
    uerange = b - a + 1
    scaling = urngrange // uerange
    past = uerange * scaling
    while True:
        r = g() - 1
        if r < past:
            return a + r // scaling


def lotbox_schedule(n, seed, dof, iters):
    """[iters][dof] indices: a fresh LotBox of n lots seeded with seed, refill_all before every iteration."""
    lots = list(range(n))
    g = Minstd(seed)
    out = np.zeros((iters, dof), dtype=np.int32)
    for it in range(iters):
        cap = 0
        for s in range(dof):
            if n - cap > 1:
                j = uniform_index(g, cap, n - 1)
                lots[cap], lots[j] = lots[j], lots[cap]
                out[it, s] = lots[cap]
            else:
                out[it, s] = lots[n - 1]
            cap += 1
    return out


# ---- shared linear algebra -----------------------------------------------------------------------------------------
def householder_null(M):
    """Columns C .. 8 of Q for the Householder QR of the 9 x C matrix M: an orthonormal basis of null(M^T), [9 - C][9]."""
    M = np.array(M, dtype=np.float64)
    C = M.shape[1]
    V, beta = [], []
    for k in range(C):
        x = M[k:, k]
        nrm = math.sqrt(float(np.dot(x, x)))
        alpha = -nrm if x[0] >= 0 else nrm
        v = x.copy()
        v[0] = x[0] - alpha
        vv = float(np.dot(v, v))
        b = 2.0 / vv if vv > 0 else 0.0
        M[k:, k:] -= np.outer(v, b * (v @ M[k:, k:]))
        V.append(v)
        beta.append(b)
    out = np.zeros((9 - C, 9))
    for q in range(C, 9):
        f = np.zeros(9)
        f[q] = 1.0
        for k in range(C - 1, -1, -1):
            f[k:] -= beta[k] * np.dot(V[k], f[k:]) * V[k]
        out[q - C] = f
    return out


def to_matrix(v):
    """The reference's to_matrix: its segments are the COLUMNS, M(k, j) = v[3 j + k]."""
    return np.asarray(v, dtype=np.float64).reshape(3, 3).T


def svd3(M, rank2=False):
    """One-sided Jacobi SVD of a 3 x 3 matrix: (s descending, U, V), M = U diag(s) V^T."""
    a = np.array(M, dtype=np.float64).T.copy()               # a[c] = column c
    v = np.eye(3)
    for _ in range(40):
        rotated = False
        for p, q in ((0, 1), (0, 2), (1, 2)):
            alpha, beta, gamma = a[p] @ a[p], a[q] @ a[q], a[p] @ a[q]
            if abs(gamma) <= 1e-15 * math.sqrt(alpha * beta):
                continue
            rotated = True
            zeta = (beta - alpha) / (2 * gamma)
            t = (1.0 if zeta >= 0 else -1.0) / (abs(zeta) + math.sqrt(1 + zeta * zeta))
            c = 1 / math.sqrt(1 + t * t)
            s = c * t
            a[p], a[q] = c * a[p] - s * a[q], s * a[p] + c * a[q]
            v[p], v[q] = c * v[p] - s * v[q], s * v[p] + c * v[q]
        if not rotated:
            break
    sig = np.sqrt(np.einsum("ij,ij->i", a, a))
    o = sorted(range(3), key=lambda i: -sig[i])              # stable: ties keep column order
    with np.errstate(all="ignore"):                          # an exactly singular matrix: its column 2 is 0
        U = np.stack([a[i] / sig[i] for i in o], axis=1)
    if rank2:
        U[:, 2] = np.cross(U[:, 0], U[:, 1])
    return sig[o], U, np.stack([v[i] for i in o], axis=1)


# ---- homography ----------------------------------------------------------------------------------------------------
def homography_4pt(a, b):
    """solve_homography_4pt: H with b ~ H a for the 4 matches a[4][2], b[4][2]."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    ma, mb = a.mean(axis=0), b.mean(axis=0)
    sa = 1.0 / (math.sqrt(2.0) * np.sum(np.linalg.norm(a - ma, axis=1)))
    sb = 1.0 / (math.sqrt(2.0) * np.sum(np.linalg.norm(b - mb, axis=1)))
    na, nb = (a - ma) * sa, (b - mb) * sb
    A = np.zeros((8, 9))
    for i in range(4):
        (a0, a1), (b0, b1) = na[i], nb[i]
        A[2 * i, [1, 2, 4, 5, 7, 8]] = [-a0, a0 * b1, -a1, a1 * b1, -1, b1]
        A[2 * i + 1, [0, 2, 3, 5, 6, 8]] = [a0, -a0 * b0, a1, -a1 * b0, 1, -b0]
    NH = to_matrix(householder_null(A.T)[0])
    Nb = np.array([[1 / sb, 0, mb[0]], [0, 1 / sb, mb[1]], [0, 0, 1]])
    Na = np.array([[sa, 0, -sa * ma[0]], [0, sa, -sa * ma[1]], [0, 0, 1]])
    return Nb @ NH @ Na


def h_error(H, p1, p2):
    """homography_geometric_error(H, p1, p2) for every match."""
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    u = (H[0, 0] * x1 + H[0, 1] * y1) + H[0, 2]
    v = (H[1, 0] * x1 + H[1, 1] * y1) + H[1, 2]
    w = (H[2, 0] * x1 + H[2, 1] * y1) + H[2, 2]
    with np.errstate(all="ignore"):
        return (x2 - u / w) ** 2 + (y2 - v / w) ** 2


def e_error(E, p1, p2):
    """essential_geometric_error(E, p1, p2) for every match."""
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    a = (E[0, 0] * x1 + E[0, 1] * y1) + E[0, 2]
    b = (E[1, 0] * x1 + E[1, 1] * y1) + E[1, 2]
    c = (E[2, 0] * x1 + E[2, 1] * y1) + E[2, 2]
    r = (x2 * a + y2 * b) + c
    with np.errstate(all="ignore"):
        return r * r / (a * a + b * b)


def homography_errors(H, p1, p2):
    with np.errstate(all="ignore"):
        Hinv = np.linalg.inv(H) if np.all(np.isfinite(H)) else np.full((3, 3), np.nan)
    return h_error(H, p1, p2) + h_error(Hinv, p2, p1)


def essential_errors(E, p1, p2):
    return e_error(E, p1, p2) + e_error(E.T, p2, p1)


# ---- the 5-point solver --------------------------------------------------------------------------------------------
# monomials xxx xxy xyy yyy xxz xyz yyz xzz yzz zzz | xx xy yy xz yz zz | x y z | 1
MONO = [(3, 0, 0), (2, 1, 0), (1, 2, 0), (0, 3, 0), (2, 0, 1), (1, 1, 1), (0, 2, 1), (1, 0, 2), (0, 1, 2), (0, 0, 3),
        (2, 0, 0), (1, 1, 0), (0, 2, 0), (1, 0, 1), (0, 1, 1), (0, 0, 2), (1, 0, 0), (0, 1, 0), (0, 0, 1), (0, 0, 0)]
XX, X, Y, Z, ONE = 10, 16, 17, 18, 19
_PAIRS = [(MONO.index(tuple(p + q for p, q in zip(MONO[a], MONO[b]))), a, b)
          for a in range(20) for b in range(20) if sum(MONO[a]) + sum(MONO[b]) <= 3]
_PO, _PA, _PB = (np.array(c) for c in zip(*_PAIRS))


def poly_mul(a, b):
    """Product of two polynomials, truncated at degree 3."""
    r = np.zeros(20)
    np.add.at(r, _PO, a[_PA] * b[_PB])
    return r


def essential_5pt(a, b):
    """solve_essential_5pt on the 5 matches a[5][2], b[5][2].  Returns (models [k][3][3] in ascending eigenvalue
    order, borderline) -- borderline: an eigenvalue with 1e-11 < |imag| < 1e-9, where the 1e-10 filter is fragile."""
    ah = np.c_[np.asarray(a, dtype=np.float64), np.ones(5)]
    bh = np.c_[np.asarray(b, dtype=np.float64), np.ones(5)]
    A = np.stack([np.outer(ah[i], bh[i]).reshape(9) for i in range(5)])     # A(i, 3 j + m) = a_j b_m
    basis = householder_null(A.T)                                           # [4][9]
    Eb = [to_matrix(basis[c]) for c in range(4)]
    Ep = np.zeros((3, 3, 20))
    Ep[:, :, X], Ep[:, :, Y], Ep[:, :, Z], Ep[:, :, ONE] = Eb
    EEt = np.array([[sum((poly_mul(Ep[i, c], Ep[j, c]) for c in range(3)), np.zeros(20)) for j in range(3)]
                    for i in range(3)])
    half_tr = 0.5 * (EEt[0, 0] + EEt[1, 1] + EEt[2, 2])
    P = np.zeros((10, 20))
    for i in range(3):
        for j in range(3):
            P[3 * i + j] = (sum((poly_mul(EEt[i, c], Ep[c, j]) for c in range(3)), np.zeros(20)) -
                            poly_mul(half_tr, Ep[i, j]))
    for c in range(3):
        c1, c2 = (c + 1) % 3, (c + 2) % 3
        P[9] += poly_mul(Ep[0, c], poly_mul(Ep[1, c1], Ep[2, c2]) - poly_mul(Ep[1, c2], Ep[2, c1]))
    # Gauss-Jordan with the reference's pivot order
    perm = list(range(10))
    for i in range(10):
        for j in range(i + 1, 10):
            if abs(P[perm[i], i]) < abs(P[perm[j], i]):
                perm[i], perm[j] = perm[j], perm[i]
        if P[perm[i], i] == 0:
            continue
        P[perm[i]] /= P[perm[i], i]
        for j in range(i + 1, 10):
            P[perm[j]] -= P[perm[i]] * P[perm[j], i]
    for i in range(9, 0, -1):
        for j in range(i):
            P[perm[j]] -= P[perm[i]] * P[perm[j], i]
    act = np.zeros((10, 10))
    for r, m in enumerate((0, 1, 2, 4, 5, 7)):                              # xxx xxy xyy xxz xyz xzz
        act[r] = -P[perm[m], XX:]
    for r, u in enumerate((0, 1, 3, 6)):                                    # xx xy xz x
        act[6 + r, u] = 1.0
    if not np.all(np.isfinite(act)):
        return [], False
    w, V = np.linalg.eig(act)
    borderline = bool(np.any((np.abs(w.imag) > 1e-11) & (np.abs(w.imag) < 1e-9)))
    real = sorted((i for i in range(10) if abs(w[i].imag) < 1e-10), key=lambda i: w[i].real)
    models = []
    for i in real:
        h = V[:, i].real
        x, y, z = h[X - XX] / h[ONE - XX], h[Y - XX] / h[ONE - XX], h[Z - XX] / h[ONE - XX]
        models.append(to_matrix(basis.T @ np.array([x, y, z, 1.0])))
    return models, borderline


# ---- Ransac::solve -------------------------------------------------------------------------------------------------
def thresholds(fx):
    thr = 0.7 / fx
    return 2.0 * 5.99 * thr * thr, 2.0 * 3.84 * thr * thr


def iteration(kind, p1, p2, idx, thr):
    """One iteration's hypotheses: (models, masks, borderline).  kind 'H' or 'E'."""
    a, b = p1[idx], p2[idx]
    if kind == "H":
        models, border = [homography_4pt(a, b)], False
        errs = [homography_errors(models[0], p1, p2)]
    else:
        models, border = essential_5pt(a, b)
        errs = [essential_errors(E, p1, p2) for E in models]
    masks = [e <= thr for e in errs]
    for e in errs:
        with np.errstate(invalid="ignore"):
            border |= bool(np.any(np.abs(e - thr) <= 1e-9 * thr))
    return models, masks, border


def ransac(kind, p1, p2, thr, confidence=0.999, max_iteration=1000, seed=648, schedule=None):
    """Ransac::solve, serially: draw, solve, count each model, accept a strictly better one and shrink the budget with
    pow(ratio, 5) (for both models, as the reference).  Returns a dict: model, inliers, mask, iterations (run),
    best_it, best_k, counts (per iteration run: [model count, each model's inliers])."""
    n = len(p1)
    dof = 4 if kind == "H" else 5
    if schedule is None:
        schedule = lotbox_schedule(n, seed, dof, max_iteration)
    K = math.log(max(1 - confidence, 1.0e-5))
    res = dict(model=np.zeros((3, 3)), inliers=0, mask=np.zeros(n, dtype=bool), iterations=0, best_it=-1, best_k=-1,
               counts=[])
    iter_max, it = max_iteration, 0
    while it < iter_max:
        models, masks, _ = iteration(kind, p1, p2, schedule[it], thr)
        res["counts"].append([len(models)] + [int(m.sum()) for m in masks])
        for k, (M, mask) in enumerate(zip(models, masks)):
            c = int(mask.sum())
            if c > res["inliers"]:
                res.update(model=M, inliers=c, mask=mask, best_it=it, best_k=k)
                ratio = c / float(n)
                with np.errstate(divide="ignore"):
                    N = K / math.log(1 - math.pow(ratio, 5)) if ratio < 1 else 0.0
                if N < iter_max:
                    iter_max = int(math.ceil(N))
        it += 1
    res["iterations"] = it
    return res


# ---- decompositions ------------------------------------------------------------------------------------------------
def normalized(t):
    q = float(t @ t)
    return t / math.sqrt(q) if q > 0 else t


def decompose_homography(H):
    """Returns (ok, R1, R2, T1, T2); ok False for a pure rotation."""
    s, U, V = svd3(H)
    Hn = H / s[1]
    S = Hn.T @ Hn - np.eye(3)
    if np.all(np.abs(S) <= 1e-3):
        R = U @ V.T
        if np.linalg.det(R) < 0:
            R = -R
        return False, R, R.copy(), np.zeros(3), np.zeros(3)
    ms00 = S[1, 2] ** 2 - S[1, 1] * S[2, 2]
    ms11 = S[0, 2] ** 2 - S[0, 0] * S[2, 2]
    ms22 = S[0, 1] ** 2 - S[0, 0] * S[1, 1]
    with np.errstate(invalid="ignore"):
        r00, r11, r22 = np.sqrt(ms00), np.sqrt(ms11), np.sqrt(ms22)
        nu = 2.0 * np.sqrt(1 + np.trace(S) - ms00 - ms11 - ms22)
    tenormsq = 2 + np.trace(S) - nu
    if S[0, 0] > S[1, 1] and S[0, 0] > S[2, 2]:
        e = -1 if S[0, 1] * S[0, 2] - S[0, 0] * S[1, 2] < 0 else 1
        n1 = np.array([S[0, 0], S[0, 1] + r22, S[0, 2] + e * r11])
        n2 = np.array([S[0, 0], S[0, 1] - r22, S[0, 2] - e * r11])
        d = S[0, 0]
    elif S[1, 1] > S[0, 0] and S[1, 1] > S[2, 2]:
        e = -1 if S[1, 1] * S[0, 2] - S[0, 1] * S[1, 2] < 0 else 1
        n1 = np.array([S[0, 1] + r22, S[1, 1], S[1, 2] - e * r00])
        n2 = np.array([S[0, 1] - r22, S[1, 1], S[1, 2] + e * r00])
        d = S[1, 1]
    else:
        e = -1 if S[1, 2] * S[0, 2] - S[0, 1] * S[2, 2] < 0 else 1
        n1 = np.array([S[0, 2] + e * r11, S[1, 2] + r00, S[2, 2]])
        n2 = np.array([S[0, 2] - e * r11, S[1, 2] - r00, S[2, 2]])
        d = S[2, 2]
    t1 = np.linalg.norm(n1) * n2 / d
    t2 = np.linalg.norm(n2) * n1 / d
    n1, n2 = normalized(n1), normalized(n2)
    t1 = t1 - tenormsq * n1
    t2 = t2 - tenormsq * n2
    R1 = Hn @ (np.eye(3) - np.outer(t1 / nu, n1))
    R2 = Hn @ (np.eye(3) - np.outer(t2 / nu, n2))
    return True, R1, R2, R1 @ (0.5 * t1), R2 @ (0.5 * t2)


def decompose_essential(E):
    """The SVD form: (R1, R2, T) with T's component of largest magnitude positive and R1 the rotation of larger trace
    (the two equal singular values of an essential matrix leave the SVD's order of u0 and u1, and with it the sign of T
    and the order of R1 and R2, to rounding)."""
    _, U, V = svd3(E, rank2=True)
    VT = V.T
    if np.linalg.det(U) < 0:
        U = -U
    if np.linalg.det(VT) < 0:
        VT = -VT
    W = np.array([[0, 1, 0], [-1, 0, 0], [0, 0, 1.0]])
    R1, R2, T = U @ W @ VT, U @ W.T @ VT, U[:, 2].copy()
    m = int(np.argmax(np.abs(T)))
    if T[m] < 0:
        T = -T
    if (R2[0, 0] + R2[1, 1]) + R2[2, 2] > (R1[0, 0] + R1[1, 1]) + R1[2, 2]:
        R1, R2 = R2, R1
    return R1, R2, T


# ---- the scored triangulation and the selection --------------------------------------------------------------------
def triangulate_rt_scored(p1, p2, R, T):
    """triangulate_from_rt_scored for one candidate: (count, mean score, points [n][3] (0 where it failed), status)."""
    P1 = np.c_[np.eye(3), np.zeros(3)]
    P2 = np.c_[R, T]
    n = len(p1)
    pts, st, total = np.zeros((n, 3)), np.zeros(n, dtype=bool), 0.0
    for i in range(n):
        ok, p, score = tri_oracle.triangulate_scored([P1, P2], [p1[i], p2[i]])
        if ok:
            pts[i], st[i] = p, True
            total += score
    cnt = int(st.sum())
    return cnt, total / max(cnt, 1), pts, st


def select_candidate(counts, scores, count_threshold):
    """stereo.cpp:155-163: a candidate with more than count_threshold points and a lower mean score than the current
    best wins -- compared against the best's score even while the best's own count is below the threshold --
    otherwise one with more points."""
    best = 0
    for i in range(len(counts)):
        if counts[i] > count_threshold and scores[i] < scores[best]:
            best = i
        elif counts[i] > counts[best]:
            best = i
    return best


def two_view(p1, p2, fx, fy, min_matches=50, min_parallax=10.0, min_triangulation=20, seed=648, confidence=0.999,
             max_iteration=1000):
    """init_sfm's two-view step as pvio_b200_batch_two_view computes it: the status is init_sfm's first early return
    that applies, and the RANSACs and the triangulation run whatever the gates say (except below 5 matches)."""
    p1 = np.ascontiguousarray(p1, dtype=np.float64).reshape(-1, 2)
    p2 = np.ascontiguousarray(p2, dtype=np.float64).reshape(-1, 2)
    n = len(p1)
    d = np.stack([p1[:, 0] * fx - p2[:, 0] * fx, p1[:, 1] * fy - p2[:, 1] * fy], 1)
    par = 0.0
    for v in np.sqrt(d[:, 0] ** 2 + d[:, 1] ** 2):
        par += v
    par /= max(n, 1)
    out = dict(parallax=par, candidate=-1, triangulated=0, R=np.eye(3), T=np.zeros(3), points=np.zeros((n, 3)),
               point_status=np.zeros(n, dtype=bool), h=None, e=None)
    if n < 5:
        out["status"] = STATUS_FEW_MATCHES
        return out
    thr_h, thr_e = thresholds(fx)
    h = ransac("H", p1, p2, thr_h, confidence, max_iteration, seed)
    e = ransac("E", p1, p2, thr_e, confidence, max_iteration, seed)
    out["h"], out["e"] = h, e
    ok, RH1, RH2, TH1, TH2 = decompose_homography(h["model"])
    TH1, TH2 = normalized(TH1), normalized(TH2)
    RE1, RE2, TE = decompose_essential(e["model"])
    TE = normalized(TE)
    Rs = [RH1, RH1, RH2, RH2, RE1, RE1, RE2, RE2]
    Ts = [TH1, -TH1, TH2, -TH2, TE, -TE, TE, -TE]
    tri = [triangulate_rt_scored(p1, p2, R, T) for R, T in zip(Rs, Ts)]
    best = select_candidate([t[0] for t in tri], [t[1] for t in tri], min_triangulation)
    out.update(candidate=best, triangulated=tri[best][0], R=Rs[best], T=Ts[best], points=tri[best][2],
               point_status=tri[best][3], counts=[t[0] for t in tri], scores=[t[1] for t in tri])
    if n < min_matches:
        out["status"] = STATUS_FEW_MATCHES
    elif par < min_parallax:
        out["status"] = STATUS_LOW_PARALLAX
    elif not ok:
        out["status"] = STATUS_PURE_ROTATION
    elif tri[best][0] < min_triangulation:
        out["status"] = STATUS_FEW_TRIANGULATED
    else:
        out["status"] = STATUS_OK
    return out
