"""TEST INFRASTRUCTURE ONLY -- NumPy restatement of OpenCV's pyramidal Lucas-Kanade tracker.

PVIO's KLT lives in OpenCV (third party, not in /root/reference; pvio-extra/CMakeLists via
depends/CMakeLists.txt:9, version unpinned): call site
pvio-extra/src/pvio/extra/opencv_image.cpp:103
    calcOpticalFlowPyrLK(prevPyr, nextPyr, pts, next, status, err, Size(21,21), level_num(),
                         TermCriteria(COUNT+EPS, 30, 0.01), OPTFLOW_USE_INITIAL_FLOW)
with pyramids from buildOpticalFlowPyramid(image, pyr, Size(21,21), levels, true) (:145).

Restated from OpenCV's published algorithm (modules/video/src/lkpyramid.cpp,
modules/imgproc/src/pyramids.cpp): pyrDown 5x5 [1 4 6 4 1]/16 with BORDER_REFLECT_101 and
(sum+128)>>8 rounding; Scharr derivatives in int16 with REFLECT_101 at the image edge and a
zero (BORDER_CONSTANT) border outside; 14-bit fixed-point bilinear weights; the 5-fraction-bit
patch; minEigThreshold 1e-4; the eps and oscillation stopping rules.
PINNED against cv2.calcOpticalFlowPyrLK (cv2 4.13.0 is installed in this image and on the GPU
box): status flags bit-exact, positions to < 1e-2 px (OpenCV's SIMD float accumulation order
differs from the exact integer sums used here) -- tests/test_klt_oracle.py.
"""
import numpy as np

WIN = 21
W_BITS = 14
FLT_SCALE = np.float32(1.0 / (1 << 20))


def pyr_down(img):
    """cv::pyrDown for 8-bit single channel (BORDER_REFLECT_101)."""
    h, w = img.shape
    oh, ow = (h + 1) // 2, (w + 1) // 2
    k = np.array([1, 4, 6, 4, 1], dtype=np.int32)

    def idx101(i, n):
        i = np.abs(i)
        return np.where(i >= n, 2 * (n - 1) - i, i)
    src = img.astype(np.int32)
    xs = np.arange(ow) * 2
    cols = [idx101(xs + d, w) for d in range(-2, 3)]
    rowf = sum(src[:, c] * kk for c, kk in zip(cols, k))          # h x ow
    ys = np.arange(oh) * 2
    rows = [idx101(ys + d, h) for d in range(-2, 3)]
    out = sum(rowf[r, :] * kk for r, kk in zip(rows, k))
    return ((out + 128) >> 8).astype(np.uint8)


def scharr_deriv(img):
    """calcSharrDeriv: returns int16 [h, w, 2] (dx, dy), REFLECT_101 at the edges."""
    h, w = img.shape
    s = img.astype(np.int32)

    def r101(i, n):
        i = np.abs(i)
        return np.where(i >= n, 2 * (n - 1) - i, i)
    ys = np.arange(h)
    up, dn = s[r101(ys - 1, h)], s[r101(ys + 1, h)]
    t0 = (up + dn) * 3 + s * 10         # vertical smoothing
    t1 = dn - up                        # vertical derivative
    xs = np.arange(w)
    xl, xr = r101(xs - 1, w), r101(xs + 1, w)
    dx = t0[:, xr] - t0[:, xl]
    dy = (t1[:, xr] + t1[:, xl]) * 3 + t1 * 10
    return np.stack([dx, dy], axis=-1).astype(np.int16)


def build_pyramid(img, max_level):
    """buildOpticalFlowPyramid's levels: it halves first and drops the NEW level when it is not larger than the window
    (a 160 x 120 frame keeps 80 x 60 and 40 x 30 and drops 20 x 15)."""
    levels = [np.ascontiguousarray(img, dtype=np.uint8)]
    for _ in range(max_level):
        h, w = levels[-1].shape
        if (w + 1) // 2 <= WIN or (h + 1) // 2 <= WIN:
            break
        levels.append(pyr_down(levels[-1]))
    return levels


def _pad_img(img):
    return np.pad(img, WIN, mode='reflect').astype(np.int32)        # BORDER_REFLECT_101


def _pad_deriv(d):
    return np.pad(d, ((WIN, WIN), (WIN, WIN), (0, 0)), mode='constant').astype(np.int32)


def _cv_round(x):
    return int(np.rint(np.float32(x)))        # cvRound: round half to even (lrint / SSE cvtss2si)


def _weights(a, b):
    one = np.float32(1.0)
    s = np.float32(1 << W_BITS)
    iw00 = _cv_round((one - a) * (one - b) * s)
    iw01 = _cv_round(a * (one - b) * s)
    iw10 = _cv_round((one - a) * b * s)
    iw11 = (1 << W_BITS) - iw00 - iw01 - iw10
    return iw00, iw01, iw10, iw11


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _patch(P, ix, iy, iw, shift):
    """bilinear fixed-point patch WIN x WIN from padded int32 image P at integer top-left (ix,iy)."""
    y0, x0 = iy + WIN, ix + WIN
    a = P[y0:y0 + WIN, x0:x0 + WIN]
    b = P[y0:y0 + WIN, x0 + 1:x0 + WIN + 1]
    c = P[y0 + 1:y0 + WIN + 1, x0:x0 + WIN]
    d = P[y0 + 1:y0 + WIN + 1, x0 + 1:x0 + WIN + 1]
    return _descale(a * iw[0] + b * iw[1] + c * iw[2] + d * iw[3], shift)


# why a point was lost (return_reasons): its window at level 0 lies outside the frame, its level-0 gradient matrix fails
# the min-eigenvalue test, it left the frame while iterating at level 0, or its final error window lies outside
TRACKED, LOST_OUTSIDE, LOST_MIN_EIG, LOST_ITERATING, LOST_ERR_WINDOW = range(5)


def calc_optical_flow_pyr_lk(prev, nxt, prev_pts, next_pts_init, max_level=3, max_iter=30, eps=0.01,
                             min_eig_threshold=1e-4, return_reasons=False):
    """Returns (next_pts float32 [n,2], status uint8 [n], err float32 [n]) (+ the reason of each status, int [n],
    with return_reasons)."""
    f32 = np.float32
    pyr_i, pyr_j = build_pyramid(prev, max_level), build_pyramid(nxt, max_level)
    max_level = min(len(pyr_i), len(pyr_j)) - 1
    n = len(prev_pts)
    prev_pts = np.asarray(prev_pts, dtype=f32)
    nxt_pts = np.array(next_pts_init, dtype=f32, copy=True)
    status = np.ones(n, dtype=np.uint8)
    err = np.zeros(n, dtype=f32)
    reason = np.zeros(n, dtype=np.int32)
    max_iter = min(max(max_iter, 0), 100)
    eps2 = min(max(eps, 0.0), 10.0) ** 2
    half = f32((WIN - 1) * 0.5)
    for level in range(max_level, -1, -1):
        I, J = pyr_i[level], pyr_j[level]
        rows, cols = I.shape
        Ip, Jp, Dp = _pad_img(I), _pad_img(J), _pad_deriv(scharr_deriv(I))
        scale = f32(1.0 / (1 << level))
        for k in range(n):
            prev_pt = prev_pts[k] * scale
            if level == max_level:
                next_pt = nxt_pts[k] * scale
            else:
                next_pt = nxt_pts[k] * f32(2.0)
            nxt_pts[k] = next_pt
            prev_pt = prev_pt - half
            ipx, ipy = int(np.floor(prev_pt[0])), int(np.floor(prev_pt[1]))
            if ipx < -WIN or ipx >= cols or ipy < -WIN or ipy >= rows:
                if level == 0:
                    status[k] = 0
                    err[k] = 0
                    reason[k] = LOST_OUTSIDE
                continue
            a, b = f32(prev_pt[0] - f32(ipx)), f32(prev_pt[1] - f32(ipy))
            iw = _weights(a, b)
            Iw = _patch(Ip, ipx, ipy, iw, W_BITS - 5)
            dIx = _patch(Dp[:, :, 0], ipx, ipy, iw, W_BITS)
            dIy = _patch(Dp[:, :, 1], ipx, ipy, iw, W_BITS)
            A11 = f32(f32(int(np.sum(dIx.astype(np.int64) ** 2))) * FLT_SCALE)
            A12 = f32(f32(int(np.sum(dIx.astype(np.int64) * dIy))) * FLT_SCALE)
            A22 = f32(f32(int(np.sum(dIy.astype(np.int64) ** 2))) * FLT_SCALE)
            D = f32(A11 * A22 - A12 * A12)
            min_eig = f32((A22 + A11 - np.sqrt(f32((A11 - A22) * (A11 - A22) + f32(4.0) * A12 * A12))) / f32(2 * WIN * WIN))
            if min_eig < min_eig_threshold or D < np.finfo(np.float32).eps:
                if level == 0:
                    status[k] = 0
                    reason[k] = LOST_MIN_EIG
                continue
            D = f32(1.0) / D
            next_pt = next_pt - half
            prev_delta = np.zeros(2, dtype=f32)
            for j in range(max_iter):
                inx, iny = int(np.floor(next_pt[0])), int(np.floor(next_pt[1]))
                if inx < -WIN or inx >= cols or iny < -WIN or iny >= rows:
                    if level == 0:
                        status[k] = 0
                        reason[k] = LOST_ITERATING
                    break
                a, b = f32(next_pt[0] - f32(inx)), f32(next_pt[1] - f32(iny))
                iwj = _weights(a, b)
                diff = _patch(Jp, inx, iny, iwj, W_BITS - 5) - Iw
                b1 = f32(f32(int(np.sum(diff.astype(np.int64) * dIx))) * FLT_SCALE)
                b2 = f32(f32(int(np.sum(diff.astype(np.int64) * dIy))) * FLT_SCALE)
                delta = np.array([f32((A12 * b2 - A22 * b1) * D), f32((A12 * b1 - A11 * b2) * D)], dtype=f32)
                next_pt = next_pt + delta
                nxt_pts[k] = next_pt + half
                if float(delta[0]) * float(delta[0]) + float(delta[1]) * float(delta[1]) <= eps2:
                    break
                if j > 0 and abs(delta[0] + prev_delta[0]) < 0.01 and abs(delta[1] + prev_delta[1]) < 0.01:
                    nxt_pts[k] = nxt_pts[k] - delta * f32(0.5)
                    break
                prev_delta = delta
            if status[k] and level == 0:
                npnt = nxt_pts[k] - half
                inx, iny = int(np.floor(npnt[0])), int(np.floor(npnt[1]))
                if inx < -WIN or inx >= cols or iny < -WIN or iny >= rows:
                    status[k] = 0
                    reason[k] = LOST_ERR_WINDOW
                    continue
                a, b = f32(npnt[0] - f32(inx)), f32(npnt[1] - f32(iny))
                iwj = _weights(a, b)
                diff = _patch(Jp, inx, iny, iwj, W_BITS - 5) - Iw
                err[k] = f32(np.sum(np.abs(diff)).astype(f32) * f32(1.0 / (32 * WIN * WIN)))
    return (nxt_pts, status, err, reason) if return_reasons else (nxt_pts, status, err)
