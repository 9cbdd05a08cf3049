"""NumPy restatement of the two ways PVIO's dataset readers remove lens distortion, pinned bit for bit against cv2 in
tests/test_undistort_oracle.py:

  radtan       cv::undistort(img, out, K, D) with K and D as cv::Mat_<float> (pvio-pc/src/euroc_dataset_reader.cpp:70-74,
               OpenCvImage::correct_distortion): cv::undistort builds OpenCV's CV_16SC2 map stripe by stripe with
               initUndistortRectifyMap (new camera matrix K) and remaps each stripe.
  equidistant  ImageUndistorter (pvio-extra/include/pvio/extra/image_undistorter.h:28-95): distort_pixel in double for
               every pixel, cast to float, cv::convertMaps(CV_32FC1 -> CV_16SC2), then the same remap.

Maps are OpenCV's pair: m1 int16 [h][w][2] (the integer source pixel) and m2 uint16 [h][w], the fractional table
index (iv & 31) * 32 + (iu & 31).  The remap is cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) on 8-bit frames in
integer arithmetic: taps outside the frame read 0, weights (32 - fx)(32 - fy), fx (32 - fy), (32 - fx) fy, fx fy,
result (sum + 512) >> 10.

Every expression below is evaluated in the order of the C++ it restates (float64 NumPy operations round like the C++
doubles; sequential sums use np.cumsum, which adds left to right)."""
import math

import numpy as np

RADTAN, EQUIDISTANT = 1, 2
INT_MIN, INT_MAX = -2 ** 31, 2 ** 31 - 1


def _cv_round(a):
    """cvRound / saturate_cast<int>: nearest, ties to even, saturated to int32"""
    return np.clip(np.rint(a), INT_MIN, INT_MAX).astype(np.int64)


def _pack(iu, iv, saturate):
    """the CV_16SC2 pair of 1/32-pixel fixed-point coordinates iu, iv"""
    a, b = iu >> 5, iv >> 5
    if saturate:                                   # convertMaps: saturate_cast<short>
        a, b = np.clip(a, -32768, 32767), np.clip(b, -32768, 32767)
    m1 = np.stack([a, b], axis=-1).astype(np.int64).astype(np.uint16).view(np.int16)   # (short): two's-complement wrap
    m2 = ((iv & 31) * 32 + (iu & 31)).astype(np.uint16)
    return m1, m2


def _inv3(a):
    """cv::Matx33d::inv(DECOMP_LU) / cv::invert(DECOMP_LU) of a 3x3 double matrix: OpenCV's closed 3x3 form"""
    d = a[0][0] * (a[1][1] * a[2][2] - a[1][2] * a[2][1]) - a[0][1] * (a[1][0] * a[2][2] - a[1][2] * a[2][0]) + \
        a[0][2] * (a[1][0] * a[2][1] - a[1][1] * a[2][0])
    d = 1.0 / d
    return [(a[1][1] * a[2][2] - a[1][2] * a[2][1]) * d, (a[0][2] * a[2][1] - a[0][1] * a[2][2]) * d,
            (a[0][1] * a[1][2] - a[0][2] * a[1][1]) * d,
            (a[1][2] * a[2][0] - a[1][0] * a[2][2]) * d, (a[0][0] * a[2][2] - a[0][2] * a[2][0]) * d,
            (a[0][2] * a[1][0] - a[0][0] * a[1][2]) * d,
            (a[1][0] * a[2][1] - a[1][1] * a[2][0]) * d, (a[0][1] * a[2][0] - a[0][0] * a[2][1]) * d,
            (a[0][0] * a[1][1] - a[0][1] * a[1][0]) * d]


def radtan_rows(fx, fy, cx, cy, k1, k2, p1, p2, width, rows, ar12):
    """initUndistortRectifyMap's scalar loop (camera matrix A = [fx 0 cx; 0 fy cy; 0 0 1], new camera matrix Ar = A
    with Ar(1, 2) = ar12, R = I, distortion k1 k2 p1 p2 and zero k3..k6, s1..s4, tau) over `rows` rows of `width`:
    the double map coordinates (u, v) [rows][width]"""
    k3 = k4 = k5 = k6 = s1 = s2 = s3 = s4 = 0.0
    ir = _inv3([[fx, 0.0, cx], [0.0, fy, ar12], [0.0, 0.0, 1.0]])
    i = np.arange(rows, dtype=np.float64)[:, None]

    def walk(a, b, c):                     # _x = i * ir[1] + ir[2], then _x += ir[0] per column
        start = i * b + c
        steps = np.full((rows, width), a)
        steps[:, :1] = start
        return np.cumsum(steps, axis=1)
    _x, _y, _w = walk(ir[0], ir[1], ir[2]), walk(ir[3], ir[4], ir[5]), walk(ir[6], ir[7], ir[8])
    w = 1.0 / _w
    x = _x * w
    y = _y * w
    x2 = x * x
    y2 = y * y
    r2 = x2 + y2
    _2xy = 2 * x * y
    kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2)
    xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2) + s1 * r2 + s2 * r2 * r2
    yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy + s3 * r2 + s4 * r2 * r2
    # matTilt is the identity (tau = 0): vecTilt = (xd + 0 + 0, 0 + yd + 0, 1), invProj = 1
    u = fx * 1.0 * xd + cx
    v = fy * 1.0 * yd + cy
    return u, v


def _f32(v):
    return float(np.float32(v))


def radtan_map(width, height, K, D):
    """cv::undistort's map for camera K = (fx, fy, cx, cy) and D = (k1, k2, p1, p2) given as float32 (Mat_<float>):
    stripes of min(max(1, 4096 / width), height) rows, Ar(1, 2) = cy - y0 per stripe.  Returns (m1, m2)."""
    fx, fy, cx, cy = (_f32(v) for v in K)
    k1, k2, p1, p2 = (_f32(v) for v in D)
    stripe = min(max(1, 4096 // max(width, 1)), height)
    us, vs = [], []
    for y0 in range(0, height, stripe):
        rows = min(stripe, height - y0)
        u, v = radtan_rows(fx, fy, cx, cy, k1, k2, p1, p2, width, rows, cy - y0)
        us.append(u)
        vs.append(v)
    u, v = np.concatenate(us), np.concatenate(vs)
    return _pack(_cv_round(u * 32.0), _cv_round(v * 32.0), saturate=False)


def equidistant_float_map(width, height, K, D):
    """ImageUndistorter's float maps (map_x_float, map_y_float) [h][w] for K = (fx, fy, cx, cy), D = (k1, k2, k3, k4),
    all double.  K.inverse() is Eigen's 3x3 cofactor inverse (cofactors times 1 / det, det = cofactor column 0 . K
    column 0); with K's zeros the summation orders of the inverse's determinant, of both matrix-vector products and of
    hnormalized do not change a result."""
    fx, fy, cx, cy = (float(v) for v in K)
    k1, k2, k3, k4 = (float(v) for v in D)
    m = [[fx, 0.0, cx], [0.0, fy, cy], [0.0, 0.0, 1.0]]

    def cof(i, j):
        i1, i2, j1, j2 = (i + 1) % 3, (i + 2) % 3, (j + 1) % 3, (j + 2) % 3
        return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1]
    det = cof(0, 0) * m[0][0] + cof(1, 0) * m[1][0] + cof(2, 0) * m[2][0]
    invdet = 1.0 / det
    ki = [[cof(c, r) * invdet for c in range(3)] for r in range(3)]     # inverse(r, c) = cofactor(c, r) / det
    v, u = np.meshgrid(np.arange(height, dtype=np.float64), np.arange(width, dtype=np.float64), indexing="ij")
    x = ki[0][0] * u + ki[0][1] * v + ki[0][2] * 1.0
    y = ki[1][0] * u + ki[1][1] * v + ki[1][2] * 1.0
    z = ki[2][0] * u + ki[2][1] * v + ki[2][2] * 1.0
    r = np.sqrt(x * x + y * y)
    theta = np.array([math.atan(t) for t in r.ravel()]).reshape(r.shape)     # glibc's atan, as the reference's
    theta2 = theta * theta
    theta4 = theta2 * theta2
    theta6 = theta2 * theta4
    theta8 = theta4 * theta4
    thetad = theta * (1 + k1 * theta2 + k2 * theta4 + k3 * theta6 + k4 * theta8)
    with np.errstate(divide="ignore", invalid="ignore"):
        scaling = np.where(r > 1e-8, thetad / r, 1.0)
        xd = x * scaling
        yd = y * scaling
        px = fx * xd + 0.0 * yd + cx * z
        py = 0.0 * xd + fy * yd + cy * z
        pz = 0.0 * xd + 0.0 * yd + 1.0 * z
        mx, my = px / pz, py / pz
    early = r < 1e-10                      # distort_pixel returns the pixel itself
    mx = np.where(early, u, mx)
    my = np.where(early, v, my)
    return mx.astype(np.float32), my.astype(np.float32)


def convert_maps(mx, my):
    """cv::convertMaps(CV_32FC1, CV_32FC1 -> CV_16SC2): cvRound(f * 32) in float, saturate_cast<short>"""
    iu = _cv_round((mx * np.float32(32)).astype(np.float32))
    iv = _cv_round((my * np.float32(32)).astype(np.float32))
    return _pack(iu, iv, saturate=True)


def equidistant_map(width, height, K, D):
    return convert_maps(*equidistant_float_map(width, height, K, D))


def undistort_map(model, width, height, K, D):
    if model == RADTAN:
        return radtan_map(width, height, K, D)
    if model == EQUIDISTANT:
        return equidistant_map(width, height, K, D)
    raise ValueError("unknown lens model")


def remap(img, m1, m2):
    """cv::remap(img, out, m1, m2, INTER_LINEAR, BORDER_CONSTANT, 0) of an 8-bit frame"""
    img = np.asarray(img, dtype=np.uint8)
    h, w = img.shape
    sx = m1[..., 0].astype(np.int64)
    sy = m1[..., 1].astype(np.int64)
    fx = (m2 & 31).astype(np.int64)
    fy = (m2 >> 5).astype(np.int64)

    def tap(x, y):
        inside = (x >= 0) & (x < w) & (y >= 0) & (y < h)
        return np.where(inside, img[np.clip(y, 0, h - 1), np.clip(x, 0, w - 1)].astype(np.int64), 0)
    s = tap(sx, sy) * (32 - fx) * (32 - fy) + tap(sx + 1, sy) * fx * (32 - fy) + \
        tap(sx, sy + 1) * (32 - fx) * fy + tap(sx + 1, sy + 1) * fx * fy
    return ((s + 512) >> 10).astype(np.uint8)


def undistort(img, model, K, D):
    h, w = np.asarray(img).shape
    return remap(img, *undistort_map(model, w, h, K, D))
