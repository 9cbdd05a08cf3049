// The image border of the tracker's kernels.  Its own header so that the fold compiles into a host program too: the
// suite checks it against cv2.borderInterpolate for every size up to 64 (tests/test_klt_oracle_edges.py).
#pragma once

#ifdef __CUDACC__
#define PVIO_KLT_HD __host__ __device__ __forceinline__
#else
#define PVIO_KLT_HD inline
#endif

namespace pvio {

// Frames narrower or lower than this are rejected (PVIO_B200_EINVAL): below it the LK window's reads fold more than twice
constexpr int kKltMinFrame = 12;

// cv::borderInterpolate(i, n, BORDER_REFLECT_101), the pixel an index outside [0, n) reads (... 2 1 | 0 1 ... n-1 | n-2 ...),
// for i in [-(n - 1), 2 (n - 1)], where one fold is enough: pyrDown's taps.
PVIO_KLT_HD int reflect101_once(int i, int n) {
    i = i < 0 ? -i : i;
    return i >= n ? 2 * (n - 1) - i : i;
}

// The same for i in [-3 (n - 1), 3 (n - 1)]: two folds, branch-free.  The LK window's 24-px patch around a point up to
// 21 px beyond the edge of a level reads indices -22 .. n + 21: one fold sends n + 21 below 0 on levels of 22 px (176 x 176
// at level 3), and frames narrower than the window fold at both edges.  Two folds cover that range for n >= 12.
PVIO_KLT_HD int reflect101(int i, int n) { return reflect101_once(reflect101_once(i, n), n); }

}  // namespace pvio
