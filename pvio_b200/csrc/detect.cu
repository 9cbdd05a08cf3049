// OpenCvImage::detect_keypoints (pvio-extra/src/pvio/extra/opencv_image.cpp:54-86): GFTT with the Harris response
// (GFTTDetector::create(1000, 1e-3, 20, 3, true), :183), sorted by response, thinned by PVIO's PoissonDiskFilter
// (pvio/src/pvio/utility/poisson_disk_filter.h) against the keypoints the frame already has, 20-pixel border.
//
// Split: everything per pixel runs on the device on the image the tracker has already uploaded (level 0 of the pyramid
// cache, i.e. the CLAHE output) --
//   harris_response_kernel  Sobel 3x3 (scale 1 / (4 * 3 * 255)), products, 3x3 box sums, det - k tr^2, fp32 throughout,
//                           BORDER_REFLECT_101 as cv::cornerHarris; image maximum by atomicMax
//   nms_compact_kernel      cv::goodFeaturesToTrack's selection: response > quality * max, equal to the 3x3 dilation,
//                           interior pixels only; survivors as 64-bit keys (response bits << 32 | pixel index)
//   cub::DeviceRadixSort    descending: by response, ties by the HIGHER address first (OpenCV's greaterThanPtr)
// -- and the two greedy passes, which are sequential by definition (each decision depends on the points accepted
// before it) and run over ~10^4 sorted candidates, stay on the host side of the C-ABI call: the minimum-distance grid
// of goodFeaturesToTrack (at most 1000 corners) and the Poisson-disk filter with the reference's exact cell walk.
//
// Parity (tests/test_gpu_detect.py): the response is NOT bit-identical to OpenCV's -- cv::cornerHarris's rounding
// depends on the SIMD path its dispatcher picks (Sobel-x matches only as fma(r0 + r2, s, r1 * 2s)) -- it agrees to
// ~4e-7 relative, and the SELECTED corner set is compared with cv2.goodFeaturesToTrack(useHarrisDetector=True) as a set:
// identical on every test image; a difference could only arise where two responses lie within that rounding.
#include <algorithm>
#include <cstring>
#include <unordered_map>
#include <vector>

#include <cub/cub.cuh>

#include "api_internal.h"

namespace pvio {
namespace {

__device__ __forceinline__ int refl(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

constexpr int kTX = 32, kTY = 16;

// one thread per pixel; the (kTX + 2) x (kTY + 2) tile of the three products in shared memory.  Every operation is a
// separately rounded fp32 operation except the one fused multiply-add of the Sobel-x column pass (this file is
// compiled with -fmad=false).
__global__ void __launch_bounds__(kTX *kTY) harris_response_kernel(const uint8_t *img, int w, int h, float k, float *resp, int *max_bits) {
    __shared__ float cxx[kTY + 2][kTX + 2], cxy[kTY + 2][kTX + 2], cyy[kTY + 2][kTX + 2];
    const int x0 = blockIdx.x * kTX, y0 = blockIdx.y * kTY, tid = threadIdx.y * kTX + threadIdx.x;
    // the box filter's border pixel is the product AT the mirror pixel: evaluate the products at reflected coordinates
    for (int e = tid; e < (kTY + 2) * (kTX + 2); e += kTX * kTY) {
        const int py = e / (kTX + 2), px = e - py * (kTX + 2);
        const int cx = refl(x0 + px - 1, w), cy = refl(y0 + py - 1, h);      // BORDER_REFLECT_101 of the box filter
        float p[3][3];
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) p[dy + 1][dx + 1] = (float)img[(size_t)refl(cy + dy, h) * w + refl(cx + dx, w)];   // Sobel's own border
        const float s = 1.0f / ((1 << 2) * 3 * 255.0f), s2 = 2.0f * s;
        const float r0 = p[0][2] - p[0][0], r1 = p[1][2] - p[1][0], r2 = p[2][2] - p[2][0];          // exact integers
        const float gx = fmaf(r0 + r2, s, r1 * s2);
        const float g0 = p[0][0] + 2.0f * p[0][1] + p[0][2], g2 = p[2][0] + 2.0f * p[2][1] + p[2][2];
        const float gy = (g2 - g0) * s;
        cxx[py][px] = gx * gx; cxy[py][px] = gx * gy; cyy[py][px] = gy * gy;
    }
    __syncthreads();
    const int x = x0 + threadIdx.x, y = y0 + threadIdx.y;
    if (x >= w || y >= h) return;
    const int px = threadIdx.x + 1, py = threadIdx.y + 1;
    float a, b, c;
    {
        const float u0 = (cxx[py - 1][px - 1] + cxx[py - 1][px]) + cxx[py - 1][px + 1];
        const float u1 = (cxx[py][px - 1] + cxx[py][px]) + cxx[py][px + 1];
        const float u2 = (cxx[py + 1][px - 1] + cxx[py + 1][px]) + cxx[py + 1][px + 1];
        a = (u0 + u1) + u2;
    }
    {
        const float u0 = (cxy[py - 1][px - 1] + cxy[py - 1][px]) + cxy[py - 1][px + 1];
        const float u1 = (cxy[py][px - 1] + cxy[py][px]) + cxy[py][px + 1];
        const float u2 = (cxy[py + 1][px - 1] + cxy[py + 1][px]) + cxy[py + 1][px + 1];
        b = (u0 + u1) + u2;
    }
    {
        const float u0 = (cyy[py - 1][px - 1] + cyy[py - 1][px]) + cyy[py - 1][px + 1];
        const float u1 = (cyy[py][px - 1] + cyy[py][px]) + cyy[py][px + 1];
        const float u2 = (cyy[py + 1][px - 1] + cyy[py + 1][px]) + cyy[py + 1][px + 1];
        c = (u0 + u1) + u2;
    }
    const float tr = a + c;
    const float r = a * c - b * b - k * (tr * tr);
    resp[(size_t)y * w + x] = r;
    if (r > 0.0f) atomicMax(max_bits, __float_as_int(r));       // positive floats order like their bit patterns
}

__global__ void nms_compact_kernel(const float *resp, int w, int h, double quality, const int *max_bits, unsigned long long *keys,
                                   int *count, int cap) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x < 1 || y < 1 || x >= w - 1 || y >= h - 1) return;      // goodFeaturesToTrack visits interior pixels only
    const float mx = __int_as_float(*max_bits);
    const float thr = (float)((double)mx * quality);             // cv::threshold(eig, eig, maxVal * qualityLevel, 0, THRESH_TOZERO)
    const float v = resp[(size_t)y * w + x];
    if (!(v > thr)) return;
    bool is_max = true;                                          // val == dilate(thresholded)(x, y): no neighbour above it
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy)
#pragma unroll
        for (int dx = -1; dx <= 1; ++dx) is_max &= !(resp[(size_t)(y + dy) * w + (x + dx)] > v);
    if (!is_max) return;
    const int slot = atomicAdd(count, 1);
    if (slot < cap) keys[slot] = ((unsigned long long)(unsigned)__float_as_int(v) << 32) | (unsigned)(y * w + x);
}

// cv::goodFeaturesToTrack's minimum-distance pass over the sorted corners (imgproc/featureselect.cpp)
void min_distance_select(const unsigned long long *keys, int n, int w, int h, double min_distance, int max_corners, std::vector<float> &out) {
    const int cell = (int)std::lround(min_distance);
    const int gw = (w + cell - 1) / cell, gh = (h + cell - 1) / cell;
    std::vector<std::vector<std::pair<float, float>>> grid((size_t)gw * gh);
    const double md2 = min_distance * min_distance;
    int ncorners = 0;
    for (int i = 0; i < n; ++i) {
        const unsigned idx = (unsigned)(keys[i] & 0xffffffffu);
        const int y = (int)(idx / (unsigned)w), x = (int)(idx - (unsigned)y * (unsigned)w);
        const int xc = x / cell, yc = y / cell;
        const int x1 = std::max(0, xc - 1), y1 = std::max(0, yc - 1), x2 = std::min(gw - 1, xc + 1), y2 = std::min(gh - 1, yc + 1);
        bool good = true;
        for (int yy = y1; yy <= y2 && good; ++yy)
            for (int xx = x1; xx <= x2 && good; ++xx)
                for (const auto &p : grid[(size_t)yy * gw + xx]) {
                    const float dx = (float)x - p.first, dy = (float)y - p.second;
                    if (dx * dx + dy * dy < md2) { good = false; break; }
                }
        if (!good) continue;
        grid[(size_t)yc * gw + xc].emplace_back((float)x, (float)y);
        out.push_back((float)x); out.push_back((float)y);
        if (++ncorners >= max_corners && max_corners > 0) break;
    }
}

// PoissonDiskFilter<2> (utility/poisson_disk_filter.h): sparse grid of cell size r / sqrt(2) holding the LAST point
// inserted per cell; test_point walks the 5 x 5 block around the candidate's cell -- as written in the reference: the
// walk advances BEFORE it looks, so the first cell of the block is never examined and one cell past its end is.
struct PoissonFilter {
    double r2, gs;
    int span;
    std::vector<std::pair<double, double>> pts;
    std::unordered_map<long long, size_t> grid;
    explicit PoissonFilter(double radius) : r2(radius * radius), gs(radius / std::sqrt(2.0)), span((int)std::ceil(std::sqrt(2.0))) {}
    static long long key(int ix, int iy) { return ((long long)ix << 32) ^ (unsigned)iy; }
    void index_of(double x, double y, int &ix, int &iy) const { ix = (int)std::floor(x / gs); iy = (int)std::floor(y / gs); }
    void preset(double x, double y) { int ix, iy; index_of(x, y, ix, iy); grid[key(ix, iy)] = pts.size(); pts.emplace_back(x, y); }
    bool test(double x, double y, int &ix, int &iy) const {
        index_of(x, y, ix, iy);
        const int bx = ix - span, by = iy - span, ex = ix + span, ey = iy + span;
        int cx = bx, cy = by;
        while (cy <= ey) {
            ++cx;
            if (cx > ex) { cx = bx; ++cy; }
            auto it = grid.find(key(cx, cy));
            if (it != grid.end()) {
                const double dx = x - pts[it->second].first, dy = y - pts[it->second].second;
                if (dx * dx + dy * dy < r2) return false;
            }
        }
        return true;
    }
    bool insert(double x, double y) {
        int ix, iy;
        if (!test(x, y, ix, iy)) return false;
        grid[key(ix, iy)] = pts.size(); pts.emplace_back(x, y);
        return true;
    }
};

int ensure(Handle *h, int w, int hgt) {
    DetectState &d = h->detect;
    const size_t px = (size_t)w * hgt;
    if (d.w != w || d.h != hgt) {
        d = DetectState{};
        d.w = w; d.h = hgt;
        d.cap = (int)std::min<size_t>(px / 4 + 1024, (size_t)1 << 22);       // local maxima of a 3x3 test: at most one per 2x2 block
        cub::DeviceRadixSort::SortKeysDescending(nullptr, d.cub_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, d.cap);
    }
    TRY(reserve(h, d.img, px, kBoth));
    TRY(reserve(h, d.raw, px, kDevice));
    TRY(reserve(h, d.resp, px, kDevice));
    TRY(reserve(h, d.keys, d.cap, kDevice));
    TRY(reserve(h, d.keys_sorted, d.cap, kBoth));
    TRY(reserve(h, d.counters, 2, kBoth));
    TRY(reserve(h, d.cub_tmp, d.cub_bytes, kDevice));
    return 0;
}

}  // namespace
}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_detect_keypoints(pvio_b200_handle hh, uint64_t frame_id, const uint8_t *image, int width, int height, int stride,
                                          double clahe_clip, int tiles_x, int tiles_y, const double *existing, int n_existing,
                                          double keypoint_distance, int max_out, double *keypoints_out, int *n_out,
                                          float *gftt_out, int *n_gftt) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !n_out) return PVIO_B200_EINVAL;
    if (width < 8 || height < 8 || n_existing < 0 || max_out < 0 || keypoint_distance <= 0.0 || clahe_clip < 0.0 ||
        (n_existing > 0 && !existing) || (max_out > 0 && !keypoints_out))
        return fail(h, PVIO_B200_EINVAL, "detect_keypoints: bad arguments");
    if (clahe_clip > 0.0 && (tiles_x < 1 || tiles_y < 1 || width % tiles_x || height % tiles_y))
        return fail(h, PVIO_B200_EINVAL, "clahe: the image size must be a multiple of the tile grid");
    TRY(ensure(h, width, height));
    DetectState &d = h->detect;
    const size_t px = (size_t)width * height;
    const uint8_t *src = klt_cached_level0(h, frame_id, width, height, clahe_clip);
    if (!src) {
        if (!image || stride < width) return fail(h, PVIO_B200_EINVAL, "detect_keypoints: frame not cached and no pixels given");
        for (int y = 0; y < height; ++y) memcpy(d.img.h + (size_t)y * width, image + (size_t)y * stride, width);
        if (clahe_clip > 0.0) {
            TRY(reserve(h, d.lut, (size_t)tiles_x * tiles_y * 256, kDevice));
            CK(h, cudaMemcpyAsync(d.raw.d, d.img.h, px, cudaMemcpyHostToDevice, h->stream));
            TRY(klt_clahe_device(h, d.raw.d, d.img.d, d.lut.d, width, height, clahe_clip, tiles_x, tiles_y));
        } else {
            CK(h, cudaMemcpyAsync(d.img.d, d.img.h, px, cudaMemcpyHostToDevice, h->stream));
        }
        src = d.img.d;
    }
    int *counters = d.counters.d;
    CK(h, cudaMemsetAsync(counters, 0, sizeof(int) * 2, h->stream));
    harris_response_kernel<<<dim3((width + kTX - 1) / kTX, (height + kTY - 1) / kTY), dim3(kTX, kTY), 0, h->stream>>>(
        src, width, height, 0.04f, d.resp.d, counters);
    nms_compact_kernel<<<dim3((width + 31) / 32, (height + 7) / 8), dim3(32, 8), 0, h->stream>>>(
        d.resp.d, width, height, 1.0e-3, counters, d.keys.d, counters + 1, d.cap);
    h->launches += 2;
    CK(h, cudaMemcpyAsync(d.counters.h, counters, sizeof(int) * 2, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    const int n = std::min(d.counters.h[1], d.cap);
    std::vector<float> corners;
    if (n > 0) {
        size_t tmp = d.cub_bytes;
        cub::DeviceRadixSort::SortKeysDescending(d.cub_tmp.d, tmp, d.keys.d, d.keys_sorted.d, n, 0, 64, h->stream);
        ++h->launches;
        CK(h, cudaMemcpyAsync(d.keys_sorted.h, d.keys_sorted.d, sizeof(unsigned long long) * n, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaStreamSynchronize(h->stream));
        CK(h, cudaGetLastError());
        min_distance_select(d.keys_sorted.h, n, width, height, 20.0, 1000, corners);          // GFTTDetector::create(1000, 1e-3, 20, 3, true)
    }
    const int ng = (int)corners.size() / 2;
    if (n_gftt) *n_gftt = ng;
    if (gftt_out) memcpy(gftt_out, corners.data(), sizeof(float) * corners.size());     // caller sizes it for 1000 corners
    // opencv_image.cpp:69-84: Poisson-disk filter against the existing keypoints, then the 20-pixel border
    PoissonFilter f(keypoint_distance);
    for (int i = 0; i < n_existing; ++i) f.preset(existing[2 * i], existing[2 * i + 1]);
    int m = 0;
    for (int i = 0; i < ng; ++i) {
        const double x = corners[2 * i], y = corners[2 * i + 1];
        if (!f.insert(x, y)) continue;
        if (x < 20 || y < 20 || x >= width - 20 || y >= height - 20) continue;
        if (m < max_out) { keypoints_out[2 * m] = x; keypoints_out[2 * m + 1] = y; }
        ++m;
    }
    *n_out = m;
    return m > max_out ? fail(h, PVIO_B200_EINVAL, "detect_keypoints: output array too small") : 0;
}
