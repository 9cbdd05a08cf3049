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
#include <cassert>
#include <climits>
#include <cmath>
#include <cstring>
#include <unordered_map>
#include <vector>

#include <cub/cub.cuh>
#include <thrust/iterator/counting_iterator.h>
#include <thrust/iterator/transform_iterator.h>

#include "api_internal.h"
#include "detect.cuh"

namespace pvio {
namespace {

__device__ __forceinline__ int refl(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

constexpr int kTX = 32, kTY = 16;

// the single call's staging (DetectState::stage, both sides): its frame, the frame CLAHE equalises, zeroed counters
struct DetectStage {
    DetectBatchFrame frame;
    KltBatchFrame clahe;
    int counters[2];                          // [0] max response bits, [1] candidate count
};

// one thread per pixel; the (kTX + 2) x (kTY + 2) tile of the three products in shared memory.  Every operation is a
// separately rounded fp32 operation except the one fused multiply-add of the Sobel-x column pass (this file is
// compiled with -fmad=false).  The frame is frames[blockIdx.z] (blocks outside a smaller frame exit).
__global__ void __launch_bounds__(kTX *kTY) harris_response_kernel(float k, const DetectBatchFrame *frames) {
    __shared__ float cxx[kTY + 2][kTX + 2], cxy[kTY + 2][kTX + 2], cyy[kTY + 2][kTX + 2];
    const DetectBatchFrame &f = frames[blockIdx.z];
    const uint8_t *img = f.img;
    float *resp = f.resp;
    int *max_bits = f.counters;
    const int w = f.w, h = f.h;
    if ((int)blockIdx.x * kTX >= w || (int)blockIdx.y * kTY >= h) return;     // block-uniform
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

// The frame is frames[blockIdx.z]; its keys go to its own segment
__global__ void nms_compact_kernel(double quality, const DetectBatchFrame *frames) {
    const DetectBatchFrame &f = frames[blockIdx.z];
    const float *resp = f.resp;
    const int *max_bits = f.counters;
    unsigned long long *keys = f.keys;
    int *count = f.counters + 1;
    const int w = f.w, h = f.h, cap = f.cap;
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

// local maxima of a 3x3 test: at most one per 2x2 block
int candidate_cap(size_t px) { return (int)std::min<size_t>(px / 4 + 1024, (size_t)1 << 22); }

int ensure(Handle *h, int w, int hgt) {
    DetectState &d = h->detect;
    const size_t px = (size_t)w * hgt;
    if (d.w != w || d.h != hgt) {
        d = DetectState{};
        d.w = w; d.h = hgt;
        d.cap = candidate_cap(px);
        cub::DeviceRadixSort::SortKeysDescending(nullptr, d.cub_bytes, (unsigned long long *)nullptr, (unsigned long long *)nullptr, d.cap);
    }
    TRY(reserve(h, d.img, px, kBoth));
    TRY(reserve(h, d.raw, px, kDevice));
    TRY(reserve(h, d.resp, px, kDevice));
    TRY(reserve(h, d.keys, d.cap, kDevice));
    TRY(reserve(h, d.keys_sorted, d.cap, kBoth));
    TRY(reserve(h, d.stage, sizeof(DetectStage), kBoth));
    TRY(reserve(h, d.cub_tmp, d.cub_bytes, kDevice));
    return 0;
}

// ---- the batched detector (pvio_b200_batch_detect_keypoints) -------------------------------------------------------
// n frames, each cached in a slot of the batched tracker or uploaded.  Every request is checked before anything is
// staged.  Then: one H2D copy of the packed staging (descriptors, zeroed counters, existing points, uploaded pixels);
// CLAHE over the uploaded frames (2 launches, clahe_clip > 0 only); Harris and NMS over every frame, grid z = frame
// (2); a segmented descending radix sort of each frame's keys, whose segment ends are read on the device (1);
// detect_select_kernel, one CTA per frame running both greedy passes (1); one D2H copy of the results, a synchronise.
// An uploaded frame whose slot has a lens (pvio_b200_batch_set_lens) is raw: it is remapped first (1 launch over every
// such frame, undistort.cu) into the detector's scratch, which CLAHE (or, without CLAHE, Harris) reads.  These frames
// come first among the CLAHE descriptors, so the remap's grid covers them alone.
constexpr int kMinDist = 20;                  // GFTT's minDistance, and the cell of its grid (lround(20))
constexpr int kCellEmpty = -(1 << 30);        // x of an empty min-distance slot: farther than 20 px from every pixel
constexpr int kSelectThreads = 128;
constexpr int kMaxBatchDetect = 65535;        // grid z: one layer per frame

// min_distance_select's distance test: float dx^2 + dy^2 against 20^2
__device__ __forceinline__ bool md_close(int x, int y, int px, int py) {
    const float dx = (float)x - (float)px, dy = (float)y - (float)py;
    return dx * dx + dy * dy < 400.0f;
}

// The two greedy passes of pvio_b200_detect_keypoints (min_distance_select, PoissonFilter, the border) for frame
// blockIdx.x, with exactly their semantics.  Working area (shared memory, or f.work when it does not fit there):
//   grid     [gh][gw] int4: the min-distance grid, two (x, y) slots per 20 x 20 cell.  Two slots suffice: accepted
//            corners are >= 20 px apart, the integer pixels of one cell differ by <= 19 per axis, and 3 points in a
//            square of side 19 are at most (sqrt(6) - sqrt(2)) * 19 = 19.67 px apart.
//   corners  [1000] float2: the accepted corners in order
//   hk, hv   the Poisson grid as an open-addressing hash table of 2^hbits cells (>= twice the points it can hold):
//            cell -> index of the LAST point inserted into it (presets: their index; corner j: n_pre + j)
// All warps initialise the area and insert the presets; warp 0 then runs the passes.
//   min distance  32 sorted candidates per step: each lane tests its candidate against the grid, the chunk is then
//                 resolved in lane order (the host's order) with shuffles: lane k is accepted if it passed and no
//                 accepted earlier lane of the chunk is closer than 20 px.  Within 20 px means within the 3 x 3 cells
//                 the host examines, so the two tests agree.  Stops at 1000 corners.
//   Poisson       corner by corner, poisson_insert (detect.cuh); a taken corner is kept if it lies inside the 20-px
//                 border.
__global__ void __launch_bounds__(kSelectThreads) detect_select_kernel(const DetectBatchFrame *frames) {
    extern __shared__ __align__(16) uint8_t smem[];
    const DetectBatchFrame &f = frames[blockIdx.x];
    uint8_t *work = f.work ? f.work : smem;
    const int ncell = f.gw * f.gh, tid = threadIdx.x;
    const unsigned long long hcap = 1ull << f.hbits;
    int4 *grid = reinterpret_cast<int4 *>(work);
    float2 *corners = reinterpret_cast<float2 *>(work + sizeof(int4) * (size_t)ncell);
    unsigned long long *hk = reinterpret_cast<unsigned long long *>(corners + kMaxCorners);
    int *hv = reinterpret_cast<int *>(hk + hcap);
    DetectResult *res = f.res;
    for (int c = tid; c < ncell; c += kSelectThreads) grid[c] = make_int4(kCellEmpty, 0, kCellEmpty, 0);
    for (unsigned long long s = tid; s < hcap; s += kSelectThreads) { hk[s] = kHashEmpty; hv[s] = -1; }
    for (int j = tid; j < (kMaxCorners + 31) / 32; j += kSelectThreads) res->mask[j] = 0;
    __syncthreads();
    const unsigned long long hm = hcap - 1;
    const double gs = f.gs;
    const int n_pre = f.pre_count ? *f.pre_count : f.n_pre;
    for (int i = tid; i < n_pre; i += kSelectThreads) {             // the last preset of a cell holds it: the largest index
        const double2 p = f.pre[i];
        // only presets in cells [-2, cxmax + 2] x [-2, cymax + 3] can meet a corner's walk: the others stay out
        const double fx = floor(p.x / gs), fy = floor(p.y / gs);
        if (!(fx >= -2.0 && fx <= f.cxmax + 2.0 && fy >= -2.0 && fy <= f.cymax + 3.0)) continue;
        const unsigned long long key = cell_key((long long)fx, (long long)fy);
        for (unsigned long long s = hash_slot(key, f.hbits);; s = (s + 1) & hm) {
            const unsigned long long k = atomicCAS(&hk[s], kHashEmpty, key);
            if (k == kHashEmpty || k == key) { atomicMax(&hv[s], i); break; }
        }
    }
    __syncthreads();
    if (tid >= 32) return;
    const int lane = tid, w = f.w, hgt = f.h, gw = f.gw, gh = f.gh;

    // cv::goodFeaturesToTrack's minimum-distance pass over the sorted candidates
    const int nk = min(f.counters[1], f.cap);
    const unsigned long long *keys = f.sorted;
    int ng = 0;
    for (int base = 0; base < nk && ng < kMaxCorners; base += 32) {
        const int i = base + lane;
        int x = 0, y = 0;
        unsigned idx = 0;
        bool ok = false;
        if (i < nk) {
            idx = (unsigned)(keys[i] & 0xffffffffull);
            y = (int)(idx / (unsigned)w); x = (int)(idx - (unsigned)y * (unsigned)w);
            const int xc = x / kMinDist, yc = y / kMinDist;
            ok = true;
            for (int yy = max(0, yc - 1); yy <= min(gh - 1, yc + 1); ++yy)
                for (int xx = max(0, xc - 1); xx <= min(gw - 1, xc + 1); ++xx) {
                    const int4 c = grid[yy * gw + xx];
                    if (md_close(x, y, c.x, c.y) || md_close(x, y, c.z, c.w)) ok = false;
                }
        }
        const unsigned passed = __ballot_sync(0xffffffffu, ok);
        if (!passed) continue;
        unsigned conf = 0;                                          // passed earlier lanes closer than 20 px
        for (int k = 0; k < 31; ++k) {
            const int xk = __shfl_sync(0xffffffffu, x, k), yk = __shfl_sync(0xffffffffu, y, k);
            if (k < lane && ((passed >> k) & 1u) && md_close(x, y, xk, yk)) conf |= 1u << k;
        }
        unsigned acc = 0;
        int nacc = 0;
        const int room = kMaxCorners - ng;
        for (int k = 0; k < 32 && nacc < room; ++k) {
            const unsigned ck = __shfl_sync(0xffffffffu, conf, k);
            if (((passed >> k) & 1u) && !(ck & acc)) { acc |= 1u << k; ++nacc; }
        }
        if ((acc >> lane) & 1u) {
            const int pos = ng + __popc(acc & ((1u << lane) - 1u));
            corners[pos] = make_float2((float)x, (float)y);
            res->corner[pos] = idx;
            int4 &c = grid[(y / kMinDist) * gw + x / kMinDist];
            if (atomicCAS(&c.x, kCellEmpty, x) == kCellEmpty) {
                c.y = y;
            } else {
                const int old = atomicCAS(&c.z, kCellEmpty, x);
                assert(old == kCellEmpty);                           // two slots per cell (above)
                c.w = y;
            }
        }
        ng += nacc;
        __syncwarp();
    }
    if (lane == 0) res->n_gftt = ng;
    __syncwarp();

    // PoissonDiskFilter against the presets, then the 20-pixel border (opencv_image.cpp:69-84)
    const double r2 = f.r2;
    const double2 *pre = f.pre;
    auto point = [pre, corners, n_pre](int v) {
        return v < n_pre ? pre[v] : make_double2((double)corners[v - n_pre].x, (double)corners[v - n_pre].y);
    };
    unsigned word = 0;
    for (int i = 0; i < ng; ++i) {
        const double x = corners[i].x, y = corners[i].y;
        const bool take = poisson_insert(hk, hv, f.hbits, gs, r2, x, y, n_pre + i, point);
        if (lane == 0) {
            if (take && !(x < 20 || y < 20 || x >= w - 20 || y >= hgt - 20)) word |= 1u << (i & 31);
            if ((i & 31) == 31 || i == ng - 1) { res->mask[i >> 5] = word; word = 0; }
        }
    }
}

// the segment [begin, end) of frame i's keys; end read on the device after the NMS kernel has counted them
struct SegBegin {
    const DetectBatchFrame *f;
    __host__ __device__ int operator()(int i) const { return f[i].key_off; }
};
struct SegEnd {
    const DetectBatchFrame *f;
    __host__ __device__ int operator()(int i) const {
        const int c = f[i].counters[1];
        return f[i].key_off + (c < f[i].cap ? c : f[i].cap);
    }
};

}  // namespace

DetectPlan detect_plan(int w, int hgt, double keypoint_distance, int n_pre) {
    DetectPlan P;
    P.cap = candidate_cap((size_t)w * hgt);
    P.gs = keypoint_distance / std::sqrt(2.0);                      // PoissonFilter's cell size
    P.cxmax = std::min(std::floor((w - 1) / P.gs), kCellLimit);
    P.cymax = std::min(std::floor((hgt - 1) / P.gs), kCellLimit);
    P.n_pre = n_pre;
    P.gw = (w + kMinDist - 1) / kMinDist;
    P.gh = (hgt + kMinDist - 1) / kMinDist;
    P.hbits = 1;
    while (((size_t)1 << P.hbits) < 2 * ((size_t)n_pre + kMaxCorners)) ++P.hbits;
    P.work = align256(sizeof(int4) * P.gw * P.gh + sizeof(float2) * kMaxCorners + 12 * ((size_t)1 << P.hbits));
    return P;
}

void detect_apply_plan(const DetectPlan &P, int w, int hgt, double keypoint_distance, DetectBatchFrame &F) {
    F.gs = P.gs; F.r2 = keypoint_distance * keypoint_distance;
    F.cxmax = P.cxmax; F.cymax = P.cymax;
    F.w = w; F.h = hgt; F.cap = P.cap;
    F.n_pre = P.n_pre; F.gw = P.gw; F.gh = P.gh; F.hbits = P.hbits;
}

int detect_sort_bytes(Handle *h, int n, size_t n_keys, size_t &bytes) {
    auto begin_it = thrust::make_transform_iterator(thrust::make_counting_iterator(0), SegBegin{nullptr});
    auto end_it = thrust::make_transform_iterator(thrust::make_counting_iterator(0), SegEnd{nullptr});
    bytes = 0;
    CK(h, cub::DeviceSegmentedRadixSort::SortKeysDescending(nullptr, bytes, (const unsigned long long *)nullptr,
                                                            (unsigned long long *)nullptr, (int)n_keys, n, begin_it, end_it, 0, 64));
    return 0;
}

int detect_run(Handle *h, const DetectBatchFrame *d_frm, int n, int max_w, int max_h, const unsigned long long *keys,
               unsigned long long *sorted, size_t n_keys, uint8_t *sort_tmp, size_t sort_bytes, size_t smem) {
    cudaStream_t st = h->stream;
    harris_response_kernel<<<dim3((max_w + kTX - 1) / kTX, (max_h + kTY - 1) / kTY, n), dim3(kTX, kTY), 0, st>>>(0.04f, d_frm);
    nms_compact_kernel<<<dim3((max_w + 31) / 32, (max_h + 7) / 8, n), dim3(32, 8), 0, st>>>(1.0e-3, d_frm);
    h->launches += 2;
    size_t tmp = sort_bytes;
    CK(h, cub::DeviceSegmentedRadixSort::SortKeysDescending(
              sort_tmp, tmp, keys, sorted, (int)n_keys, n,
              thrust::make_transform_iterator(thrust::make_counting_iterator(0), SegBegin{d_frm}),
              thrust::make_transform_iterator(thrust::make_counting_iterator(0), SegEnd{d_frm}), 0, 64, st));
    ++h->launches;
    if (smem > 48 * 1024)
        CK(h, cudaFuncSetAttribute(detect_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    detect_select_kernel<<<n, kSelectThreads, smem, st>>>(d_frm);
    ++h->launches;
    CK(h, cudaGetLastError());
    return 0;
}

int batch_detect_impl(Handle *h, int n, const pvio_b200_detect_request *reqs, double clahe_clip, int tiles_x, int tiles_y) {
    if (n < 0 || n > kMaxBatchDetect) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: bad request count");
    if (n == 0) return 0;
    if (!reqs || clahe_clip < 0.0) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: bad arguments");
    const bool do_clahe = clahe_clip > 0.0;
    const KltBatchState &B = h->kltb;
    std::vector<const uint8_t *> cached(n, nullptr);
    std::vector<const SlotLens *> lens(n, nullptr);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_detect_request &a = reqs[i];
        if (a.slot < 0 || a.slot > kMaxBatchSlot) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: slot out of range");
        if (a.width < 8 || a.height < 8 || a.n_existing < 0 || a.max_out < 0 || a.keypoint_distance <= 0.0 || !a.n_out ||
            (a.n_existing > 0 && !a.existing) || (a.max_out > 0 && !a.keypoints_out))
            return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: bad arguments");
        if (a.frame_id && (size_t)a.slot < B.slots.size()) {
            const KltPyramids &s = B.slots[a.slot];
            if (s.w == a.width && s.h == a.height)
                for (int k = 0; k < 2; ++k)
                    if (s.pyr_id[k] == a.frame_id && s.pyr_clahe[k] == clahe_clip) cached[i] = s.pyr[k].d;
        }
        if (cached[i]) continue;
        if (!a.image) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: frame not cached in its slot and no pixels given");
        if (a.stride < a.width) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: bad stride");
        if (do_clahe && (tiles_x < 1 || tiles_y < 1 || a.width % tiles_x || a.height % tiles_y))
            return fail(h, PVIO_B200_EINVAL, "clahe: the image size must be a multiple of the tile grid");
        lens[i] = slot_lens(B, a.slot);
        if (lens[i] && (lens[i]->w != a.width || lens[i]->h != a.height))
            return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: the frame shape differs from the slot's lens");
    }

    // sizes: per frame its key segment and its working area; the staging and the scratch of the call
    struct Plan : DetectPlan {
        size_t pix_off, eq_off, und_off, resp_off, work_off;
        int key_off;
    };
    std::vector<Plan> plan(n);
    size_t n_keys = 0, n_pre = 0, pix_bytes = 0, eq_bytes = 0, und_bytes = 0, resp_bytes = 0, smem = 0;
    int n_eq = 0, n_lens = 0, max_w = 0, max_h = 0, eq_w = 0, eq_h = 0, und_w = 0, und_h = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_detect_request &a = reqs[i];
        Plan &P = plan[i];
        static_cast<DetectPlan &>(P) = detect_plan(a.width, a.height, a.keypoint_distance, a.n_existing);
        const size_t px = (size_t)a.width * a.height;
        P.key_off = (int)std::min<size_t>(n_keys, INT_MAX);
        n_keys += P.cap;
        n_pre += P.n_pre;
        if (P.work <= kSelectSmem) smem = std::max(smem, P.work);
        P.resp_off = resp_bytes;
        resp_bytes += align256(sizeof(float) * px);
        max_w = std::max(max_w, a.width); max_h = std::max(max_h, a.height);
        if (!cached[i]) {
            P.pix_off = pix_bytes;
            pix_bytes += align256(px);
            if (do_clahe) {
                P.eq_off = eq_bytes;
                eq_bytes += align256(px);
                ++n_eq;
                eq_w = std::max(eq_w, a.width); eq_h = std::max(eq_h, a.height);
            }
            if (lens[i]) {
                P.und_off = und_bytes;
                und_bytes += align256(px);
                ++n_lens;
                und_w = std::max(und_w, a.width); und_h = std::max(und_h, a.height);
            }
        }
    }
    const int n_kf = do_clahe ? n_eq : n_lens;     // frames CLAHE or the remap read: those with a lens first
    if (n_keys > (size_t)INT_MAX) return fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: too many pixels in one call");
    size_t work_bytes = 0;
    for (auto &P : plan)
        if (P.work > smem) { P.work_off = work_bytes; work_bytes += P.work; }

    // staging: frame descriptors, remap / CLAHE descriptors, counters, presets, pixels (uploaded) | results (downloaded);
    // device scratch: responses | keys | sorted keys | equalised frames | CLAHE tables | working areas | sort temporaries |
    // undistorted frames
    const size_t tiles = do_clahe ? (size_t)tiles_x * tiles_y : 0;
    size_t cub_bytes = 0;
    TRY(detect_sort_bytes(h, n, n_keys, cub_bytes));
    DetectBatchState &D = h->detectb;
    Stage S(D.stage, &D.scratch);
    const auto sFrm = S.add<DetectBatchFrame>(Stage::kUp, n);
    const auto sKf = S.add<KltBatchFrame>(Stage::kUp, n_kf);
    const auto sCnt = S.add<int>(Stage::kUp, 2 * n);
    const auto sPre = S.add<double2>(Stage::kUp, n_pre);
    const auto sPix = S.add<uint8_t>(Stage::kUp, pix_bytes);
    const auto sRes = S.add<DetectResult>(Stage::kDown, n);
    const auto sResp = S.add<uint8_t>(Stage::kScratch, resp_bytes);
    const auto sKeys = S.add<unsigned long long>(Stage::kScratch, n_keys);
    const auto sSorted = S.add<unsigned long long>(Stage::kScratch, n_keys);
    const auto sEq = S.add<uint8_t>(Stage::kScratch, eq_bytes);
    const auto sLut = S.add<uint8_t>(Stage::kScratch, tiles * 256 * n_eq);
    const auto sWork = S.add<uint8_t>(Stage::kScratch, work_bytes);
    const auto sCub = S.add<uint8_t>(Stage::kScratch, cub_bytes);
    const auto sUnd = S.add<uint8_t>(Stage::kScratch, und_bytes);
    TRY(S.place(h));

    DetectBatchFrame *frm = S.host(sFrm);
    KltBatchFrame *kf = S.host(sKf);
    double2 *pre = S.host(sPre);
    memset(S.host(sCnt), 0, sizeof(int) * 2 * n);
    size_t p = 0;
    int q_lens = 0, q_plain = n_lens;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_detect_request &a = reqs[i];
        const Plan &P = plan[i];
        const uint8_t *img = cached[i];
        if (!img) {
            uint8_t *dst = S.host(sPix) + P.pix_off;
            for (int y = 0; y < a.height; ++y) memcpy(dst + (size_t)y * a.width, a.image + (size_t)y * a.stride, a.width);
            uint8_t *up = S.dev(sPix) + P.pix_off;
            img = up;
            if (do_clahe || lens[i]) {        // raw pixels: remap and / or CLAHE into the detector's scratch
                const int q = lens[i] ? q_lens++ : q_plain++;
                KltBatchFrame &K = kf[q];
                memset(&K, 0, sizeof(K));
                K.raw = up;
                if (lens[i]) {
                    K.lens_src = up; K.m1 = lens[i]->m1(); K.m2 = lens[i]->m2();
                    K.raw = S.dev(sUnd) + P.und_off;
                }
                K.levels = 1;
                K.w[0] = a.width; K.h[0] = a.height;
                img = K.raw;
                if (do_clahe) {
                    K.lut = S.dev(sLut) + (size_t)q * tiles * 256;
                    K.pyr = S.dev(sEq) + P.eq_off;
                    klt_clahe_params(a.width, a.height, clahe_clip, tiles_x, tiles_y, K.tw, K.th, K.clip, K.lut_scale);
                    img = K.pyr;
                }
            }
        }
        DetectBatchFrame &F = frm[i];
        memset(&F, 0, sizeof(F));
        F.img = img;
        F.resp = reinterpret_cast<float *>(S.dev(sResp) + P.resp_off);
        F.keys = S.dev(sKeys) + P.key_off;
        F.sorted = S.dev(sSorted) + P.key_off;
        F.counters = S.dev(sCnt) + 2 * i;
        F.pre = S.dev(sPre) + p;
        for (int j = 0; j < a.n_existing; ++j) pre[p++] = make_double2(a.existing[2 * j], a.existing[2 * j + 1]);
        F.work = P.work > smem ? S.dev(sWork) + P.work_off : nullptr;
        F.res = S.dev(sRes) + i;
        detect_apply_plan(P, a.width, a.height, a.keypoint_distance, F);
        F.key_off = P.key_off;
    }

    cudaStream_t st = h->stream;
    TRY(S.upload(h));
    if (n_lens > 0) undistort_frames(h, S.dev(sKf), n_lens, und_w, und_h);
    if (n_eq > 0) klt_batch_clahe(h, S.dev(sKf), n_eq, tiles_x, tiles_y, eq_w, eq_h);
    TRY(detect_run(h, S.dev(sFrm), n, max_w, max_h, S.dev(sKeys), S.dev(sSorted), n_keys, S.dev(sCub), cub_bytes, smem));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(st));

    // per request: the corners, and the keypoints the mask keeps, in order
    const DetectResult *rr = S.host(sRes);
    bool overflow = false;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_detect_request &a = reqs[i];
        const DetectResult &R = rr[i];
        const int ng = R.n_gftt;
        if (a.n_gftt) *a.n_gftt = ng;
        int m = 0;
        for (int j = 0; j < ng; ++j) {
            const unsigned idx = R.corner[j], y = idx / (unsigned)a.width, x = idx - y * (unsigned)a.width;
            if (a.gftt_out) { a.gftt_out[2 * j] = (float)x; a.gftt_out[2 * j + 1] = (float)y; }
            if (!((R.mask[j >> 5] >> (j & 31)) & 1u)) continue;
            if (m < a.max_out) { a.keypoints_out[2 * m] = (double)x; a.keypoints_out[2 * m + 1] = (double)y; }
            ++m;
        }
        *a.n_out = m;
        overflow |= m > a.max_out;
    }
    return overflow ? fail(h, PVIO_B200_EINVAL, "batch_detect_keypoints: an output array is too small") : 0;
}

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
    DetectStage &S = *reinterpret_cast<DetectStage *>(d.stage.h);
    DetectStage *dS = reinterpret_cast<DetectStage *>(d.stage.d);
    memset(&S, 0, sizeof(S));
    const uint8_t *src = klt_cached_level0(h, frame_id, width, height, clahe_clip);
    const bool clahe = !src && clahe_clip > 0.0;
    if (!src) {
        if (!image || stride < width) return fail(h, PVIO_B200_EINVAL, "detect_keypoints: frame not cached and no pixels given");
        for (int y = 0; y < height; ++y) memcpy(d.img.h + (size_t)y * width, image + (size_t)y * stride, width);
        if (clahe) {
            TRY(reserve(h, d.lut, (size_t)tiles_x * tiles_y * 256, kDevice));
            KltBatchFrame &K = S.clahe;
            K.raw = d.raw.d; K.lut = d.lut.d; K.pyr = d.img.d;
            K.levels = 1; K.w[0] = width; K.h[0] = height;
            klt_clahe_params(width, height, clahe_clip, tiles_x, tiles_y, K.tw, K.th, K.clip, K.lut_scale);
        }
        CK(h, cudaMemcpyAsync(clahe ? d.raw.d : d.img.d, d.img.h, px, cudaMemcpyHostToDevice, h->stream));
        src = d.img.d;
    }
    DetectBatchFrame &F = S.frame;
    F.img = src; F.resp = d.resp.d; F.keys = d.keys.d; F.counters = dS->counters;
    F.w = width; F.h = height; F.cap = d.cap;
    CK(h, cudaMemcpyAsync(dS, &S, sizeof(S), cudaMemcpyHostToDevice, h->stream));
    if (clahe) klt_batch_clahe(h, &dS->clahe, 1, tiles_x, tiles_y, width, height);
    harris_response_kernel<<<dim3((width + kTX - 1) / kTX, (height + kTY - 1) / kTY), dim3(kTX, kTY), 0, h->stream>>>(0.04f, &dS->frame);
    nms_compact_kernel<<<dim3((width + 31) / 32, (height + 7) / 8), dim3(32, 8), 0, h->stream>>>(1.0e-3, &dS->frame);
    h->launches += 2;
    CK(h, cudaMemcpyAsync(S.counters, dS->counters, sizeof(int) * 2, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    const int n = std::min(S.counters[1], d.cap);
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
