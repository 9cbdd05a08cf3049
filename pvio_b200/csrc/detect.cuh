// The batched detector's device stages (detect.cu), shared with the feature tracker (feature_track.cu): the frame
// descriptor the kernels read, the per-frame result, and PoissonDiskFilter<2>::insert as a warp-collective walk over a
// hash table of cells.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "api_internal.h"

namespace pvio {

constexpr int kMaxCorners = 1000;             // GFTTDetector::create(1000, ...)

// the per-frame results of a batched detection
struct DetectResult {
    int n_gftt, pad;
    unsigned mask[(kMaxCorners + 31) / 32];   // bit j: corner j passes the Poisson filter and the 20-pixel border
    unsigned corner[kMaxCorners];             // the GFTT corners in order, as pixel indices y * w + x
};

// one frame as the kernels read it (the single call: frame 0 of one)
struct DetectBatchFrame {
    const uint8_t *img;                       // the equalised frame (a cached level 0, uploaded pixels, or CLAHE output)
    float *resp;                              // [h][w] Harris response
    unsigned long long *keys, *sorted;        // its segment of the candidate keys, unsorted / sorted descending
    int *counters;                            // [2] max response bits, candidate count
    const double2 *pre;                       // [n_pre] the frame's existing keypoints, in order
    const int *pre_count;                     // device count of pre, or nullptr: n_pre
    uint8_t *work;                            // the select kernel's working area in global memory, or nullptr: on chip
    DetectResult *res;
    double gs, r2;                            // Poisson cell size r / sqrt(2) and r^2
    double cxmax, cymax;                      // the cells of the frame's last pixel column / row (capped at 2^30)
    int w, h, cap, key_off;                   // key_off: the segment's first key
    int n_pre, gw, gh, hbits;                 // min-distance grid gw x gh; Poisson hash table of 2^hbits cells
};

// The sizes of one frame of a batched detection with at most n_pre existing keypoints
struct DetectPlan {
    int cap, n_pre, gw, gh, hbits;
    double gs, cxmax, cymax;
    size_t work;                              // bytes of the select kernel's working area
};
DetectPlan detect_plan(int w, int hgt, double keypoint_distance, int n_pre);
// the descriptor fields detect_plan fixes (the caller sets the pointers, key_off and pre_count)
void detect_apply_plan(const DetectPlan &P, int w, int hgt, double keypoint_distance, DetectBatchFrame &F);
constexpr size_t kSelectSmem = 96 * 1024;     // larger working areas go to global memory
// the sort temporaries of a batched detection over n frames with n_keys keys in all
int detect_sort_bytes(Handle *h, int n, size_t n_keys, size_t &bytes);
// Harris, non-maximum suppression, the segmented sort and the select kernel over n frames whose descriptors are at
// d_frm (device memory; counters zeroed), whose key segments lie in keys / sorted: 4 launches.  smem: the select
// kernel's dynamic shared memory.
int detect_run(Handle *h, const DetectBatchFrame *d_frm, int n, int max_w, int max_h, const unsigned long long *keys,
               unsigned long long *sorted, size_t n_keys, uint8_t *sort_tmp, size_t sort_bytes, size_t smem);

// ---- PoissonDiskFilter<2> on the device -------------------------------------------------------------------------------
// A hash table of 2^hbits cells (keys hk, values hv): cell -> index of the LAST point inserted into it.
constexpr unsigned long long kHashEmpty = ~0ull;
constexpr double kCellLimit = 1073741824.0;   // 2^30: the Poisson cell indices the host pass forms without int overflow

// Poisson cells (ix, iy) in [-2^20, 2^30 + 2] as hash keys; never kHashEmpty
__device__ __forceinline__ unsigned long long cell_key(long long ix, long long iy) {
    return ((unsigned long long)(ix + (1 << 20)) << 32) | (unsigned long long)(iy + (1 << 20));
}
__device__ __forceinline__ unsigned long long hash_slot(unsigned long long key, int hbits) {
    return (key * 0x9E3779B97F4A7C15ull) >> (64 - hbits);
}
__device__ inline int hash_find(const unsigned long long *hk, const int *hv, int hbits, unsigned long long key) {
    const unsigned long long m = (1ull << hbits) - 1;
    for (unsigned long long s = hash_slot(key, hbits);; s = (s + 1) & m) {
        const unsigned long long k = hk[s];
        if (k == key) return hv[s];
        if (k == kHashEmpty) return -1;
    }
}

// PoissonDiskFilter::insert of point (x, y), called by all 32 lanes of a warp with the same point: lane t < 25
// examines cell t + 1 of the reference's walk over the 5 x 5 block (which skips the block's first cell and examines
// the one past its end), then a vote.  A taken point becomes its cell's last point with index `self`.  pt(v) is the
// point of index v.  Returns, on every lane, whether the point was taken.
template <typename Pt>
__device__ bool poisson_insert(unsigned long long *hk, int *hv, int hbits, double gs, double r2, double x, double y,
                               int self, Pt pt) {
    const int lane = threadIdx.x & 31;
    const double fx = floor(x / gs), fy = floor(y / gs);
    // beyond 2^30 (or a NaN radius) the host's cell arithmetic overflows and its walk meets no point: no test
    const bool regular = fx <= kCellLimit && fy <= kCellLimit;
    bool near = false;
    if (regular && lane < 25) {
        const int t = lane + 1;
        const int v = hash_find(hk, hv, hbits, cell_key((long long)fx - 2 + t % 5, (long long)fy - 2 + t / 5));
        if (v >= 0) {
            const double2 p = pt(v);
            const double dx = x - p.x, dy = y - p.y;
            near = dx * dx + dy * dy < r2;
        }
    }
    const bool take = !__any_sync(0xffffffffu, near);
    if (lane == 0 && take && regular) {
        const unsigned long long key = cell_key((long long)fx, (long long)fy), hm = (1ull << hbits) - 1;
        unsigned long long s = hash_slot(key, hbits);
        while (hk[s] != kHashEmpty && hk[s] != key) s = (s + 1) & hm;
        hk[s] = key; hv[s] = self;
    }
    __syncwarp();
    return take;
}

}  // namespace pvio
