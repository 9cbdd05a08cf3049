// PVIO's Ransac<> (utility/ransac.h) as the batched calls run it: the sample schedule on the device, every iteration
// evaluated speculatively, and Ransac::solve's serial acceptance rule replayed on the host over the counts.  Shared by
// pvio_b200_batch_two_view (twoview.cu) and pvio_b200_batch_window_plane_ransac (plane_ransac.cu).
#pragma once

#include <algorithm>
#include <cmath>
#include <cstdint>

namespace pvio {
namespace {

// ---- the sample schedule (random.h: LotBox over std::default_random_engine) ------------------------------------------
constexpr uint64_t kMinstdM = 2147483647u;

struct Minstd {                               // std::minstd_rand0, libstdc++'s std::default_random_engine
    uint64_t x;
    __host__ __device__ explicit Minstd(int32_t seed) {
        const uint64_t s = (uint64_t)(uint32_t)seed % kMinstdM;   // LotBox::seed takes an unsigned int
        x = s == 0 ? 1 : s;
    }
    __host__ __device__ uint64_t next() { x = x * 16807u % kMinstdM; return x; }
};

// std::uniform_int_distribution<size_t>(a, b) for a < b: the engine's range (2^31 - 3) exceeds the requested one, so
// libstdc++ downscales: rejection at `past`, then one division by `scaling`
__host__ __device__ __forceinline__ int uniform_index(Minstd &g, int a, int b) {
    const uint64_t urngrange = kMinstdM - 2, uerange = (uint64_t)(b - a) + 1;
    const uint64_t scaling = urngrange / uerange, past = uerange * scaling;
    uint64_t r;
    do r = g.next() - 1; while (r >= past);
    return a + (int)(r / scaling);
}

// Ransac::solve's draws: a fresh LotBox of n lots, `dof` draws without replacement per iteration, refill_all between
// iterations.  The last lot is taken without a draw.
__device__ void lotbox_schedule(int n, int32_t seed, int dof, int iters, int *lots, int *out) {
    for (int i = 0; i < n; ++i) lots[i] = i;
    Minstd g(seed);
    for (int it = 0; it < iters; ++it) {
        int cap = 0;
        for (int s = 0; s < dof; ++s) {
            int v;
            if (n - cap > 1) {
                const int j = uniform_index(g, cap, n - 1);
                const int t = lots[cap]; lots[cap] = lots[j]; lots[j] = t;
                v = lots[cap];
            } else {
                v = lots[n - 1];
            }
            ++cap;
            out[dof * it + s] = v;
        }
    }
}

// Ransac::solve's loop (ransac.h:59-94) over the evaluated counts: row `it` of the counts holds the model count and
// each model's inlier count (single: the inlier count of the iteration's one model).  The budget shrinks with
// pow(ratio, 5) whatever the model's DoF, as ransac.h:88 does.  Returns {inliers, iterations run, winning iteration,
// winning model}.
void ransac_replay(const int *cnt, int stride, bool single, int n, int iters, double confidence, int *res) {
    const double K = std::log(std::max(1 - confidence, 1.0e-5));
    size_t inliers = 0, iter_max = (size_t)iters, iter = 0;
    int best_it = -1, best_k = -1;
    for (; iter < iter_max; ++iter) {
        const int *row = cnt + stride * iter;
        const int nm = single ? 1 : row[0];
        for (int m = 0; m < nm; ++m) {
            const size_t c = (size_t)(single ? row[0] : row[1 + m]);
            if (c > inliers) {
                inliers = c; best_it = (int)iter; best_k = m;
                const double ratio = inliers / (double)n;
                const double N = K / std::log(1 - std::pow(ratio, 5));
                if (N < (double)iter_max) iter_max = (size_t)std::ceil(N);
            }
        }
    }
    res[0] = (int)inliers; res[1] = (int)iter; res[2] = best_it; res[3] = best_k;
}

}  // namespace
}  // namespace pvio
