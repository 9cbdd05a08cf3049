// std::sort of (keypoint index, track length) pairs with the comparator of the reference's track-length thinning
// (longer tracks first; std::sort is not stable, so the order of equal lengths is libstdc++'s), and, with
// -DWITH_RESTATED, the same through pvio_b200/csrc/introsort.cuh.  Built by oracle/feature_oracle.py.
#include <algorithm>
#include <cstddef>
#include <utility>
#include <vector>

extern "C" void std_sort_by_length(int n, const int *index, const int *length, int *out) {
    std::vector<std::pair<size_t, size_t>> v(n);
    for (int i = 0; i < n; ++i) v[i] = {(size_t)index[i], (size_t)length[i]};
    std::sort(v.begin(), v.end(), [](const auto &a, const auto &b) { return a.second > b.second; });
    for (int i = 0; i < n; ++i) out[i] = (int)v[i].first;
}

#ifdef WITH_RESTATED
#define __host__
#define __device__
#include "introsort.cuh"
extern "C" void restated_sort_by_length(int n, const int *index, const int *length, int *out) {
    std::vector<std::pair<int, int>> v(n);
    for (int i = 0; i < n; ++i) v[i] = {index[i], length[i]};
    pvio::gcc_sort(v.data(), n, [](const std::pair<int, int> &a, const std::pair<int, int> &b) { return a.second > b.second; });
    for (int i = 0; i < n; ++i) out[i] = v[i].first;
}
#endif
