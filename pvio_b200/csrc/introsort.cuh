// std::sort as libstdc++ (GCC) implements it, restated so that the device orders elements exactly as the reference's
// host code does.  std::sort is not stable: which of two equal elements comes first depends on the algorithm, and the
// reference's track-length sort (frame.cpp:108-130) lets that order decide which of two close keypoints survives.
//
// introsort: partition while the range is longer than 16 elements, pivot = median of (first + 1, middle, last - 1)
// moved to the first position, Hoare-style unguarded partition; after 2 floor(log2 n) levels a range is heap-sorted
// instead; one final insertion sort over the whole array (guarded over the first 16, unguarded after).
// Single-threaded; `less` is the comparator std::sort is given.  Compiles for the host (tests) and the device.
#pragma once

namespace pvio {
namespace gcc_sort_detail {

template <typename T>
__host__ __device__ inline void swap_(T &a, T &b) { T t = a; a = b; b = t; }

// std::__adjust_heap / std::__push_heap
template <typename T, typename Less>
__host__ __device__ void adjust_heap(T *first, int hole, int len, T value, Less less) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (less(first[child], first[child - 1])) --child;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    int parent = (hole - 1) / 2;
    while (hole > top && less(first[parent], value)) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}

// std::__partial_sort(first, last, last): std::__make_heap, then std::__sort_heap
template <typename T, typename Less>
__host__ __device__ void heap_sort(T *first, int len, Less less) {
    if (len < 2) return;
    for (int parent = (len - 2) / 2;; --parent) {
        adjust_heap(first, parent, len, first[parent], less);
        if (parent == 0) break;
    }
    for (int last = len - 1; last > 0; --last) {
        T value = first[last];
        first[last] = first[0];
        adjust_heap(first, 0, last, value, less);
    }
}

// std::__move_median_to_first
template <typename T, typename Less>
__host__ __device__ void median_to_first(T *result, T *a, T *b, T *c, Less less) {
    if (less(*a, *b)) {
        if (less(*b, *c)) swap_(*result, *b);
        else if (less(*a, *c)) swap_(*result, *c);
        else swap_(*result, *a);
    } else if (less(*a, *c)) {
        swap_(*result, *a);
    } else if (less(*b, *c)) {
        swap_(*result, *c);
    } else {
        swap_(*result, *b);
    }
}

// std::__unguarded_partition_pivot
template <typename T, typename Less>
__host__ __device__ T *partition_pivot(T *first, T *last, Less less) {
    T *mid = first + (last - first) / 2;
    median_to_first(first, first + 1, mid, last - 1, less);
    T *lo = first + 1, *hi = last;
    while (true) {
        while (less(*lo, *first)) ++lo;
        --hi;
        while (less(*first, *hi)) --hi;
        if (!(lo < hi)) return lo;
        swap_(*lo, *hi);
        ++lo;
    }
}

// std::__unguarded_linear_insert
template <typename T, typename Less>
__host__ __device__ void linear_insert(T *last, Less less) {
    T value = *last;
    T *next = last - 1;
    while (less(value, *next)) {
        *last = *next;
        last = next;
        --next;
    }
    *last = value;
}

// std::__insertion_sort
template <typename T, typename Less>
__host__ __device__ void insertion_sort(T *first, T *last, Less less) {
    if (first == last) return;
    for (T *i = first + 1; i != last; ++i) {
        if (less(*i, *first)) {
            T value = *i;
            for (T *j = i; j != first; --j) *j = *(j - 1);
            *first = value;
        } else {
            linear_insert(i, less);
        }
    }
}

}  // namespace gcc_sort_detail

// std::sort(a, a + n, less) with libstdc++'s algorithm.  The recursion on the right part of each partition becomes an
// explicit stack.  The parts are disjoint and each is partitioned from its own contents and depth alone, so the order
// in which they are taken does not change the result.  Depths on the stack strictly decrease from bottom to top, so it
// never holds more than 2 log2 n + 1 <= 61 entries.
template <typename T, typename Less>
__host__ __device__ void gcc_sort(T *a, int n, Less less) {
    using namespace gcc_sort_detail;
    constexpr int kThreshold = 16;
    if (n < 2) return;
    int lg = 0;
    while ((n >> (lg + 1)) != 0) ++lg;                      // std::__lg
    struct Range { T *first, *last; int depth; };
    Range stack[64];
    int top = 0;
    stack[top++] = Range{a, a + n, 2 * lg};
    while (top > 0) {                                       // std::__introsort_loop
        const Range r = stack[--top];
        T *first = r.first, *last = r.last;
        int depth = r.depth;
        while (last - first > kThreshold) {
            if (depth == 0) {
                heap_sort(first, (int)(last - first), less);
                break;
            }
            --depth;
            T *cut = partition_pivot(first, last, less);
            stack[top++] = Range{cut, last, depth};
            last = cut;
        }
    }
    // std::__final_insertion_sort
    if (n > kThreshold) {
        insertion_sort(a, a + kThreshold, less);
        for (T *i = a + kThreshold; i != a + n; ++i) linear_insert(i, less);
    } else {
        insertion_sort(a, a + n, less);
    }
}

}  // namespace pvio
