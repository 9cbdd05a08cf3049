// Frame-major observation table, built on the device once per upload.
//
// The shim (and the ABI) hand over the reprojection blocks the way bundle_adjustor.cpp:142-161 walks them: by
// landmark.  The sweeps want them by (target frame, anchor frame): then a warp's 32 residual blocks share both
// poses.  One CTA per window: count per (chunk, frame), scan, place -- deterministic (within a segment the
// blocks stay in landmark order), no host work, no extra host->device bytes.
#pragma once
#include "ba_types.h"

namespace pvio {

struct FobsArgs : BatchArrays {      // obs -> fz, flm, seg
    int w0;
    const int32_t *slots;            // may be NULL: CTA b builds window slots[b] instead of w0 + b
};

__host__ __device__ __forceinline__ int seg_index(int t, int a) { return t * (t - 1) / 2 + a; }

__global__ void __launch_bounds__(256) fobs_build_kernel(FobsArgs a) {
    const int w = a.slots ? a.slots[blockIdx.x] : blockIdx.x + a.w0;
    const WinHdr &H = a.hdr[w];
    const int N = H.N, nch = H.n_chunks;
    const int tid = threadIdx.x, lane = tid & 31, wv = tid >> 5;
    __shared__ int cnt[kMaxChunks][kMaxFrames];      // entries of (chunk, target); then their first position
    __shared__ int segb[kMaxSeg + 1];
    const LmRec *lms = a.lms + (size_t)w * a.Mcap;
    const ObsRec *obs = a.obs + (size_t)w * a.Kcap;
    for (int ch = wv; ch < nch; ch += 8) {
        const int c = H.chunk_meta[ch] & 0xff;
        const unsigned m = lane < c ? lm_mask(lms[H.chunk_begin[ch] + lane].meta) : 0u;
        for (int t = 0; t < N; ++t) {
            const unsigned b = __ballot_sync(0xffffffffu, (m >> t) & 1u);
            if (lane == 0) cnt[ch][t] = __popc(b);
        }
    }
    for (int i = tid; i <= kMaxSeg; i += 256) segb[i] = 0;
    __syncthreads();
    // segment sizes: thread per target frame walks the chunks (anchors are sorted, chunks of one anchor adjacent)
    if (tid < N) {
        const int t = tid;
        for (int ch = 0; ch < nch; ++ch) {
            const int an = H.chunk_meta[ch] >> 8;
            if (an < t) segb[seg_index(t, an)] += cnt[ch][t];
        }
    }
    __syncthreads();
    if (tid == 0) {                                   // exclusive scans over <= 120 segments: positions and rows of 32
        int32_t *sg = a.seg + (size_t)w * kSegTab;
        int pos = 0, row = 0;
        const int nsp = N * (N - 1) / 2;
        for (int sp = 0; sp <= kMaxSeg; ++sp) {
            const int len = sp < nsp ? segb[sp] : 0;
            segb[sp] = pos;
            sg[sp] = pos;
            sg[kMaxSeg + 1 + sp] = row;
            pos += len;
            row += (len + 31) >> 5;
        }
    }
    __syncthreads();
    if (tid < N) {                                    // first position of every (chunk, target)
        const int t = tid;
        int run = 0, prev = -1;
        for (int ch = 0; ch < nch; ++ch) {
            const int an = H.chunk_meta[ch] >> 8;
            if (an != prev) { run = 0; prev = an; }
            const int c = cnt[ch][t];
            cnt[ch][t] = (an < t ? segb[seg_index(t, an)] : 0) + run;
            run += c;
        }
    }
    __syncthreads();
    float2 *fz = a.fz + (size_t)w * a.Kcap;
    FLm *flm = a.flm + (size_t)w * a.Kcap;
    for (int ch = wv; ch < nch; ch += 8) {
        const int c = H.chunk_meta[ch] & 0xff;
        const int l = H.chunk_begin[ch] + lane;
        LmRec lr;
        lr.meta = 0; lr.obs_begin = 0;
        if (lane < c) lr = lms[l];
        const unsigned m = lane < c ? lm_mask(lr.meta) : 0u;
        for (int t = 0; t < N; ++t) {
            const unsigned b = __ballot_sync(0xffffffffu, (m >> t) & 1u);
            if ((m >> t) & 1u) {
                const int pos = cnt[ch][t] + __popc(b & ((1u << lane) - 1u));
                const ObsRec o = obs[lr.obs_begin + __popc(m & ((1u << t) - 1u))];
                fz[pos] = make_float2(o.zx, o.zy);
                flm[pos] = (FLm)l;
            }
        }
    }
}

}  // namespace pvio
