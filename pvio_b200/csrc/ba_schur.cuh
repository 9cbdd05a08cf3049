// Schur elimination of the inverse depths: last kernel of the linearise stage.
//
// lin_obs_kernel + lm_finish (ba_linearize.cuh) leave, per landmark l, the UNSCALED vectors h_lf of every frame f that
// sees it (targets: Y^T j; a free anchor: -sum_t h_lt; free frames that do not see it: zeros) in the frame-major record
// array hs[f][l][6], the pivot w_l = 1 / (H_ll + reg) with w_l g_l in lm_w, the frame mask in lm_msk, and the DIRECT
// part of the reduced system in Hred / gred.  This kernel completes what SPARSE_SCHUR does inside ceres::Solve
// (bundle_adjustor.cpp:249, solver_options.h:27) -- and, with victim_only, the landmark Schur complement of
// BundleAdjustor::marginalize_frame (bundle_adjustor.cpp:512-545):
//     S(f, g) = sum_l w_l h_lf h_lg^T  over the FREE frame pairs,   c(f) = sum_l w_l g_l h_lf,   Hred -= S,  gred -= c.
// Slabs of kSlab landmarks travel hs / lm_w / lm_msk -> shared memory as bulk copies (TMA engine: one per free frame plus
// two) into a two-slab ring signalled by mbarriers; no thread touches the records between the copy and the tiles.
// The tile phase is output stationary: a thread owns a 6 x 12 register tile (frame f x frames g0, g1; float2 pairs of
// fma.rn.f32 with the w_l h_lf element as the broadcast operand) of ONE record stream; the kThreads / T record
// streams of a CTA (T = tiles of the window) are combined at the end through a shared staging buffer, in fp64,
// deterministically.  Lanes of a warp hold DIFFERENT tiles of the SAME record, so a record is fetched from shared
// memory once per warp (lanes sharing a frame read by broadcast): the earlier 6 x 6 tiles with the k-split across
// adjacent lanes were shared-memory bound.
#pragma once
#include "ba_linearize.cuh"

namespace pvio {

constexpr int kSlab = 64;                       // landmarks per staged slab
constexpr int kSlots = 2;                       // slabs in flight per CTA (ring of bulk copies)
constexpr int kFlushVals = 39;                  // staged values per thread and pass (78 = 72 tile + 6 gradient, two passes)

template <typename real>
__host__ __device__ inline int schur_fstride(int slab) { return slab * 6 + 16 / (int)sizeof(real); }   // + 16 bytes: frames land 4 banks apart

// shared memory: fp64 sums | mbarriers | staging of the final combination | ring of (masks, pivots, frame slabs)
template <typename real>
__host__ __device__ inline size_t schur_ring_slot_bytes(int nfree) {
    return sizeof(int32_t) * kSlab + sizeof(real) * 2 * kSlab + sizeof(real) * (size_t)nfree * schur_fstride<real>(kSlab);
}
template <typename real>
__host__ __device__ inline size_t schur_smem_layout(int N, size_t *o_g, size_t *o_bar, size_t *o_tab, size_t *o_ring) {
    const size_t npairs = (size_t)N * (N + 1) / 2;
    size_t off = sizeof(double) * npairs * 36;                                  // Ss
    *o_g = off; off += sizeof(double) * (size_t)N * 6;                          // gsc
    *o_bar = off; off += 8 * (kSlots + 1);                                      // one mbarrier per ring slot + one for the direct part
    *o_tab = off; off += sizeof(int32_t) * (80 + 8);                            // per tile: f | g0 << 8 | g1 << 16 | flags << 24; then the ring's release counters
    off = (off + 127) & ~(size_t)127;
    *o_ring = off;
    return off;
}

// the staging buffer of the final combination ([kThreads][kFlushVals] real) ALIASES the ring: it is used only when no
// copy is in flight
template <typename real>
__host__ __device__ inline size_t schur_smem_bytes(int N, int nthreads, int nfree) {
    size_t a, b, c, d;
    const size_t ring = kSlots * schur_ring_slot_bytes<real>(nfree), stage = sizeof(real) * (size_t)nthreads * kFlushVals;
    return schur_smem_layout<real>(N, &a, &b, &c, &d) + (ring > stage ? ring : stage);
}

// number of 6 x 12 tiles of a window with nf free frames: row fi has fi / 2 + 1 column pairs
__host__ __device__ inline int schur_tiles(int nf) { int t = 0; for (int f = 0; f < nf; ++f) t += f / 2 + 1; return t; }

template <typename real, int kThreads, int kMinBlocks>
__global__ void __launch_bounds__(kThreads, kMinBlocks)
schur_kernel(PipeArgs a_in) {
    typedef typename Vec2<real>::type real2;
    PipeArgs a = a_in;
    const int w = a.slots ? a.slots[blockIdx.y] : blockIdx.y + a.w0;
    if (a.loop) {
        const WinCtrl &c = a.ctrl[w];
        if (c.done || c.reuse) return;
        pipe_select(a, c.buf);
    }
    const WinHdr &H = a.hdr[w];
    const int N = H.N, M = H.M;
    const int tid = threadIdx.x;
    const int npairs = N * (N + 1) / 2;
    const int FS = schur_fstride<real>(kSlab);

    extern __shared__ __align__(16) unsigned char smem_raw[];
    size_t o_g, o_bar, o_tab, o_ring;
    schur_smem_layout<real>(N, &o_g, &o_bar, &o_tab, &o_ring);
    double *Ss = reinterpret_cast<double *>(smem_raw);              // [npairs][36]
    double *gsc = reinterpret_cast<double *>(smem_raw + o_g);       // [N][6]
    uint64_t *bars = reinterpret_cast<uint64_t *>(smem_raw + o_bar);
    int32_t *ttab = reinterpret_cast<int32_t *>(smem_raw + o_tab);  // [ntile]
    int32_t *rel = ttab + 80;                                       // [kSlots] warps that are done with the slab in the slot
    real *stage = reinterpret_cast<real *>(smem_raw + o_ring);      // [kThreads][kFlushVals], aliases the ring

    const unsigned allm = (1u << N) - 1u;
    const unsigned freem = ~(unsigned)H.fixed_mask & allm;
    const int nfree = __popc(freem);
    const size_t slot_bytes = schur_ring_slot_bytes<real>(nfree);
    auto slot_msk = [&](int slot) { return reinterpret_cast<int32_t *>(smem_raw + o_ring + slot * slot_bytes); };
    auto slot_w = [&](int slot) { return reinterpret_cast<real2 *>(smem_raw + o_ring + slot * slot_bytes + sizeof(int32_t) * kSlab); };
    auto slot_h = [&](int slot) { return reinterpret_cast<real *>(smem_raw + o_ring + slot * slot_bytes + sizeof(int32_t) * kSlab + sizeof(real) * 2 * kSlab); };
    const int ntile = schur_tiles(nfree);
    const int nsub = ntile > 0 ? kThreads / ntile : 0;              // record streams of this CTA
    const int tile = ntile > 0 ? tid % ntile : 0, kk = ntile > 0 ? tid / ntile : 0;
    const bool t_active = ntile > 0 && kk < nsub;
    int fi = 0, gp = 0;                                             // free-frame indices of the tile: row fi, columns 2 gp, 2 gp + 1
    bool t_diag = false;
    if (ntile > 0) {
        int rem = tile;
        while (rem >= fi / 2 + 1) { rem -= fi / 2 + 1; ++fi; }
        gp = rem;
        t_diag = (gp == fi / 2);                                    // the tile holding block (f, f): it also owns c(f)
    }
    const int gi1 = 2 * gp + 1 <= fi ? 2 * gp + 1 : 2 * gp;          // second column frame (unused above the diagonal)
    const int bf = ntile > 0 ? __fns(freem, 0, fi + 1) : 0, bg0 = ntile > 0 ? __fns(freem, 0, 2 * gp + 1) : 0,
              bg1 = ntile > 0 ? __fns(freem, 0, gi1 + 1) : 0;
    if (tid < ntile) ttab[tid] = bf | (bg0 << 8) | (bg1 << 16) | ((2 * gp + 1 <= fi ? 1 : 0) << 24) | ((t_diag ? 1 : 0) << 25);
    const int steps_per_slab = nsub > 0 ? (kSlab + nsub - 1) / nsub : 0;

    const real *hs = reinterpret_cast<const real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    const real2 *lm_w = reinterpret_cast<const real2 *>(a.lm_w) + (size_t)w * a.Mcap;
    const int32_t *lm_msk = a.lm_msk + (size_t)w * a.Mcap;

    // slabs of this CTA: gridDim.x CTAs share a window (latency path), slab i -> CTA i mod gridDim.x
    const int n_slab_all = (M + kSlab - 1) / kSlab;
    const int n_slab = (ntile > 0 && n_slab_all > (int)blockIdx.x) ? (n_slab_all - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
    auto slab_id = [&](int i) { return (int)blockIdx.x + i * (int)gridDim.x; };
    auto issue = [&](int i) {                                       // one thread: bulk copies of slab i into ring slot i % kSlots
        const int l0 = slab_id(i) * kSlab;
        const int cnt = min(kSlab, ((M - l0) + 3) & ~3);            // copy granule: 4 records (16 bytes of masks)
        const uint32_t hb = (uint32_t)(cnt * 6 * sizeof(real)), wb = (uint32_t)(cnt * 2 * sizeof(real)), mb = (uint32_t)(cnt * 4);
        const int sl = i % kSlots;
        const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[sl]);
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(hb * (uint32_t)nfree + wb + mb) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"((uint32_t)__cvta_generic_to_shared(slot_msk(sl))), "l"(lm_msk + l0), "r"(mb), "r"(bar) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"((uint32_t)__cvta_generic_to_shared(slot_w(sl))), "l"(lm_w + l0), "r"(wb), "r"(bar) : "memory");
        unsigned fm = freem;
        for (int s = 0; s < nfree; ++s, fm &= fm - 1) {
            const int f = __ffs(fm) - 1;
            const uint32_t dst = (uint32_t)__cvta_generic_to_shared(slot_h(sl) + (size_t)s * FS);
            const real *src = hs + ((size_t)f * a.Mcap + l0) * 6;
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                         :: "r"(dst), "l"(src), "r"(hb), "r"(bar) : "memory");
        }
    };
    // Hred = D - S: when this CTA owns the window the direct part D (written by the linearise kernel) is pulled into
    // the fp64 accumulators by a bulk copy that overlaps the tile loop, the flushes subtract from it, the epilogue is
    // plain stores (no load latency at the end); several CTAs per window start from zero and finish with atomics.
    const bool exclusive = (gridDim.x == 1);
    const int npairs_cap = a.Ncap * (a.Ncap + 1) / 2;
    double *Hred_o = a.Hred + (size_t)w * npairs_cap * 36;
    double *gred_o = a.gred + (size_t)w * a.Ncap * 6;
    if (tid == 0) {
        for (int j = 0; j < kSlots + 1; ++j)
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"((uint32_t)__cvta_generic_to_shared(&bars[j])) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid < kSlots) rel[tid] = 0;
    if (!exclusive) for (int i = tid; i < npairs * 36 + N * 6; i += kThreads) Ss[i] = 0.0;          // Ss, gsc contiguous
    __syncthreads();
    if (exclusive && tid == 0) {
        const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[kSlots]);
        const uint32_t hb = (uint32_t)(npairs * 36 * sizeof(double)), gb = (uint32_t)(N * 6 * sizeof(double));
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(hb + gb) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"((uint32_t)__cvta_generic_to_shared(Ss)), "l"(Hred_o), "r"(hb), "r"(bar) : "memory");
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                     :: "r"((uint32_t)__cvta_generic_to_shared(gsc)), "l"(gred_o), "r"(gb), "r"(bar) : "memory");
    }
    bool d_ready = !exclusive;
    // Partial sums stay in `real` for at most 128 terms per thread: flush (-> fp64) after every fl_every-th slab and at the
    // end.  The staging buffer of a flush aliases the ring, so no copy may be in flight or resident across a flush
    // point.  Slab j is therefore issued at the later of two events: its slot is free (every warp is done with slab
    // j - kSlots: the LAST warp to leave that slab issues the copy -- the warps of a CTA are not held together by a barrier
    // per slab, they drift up to kSlots slabs apart) and the last flush before j is over (thread 0 issues it after the flush).
    const int fl_every = steps_per_slab > 0 ? max(1, 128 / steps_per_slab) : 1;
    const int fl_mul = (65536 + fl_every - 1) / fl_every;           // (p + 1) % fl_every == 0 without a division (p + 1 < 2^10)
    auto flush_point = [&](int p) { const int q = ((p + 1) * fl_mul) >> 16; return q * fl_every == p + 1 || p == n_slab - 1; };
    auto no_flush_in = [&](int lo, int hi) { bool b = false; for (int p = lo; p < hi; ++p) b |= flush_point(p); return !b; };
    if (tid == 0)
        for (int j = 0; j < kSlots && j < n_slab; ++j) if (no_flush_in(0, j)) issue(j);

    real2 acc[36];                               // acc[i * 6 + p]: row i of w h_f x column pair p of (h_g0 | h_g1)
    real2 accg[3];
#pragma unroll
    for (int i = 0; i < 36; ++i) acc[i] = mk2((real)0, (real)0);
#pragma unroll
    for (int i = 0; i < 3; ++i) accg[i] = mk2((real)0, (real)0);

    auto flush = [&]() {                         // all threads: partial tiles -> fp64 sums in shared memory
        if (!d_ready) {                          // the direct part must have landed in Ss / gsc
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[kSlots]);
            uint32_t done = 0;
            while (!done)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                             : "=r"(done) : "r"(bar), "r"(0u) : "memory");
            d_ready = true;
        }
#pragma unroll
        for (int pass = 0; pass < 2; ++pass) {
            real *st = stage + (size_t)tid * kFlushVals;
#pragma unroll
            for (int e = 0; e < 18; ++e) { st[2 * e] = acc[pass * 18 + e].x; st[2 * e + 1] = acc[pass * 18 + e].y; }
            const real ag[6] = {accg[0].x, accg[0].y, accg[1].x, accg[1].y, accg[2].x, accg[2].y};
#pragma unroll
            for (int e = 0; e < 3; ++e) st[36 + e] = ag[pass * 3 + e];
            __syncthreads();
            for (int e = tid; e < ntile * kFlushVals; e += kThreads) {
                const int tl = e / kFlushVals, v = e - tl * kFlushVals;
                double s = 0.0;
                for (int k = 0; k < nsub; ++k) s += (double)stage[(size_t)(k * ntile + tl) * kFlushVals + v];
                const int tt = ttab[tl];                                    // owner tile of this value
                const int f = tt & 0xff;
                if (v < 36) {
                    const int i = pass * 3 + v / 12, c = v % 12;            // row i, column c of the 6 x 12 tile
                    const int g = c >= 6 ? (tt >> 16) & 0xff : (tt >> 8) & 0xff;
                    if (c < 6 || ((tt >> 24) & 1)) Ss[pair_idx(f, g) * 36 + i * 6 + (c % 6)] -= s;
                } else if ((tt >> 25) & 1) {
                    gsc[f * 6 + pass * 3 + (v - 36)] -= s;
                }
            }
            __syncthreads();
        }
#pragma unroll
        for (int i = 0; i < 36; ++i) acc[i] = mk2((real)0, (real)0);
#pragma unroll
        for (int i = 0; i < 3; ++i) accg[i] = mk2((real)0, (real)0);
    };

    for (int i = 0; i < n_slab; ++i) {
        {   // wait for slab i
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[i % kSlots]);
            const uint32_t parity = (uint32_t)((i / kSlots) & 1);
            uint32_t done = 0;
            while (!done)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                             : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        }
        const int cnt = min(kSlab, M - slab_id(i) * kSlab);
        if (t_active) {
            const int32_t *mk = slot_msk(i % kSlots);
            const real2 *wv = slot_w(i % kSlots);
            const real *buf = slot_h(i % kSlots);
            const real *pf = buf + (size_t)fi * FS, *pg0 = buf + (size_t)(2 * gp) * FS, *pg1 = buf + (size_t)gi1 * FS;
            // running pointers: one add per stream step instead of index arithmetic per operand
            const int32_t *mp = mk + kk;
            const real2 *wp = wv + kk;
            const real2 *hf = reinterpret_cast<const real2 *>(pf + kk * 6), *g0 = reinterpret_cast<const real2 *>(pg0 + kk * 6),
                        *g1 = reinterpret_cast<const real2 *>(pg1 + kk * 6);
            const unsigned need_f = 1u << bf, need_g = (1u << bg0) | (1u << bg1);
            for (int s = kk; s < cnt; s += nsub, mp += nsub, wp += nsub, hf += 3 * nsub, g0 += 3 * nsub, g1 += 3 * nsub) {
                const unsigned m = (unsigned)*mp;
                if (!(m & need_f) || !(m & need_g)) continue;
                const real2 ws = *wp;
                const real2 f01 = hf[0], f23 = hf[1], f45 = hf[2];
                const real2 gv[6] = {g0[0], g0[1], g0[2], g1[0], g1[1], g1[2]};
                const real2 wf01 = bmul(ws.x, f01), wf23 = bmul(ws.x, f23), wf45 = bmul(ws.x, f45);
                const real fv[6] = {wf01.x, wf01.y, wf23.x, wf23.y, wf45.x, wf45.y};
#pragma unroll
                for (int ii = 0; ii < 6; ++ii)
#pragma unroll
                    for (int p = 0; p < 6; ++p) acc[ii * 6 + p] = bfma(fv[ii], gv[p], acc[ii * 6 + p]);
                if (t_diag) {
                    accg[0] = bfma(ws.y, f01, accg[0]); accg[1] = bfma(ws.y, f23, accg[1]); accg[2] = bfma(ws.y, f45, accg[2]);
                }
            }
        }
        if (flush_point(i)) {
            __syncthreads();                                        // slab i consumed by everybody, nothing in flight
            flush();
            if (tid == 0) {
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                for (int j = i + 1; j <= i + kSlots && j < n_slab; ++j) if (no_flush_in(i + 1, j)) issue(j);
            }
        } else {
            __syncwarp();
            if ((tid & 31) == 0) {
                const int sl = i % kSlots;
                __threadfence_block();
                if (atomicAdd(&rel[sl], 1) == kThreads / 32 - 1) {  // last warp out of slab i: its slot takes slab i + kSlots
                    rel[sl] = 0;
                    const int j = i + kSlots;
                    if (j < n_slab && no_flush_in(i + 1, j)) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        issue(j);
                    }
                }
            }
        }
    }
    // ---- reduced system out: Ss / gsc hold D - S (one CTA per window) or -S (several)
    if (exclusive) {
        if (!d_ready) {                          // no slab at all: still wait for the copy before leaving
            const uint32_t bar = (uint32_t)__cvta_generic_to_shared(&bars[kSlots]);
            uint32_t done = 0;
            while (!done)
                asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
                             : "=r"(done) : "r"(bar), "r"(0u) : "memory");
        }
        if (n_slab > 0) {
            for (int e = tid; e < npairs * 36; e += kThreads) Hred_o[e] = Ss[e];
            for (int e = tid; e < N * 6; e += kThreads) gred_o[e] = gsc[e];
        }
    } else {
        for (int e = tid; e < npairs * 36; e += kThreads) { const double v = Ss[e]; if (v != 0.0) atomicAdd(&Hred_o[e], v); }
        for (int e = tid; e < N * 6; e += kThreads) { const double v = gsc[e]; if (v != 0.0) atomicAdd(&gred_o[e], v); }
    }
}

}  // namespace pvio
