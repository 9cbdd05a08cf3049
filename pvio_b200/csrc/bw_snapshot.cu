// Snapshots of the resident slots (pvio_b200_batch_window_save / restore): a sequence's window slot and tracker slot
// saved to a host blob, and restored into any slot of any handle.
#include <cmath>
#include <cstddef>
#include <memory>
#include <vector>

#include "batch_window.cuh"
#include "klt_border.cuh"

namespace pvio {

// ------------------------------------------------------------------------ snapshots (pvio_b200_batch_window_save / restore)
// A blob: SnapHead, then sections that each start at a multiple of 16 bytes, zero between them.  The host region (ids,
// frame masks, roles, per-factor sample counts: what the host mirror holds) follows the head; the device region, from
// dev0, holds what only the device keeps.  Sections of a part the blob lacks are empty.
constexpr int32_t kSnapWindow = 1, kSnapTracker = 2;
struct SnapHead {
    uint32_t magic, version;
    int64_t size;                                 // bytes of the blob
    int32_t parts;                                // kSnapWindow | kSnapTracker
    int32_t N, T, fixed, next_id, n_prior, inertial, n_planes, newest_kf, skipped;     // the window
    int32_t linked;                               // the window's link to the blob's tracker part (both parts held)
    int32_t n[2];                                 // the tracker: keypoints of its newest and its previous frame
    int32_t frame_no, w, h, levels;               //   the newest frame's number and pyramid shape (levels 0: none)
    int32_t pad[3];
    uint64_t frame_id, prev_frame_id;             //   its frame ids
    uint64_t link_frame;                          // the tracker frame id of the window's newest frame (linked)
    double K[4];                                  // fx, fy, cx, cy of the newest frame
    double clahe;                                 // the CLAHE clip its pyramid was built with
};
static_assert(sizeof(SnapHead) == 160 && offsetof(SnapHead, frame_id) == 96, "the head has no implicit padding");

// byte offsets of a blob's sections
struct SnapOff {
    int64_t ids, mask, role, nsmp, dev0;          // host region, then the start of the device region
    int64_t cst, tkp, valid, rho, qual, tz, frames, imu, pS, pe, px0, aux, smp, planes;   // window, device region
    int64_t kz, kb, kp, lvl[kMaxLevels];          // tracker: keypoints, births, prev_index (newest frame first), pyramid
    int64_t size;
};
static int64_t a16(int64_t x) { return (x + 15) & ~(int64_t)15; }

// the IMU factors of a blob's window
static int snap_factors(const SnapHead &H) { return (H.parts & kSnapWindow) && H.inertial ? std::max(H.N - 1, 0) : 0; }

// the sections of a blob with head H (its counts already in range), n_fac factors holding `rows` samples in all
static SnapOff snap_layout(const SnapHead &H, int64_t n_fac, int64_t rows) {
    const bool win = H.parts & kSnapWindow, trk = H.parts & kSnapTracker;
    const int64_t T = win ? H.T : 0, N = win ? H.N : 0, F = snap_factors(H), d = win ? 15 * (int64_t)H.n_prior : 0;
    const int64_t nk = trk ? (int64_t)H.n[0] + H.n[1] : 0;
    SnapOff o{};
    int64_t p = sizeof(SnapHead);
    auto sec = [&p](int64_t &at, int64_t bytes) { at = p; p += a16(bytes); };
    sec(o.ids, 4 * T); sec(o.mask, 4 * T); sec(o.role, T); sec(o.nsmp, 4 * F);
    o.dev0 = p;
    sec(o.cst, win ? (int64_t)sizeof(WinConst) : 0);
    sec(o.tkp, 4 * T); sec(o.valid, T); sec(o.rho, 8 * T); sec(o.qual, 8 * T); sec(o.tz, 16 * T * N);
    sec(o.frames, 8 * kFrameStride * N); sec(o.imu, 8 * kImuStride * F);
    sec(o.pS, 8 * d * d); sec(o.pe, 8 * d); sec(o.px0, 8 * kFrameStride * (d / 15));
    sec(o.aux, 8 * kImuAux * n_fac); sec(o.smp, 8 * 7 * rows); sec(o.planes, 32 * (int64_t)(win ? H.n_planes : 0));
    sec(o.kz, 16 * nk); sec(o.kb, 4 * nk); sec(o.kp, 4 * nk);
    if (trk && H.levels > 0) {
        KltPyramids k;
        klt_layout(k, H.w, H.h, H.levels);
        for (int l = 0; l < H.levels; ++l) sec(o.lvl[l], (int64_t)k.lw[l] * k.lh[l]);
    }
    o.size = p;
    return o;
}

// one record of a save or restore call as the kernels read it: its blob at byte `base` of the call's area (save: the
// area holds the device region only, so base + dev0 is where that region starts), the window slot (-1: none) and the
// tracker slot's buffers (trk 0: none)
struct SnapRec {
    SnapOff o;
    int64_t base;
    int32_t slot, N, T, F, n_prior, n_planes, fac_off, n_fac;
    int32_t rows, link, trk, levels;              // link: the rows' keypoint indices are kept (else -1)
    int32_t n[2];
    double2 *kz[2];                               // the tracker slot's keypoints, births, prev_index: newest, previous
    int32_t *kb[2], *kp[2];
    uint8_t *pyr;                                 // the newest frame's pyramid
    int64_t poff[kMaxLevels];
    int32_t lw[kMaxLevels], lh[kMaxLevels];
};
static_assert(sizeof(SnapRec) % 16 == 0, "the blob area after the records starts 16-byte aligned");
struct SnapFac { int32_t factor, n; int64_t smp; };     // a factor with samples: n rows at blob byte smp
static_assert(sizeof(SnapFac) == 16, "the blob area after the factors starts 16-byte aligned");

constexpr int kSnapThreads = 256;

template <typename T>
__device__ __forceinline__ void snap_copy(T *dst, const T *src, int64_t n) {
    for (int64_t i = threadIdx.x; i < n; i += kSnapThreads) dst[i] = src[i];
}
// zero bytes [bytes, a16(bytes)) of the section at p
__device__ __forceinline__ void snap_pad(uint8_t *p, int64_t bytes) {
    for (int64_t i = bytes; i & 15; ++i) p[i] = 0;
}
// the bytes of 4-byte word q of a 16-byte chunk below `left` bytes, the others 0
__device__ __forceinline__ unsigned snap_keep(unsigned x, int64_t left, int q) {
    const int64_t k = left - 4 * q;
    return k >= 4 ? x : k <= 0 ? 0u : x & ((1u << (8 * k)) - 1u);
}
// one pyramid level of `bytes` bytes in 16-byte copies, the last chunk's bytes past the level 0
__device__ __forceinline__ void snap_level(uint4 *dst, const uint4 *src, int64_t bytes) {
    const int64_t nc = (bytes + 15) >> 4;
    for (int64_t i = threadIdx.x; i < nc; i += kSnapThreads) {
        uint4 v = src[i];
        const int64_t left = bytes - 16 * i;
        if (left < 16) { v.x = snap_keep(v.x, left, 0); v.y = snap_keep(v.y, left, 1); v.z = snap_keep(v.z, left, 2); v.w = snap_keep(v.w, left, 3); }
        dst[i] = v;
    }
}

// One CTA per save record: the device region of its blob from the slot's track table, frames, IMU records, prior,
// samples and planes, and from the tracker slot's keypoint buffers and newest pyramid.  Keypoints of frames a row does
// not observe are written 0, keypoint indices -1 without the link, the sections' padding 0.
__global__ void __launch_bounds__(kSnapThreads) bw_save_kernel(BwArgs a, const SnapRec *recs, const SnapFac *facs,
                                                                uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    const SnapOff &o = R.o;
    uint8_t *b = area + R.base;
    if (R.slot >= 0) {
        const int w = R.slot, N = R.N, T = R.T;
        const size_t base = (size_t)w * a.Mcap;
        int32_t *kp = reinterpret_cast<int32_t *>(b + o.tkp);
        double *rho = reinterpret_cast<double *>(b + o.rho), *q = reinterpret_cast<double *>(b + o.qual);
#pragma unroll 1
        for (int r = threadIdx.x; r < T; r += kSnapThreads) {
            kp[r] = R.link ? a.tkp[base + r] : -1;
            b[o.valid + r] = a.tvalid[base + r];
            rho[r] = a.trho[base + r]; q[r] = a.tqual[base + r];
        }
        double2 *z = reinterpret_cast<double2 *>(b + o.tz);
        for (int i = threadIdx.x; i < T * N; i += kSnapThreads) {
            const int r = i / N, f = i - r * N;
            z[i] = ((a.tmask[base + r] >> f) & 1u) ? a.tz[(base + r) * a.Ncap + f] : make_double2(0.0, 0.0);
        }
        // the constants with the origin the slot's solves use (the mean frame position at its last re-layout)
        WinConst *c = reinterpret_cast<WinConst *>(b + o.cst);
        snap_copy(reinterpret_cast<double *>(c), reinterpret_cast<const double *>(&a.cst[w]),
                  (int64_t)(offsetof(WinConst, pad) / sizeof(double)));
        if (threadIdx.x == 0) c->pad = 0.0;
        const size_t dcap = 15 * (size_t)a.Ncap, d = 15 * (size_t)R.n_prior;
        snap_copy(reinterpret_cast<double *>(b + o.frames), a.frames + (size_t)w * a.Ncap * kFrameStride, (int64_t)N * kFrameStride);
        snap_copy(reinterpret_cast<double *>(b + o.imu), a.imu_data + (size_t)w * a.Ncap * kImuStride, (int64_t)R.F * kImuStride);
        snap_copy(reinterpret_cast<double *>(b + o.pS), a.prior_S + w * dcap * dcap, (int64_t)(d * d));
        snap_copy(reinterpret_cast<double *>(b + o.pe), a.prior_e + w * dcap, (int64_t)d);
        snap_copy(reinterpret_cast<double *>(b + o.px0), a.prior_x0 + (size_t)w * a.Ncap * kFrameStride, (int64_t)R.n_prior * kFrameStride);
        for (int j = 0; j < R.n_fac; ++j) {
            const SnapFac f = facs[R.fac_off + j];
            const size_t F = (size_t)w * a.Ncap + f.factor;
            snap_copy(reinterpret_cast<double *>(b + o.aux) + (size_t)j * kImuAux, a.imu_aux + F * kImuAux, kImuAux);
            snap_copy(reinterpret_cast<double *>(b + f.smp), a.imu_s + F * a.Scap * 7, (int64_t)f.n * 7);
        }
        snap_copy(reinterpret_cast<double *>(b + o.planes), a.tplane + (size_t)w * a.Pcap * 4, (int64_t)R.n_planes * 4);
        if (threadIdx.x == 0) {
            snap_pad(b + o.tkp, 4 * (int64_t)T); snap_pad(b + o.valid, T); snap_pad(b + o.rho, 8 * (int64_t)T);
            snap_pad(b + o.qual, 8 * (int64_t)T); snap_pad(b + o.pS, 8 * (int64_t)(d * d)); snap_pad(b + o.pe, 8 * (int64_t)d);
            snap_pad(b + o.aux, 8 * (int64_t)kImuAux * R.n_fac); snap_pad(b + o.smp, 56 * (int64_t)R.rows);
        }
    }
    if (R.trk) {
        const int64_t nk = (int64_t)R.n[0] + R.n[1];
        double2 *z = reinterpret_cast<double2 *>(b + o.kz);
        int32_t *kb = reinterpret_cast<int32_t *>(b + o.kb), *kp = reinterpret_cast<int32_t *>(b + o.kp);
        const int n0 = R.n[0], n1 = R.n[1];
        snap_copy(z, R.kz[0], n0); snap_copy(kb, R.kb[0], n0); snap_copy(kp, R.kp[0], n0);
        snap_copy(z + n0, R.kz[1], n1); snap_copy(kb + n0, R.kb[1], n1); snap_copy(kp + n0, R.kp[1], n1);
        if (threadIdx.x == 0) { snap_pad(b + o.kb, 4 * nk); snap_pad(b + o.kp, 4 * nk); }
        for (int l = 0; l < R.levels; ++l)
            snap_level(reinterpret_cast<uint4 *>(b + o.lvl[l]), reinterpret_cast<const uint4 *>(R.pyr + R.poff[l]),
                       (int64_t)R.lw[l] * R.lh[l]);
    }
}

// One CTA per restore record: the blob's window into the slot's track table (rows [0, T)), frames, IMU records, prior,
// samples, planes and constants; its tracker part into the tracker slot's buffers (newest frame in buffer 0) and the
// newest frame's pyramid
__global__ void __launch_bounds__(kSnapThreads) bw_restore_kernel(BwArgs a, const SnapRec *recs, const SnapFac *facs,
                                                                   const uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    const SnapOff &o = R.o;
    const uint8_t *b = area + R.base;
    if (R.slot >= 0) {
        const int w = R.slot, N = R.N, T = R.T;
        const size_t base = (size_t)w * a.Mcap;
        const int32_t *id = reinterpret_cast<const int32_t *>(b + o.ids), *kp = reinterpret_cast<const int32_t *>(b + o.tkp);
        const uint32_t *m = reinterpret_cast<const uint32_t *>(b + o.mask);
        const double *rho = reinterpret_cast<const double *>(b + o.rho), *q = reinterpret_cast<const double *>(b + o.qual);
#pragma unroll 1
        for (int r = threadIdx.x; r < T; r += kSnapThreads) {
            a.tid[base + r] = id[r]; a.tmask[base + r] = m[r]; a.trole[base + r] = static_cast<int8_t>(b[o.role + r]);
            a.tkp[base + r] = R.link ? kp[r] : -1;
            a.tvalid[base + r] = b[o.valid + r];
            a.trho[base + r] = rho[r]; a.tqual[base + r] = q[r];
        }
        const double2 *z = reinterpret_cast<const double2 *>(b + o.tz);
        for (int i = threadIdx.x; i < T * N; i += kSnapThreads) {
            const int r = i / N, f = i - r * N;
            a.tz[(base + r) * a.Ncap + f] = z[i];
        }
        const size_t dcap = 15 * (size_t)a.Ncap, d = 15 * (size_t)R.n_prior;
        snap_copy(a.frames + (size_t)w * a.Ncap * kFrameStride, reinterpret_cast<const double *>(b + o.frames), (int64_t)N * kFrameStride);
        snap_copy(a.imu_data + (size_t)w * a.Ncap * kImuStride, reinterpret_cast<const double *>(b + o.imu), (int64_t)R.F * kImuStride);
        snap_copy(const_cast<double *>(a.prior_S) + w * dcap * dcap, reinterpret_cast<const double *>(b + o.pS), (int64_t)(d * d));
        snap_copy(const_cast<double *>(a.prior_e) + w * dcap, reinterpret_cast<const double *>(b + o.pe), (int64_t)d);
        snap_copy(const_cast<double *>(a.prior_x0) + (size_t)w * a.Ncap * kFrameStride, reinterpret_cast<const double *>(b + o.px0),
                  (int64_t)R.n_prior * kFrameStride);
        for (int j = 0; j < R.n_fac; ++j) {
            const SnapFac f = facs[R.fac_off + j];
            const size_t F = (size_t)w * a.Ncap + f.factor;
            snap_copy(a.imu_aux + F * kImuAux, reinterpret_cast<const double *>(b + o.aux) + (size_t)j * kImuAux, kImuAux);
            snap_copy(a.imu_s + F * a.Scap * 7, reinterpret_cast<const double *>(b + f.smp), (int64_t)f.n * 7);
        }
        snap_copy(a.tplane + (size_t)w * a.Pcap * 4, reinterpret_cast<const double *>(b + o.planes), (int64_t)R.n_planes * 4);
        snap_copy(reinterpret_cast<double *>(&a.cst[w]), reinterpret_cast<const double *>(b + o.cst),
                  (int64_t)(sizeof(WinConst) / sizeof(double)));
    }
    if (R.trk) {
        const double2 *z = reinterpret_cast<const double2 *>(b + o.kz);
        const int32_t *kb = reinterpret_cast<const int32_t *>(b + o.kb), *kp = reinterpret_cast<const int32_t *>(b + o.kp);
        const int n0 = R.n[0], n1 = R.n[1];
        snap_copy(R.kz[0], z, n0); snap_copy(R.kb[0], kb, n0); snap_copy(R.kp[0], kp, n0);
        snap_copy(R.kz[1], z + n0, n1); snap_copy(R.kb[1], kb + n0, n1); snap_copy(R.kp[1], kp + n0, n1);
        for (int l = 0; l < R.levels; ++l)         // the level's storage is 256-byte aligned: the last chunk fits
            snap_level(reinterpret_cast<uint4 *>(R.pyr + R.poff[l]), reinterpret_cast<const uint4 *>(b + o.lvl[l]),
                       (int64_t)R.lw[l] * R.lh[l]);
    }
}

// After the re-layout of a restore (which sets each window's origin to its mean frame position), one CTA per record:
// the origin the window had when it was saved, so that its next solve or drop runs exactly as the source's would
__global__ void __launch_bounds__(32) bw_restore_origin_kernel(BwArgs a, const SnapRec *recs, const uint8_t *area) {
    const SnapRec &R = recs[blockIdx.x];
    if (R.slot < 0 || threadIdx.x >= 3) return;
    const WinConst *c = reinterpret_cast<const WinConst *>(area + R.base + R.o.cst);
    a.cst[R.slot].origin[threadIdx.x] = c->origin[threadIdx.x];
}

// a tracker slot's keypoint buffers as a SnapRec names them (the newest frame's first), and pyramid k of its cache c
// (c null or k < 0: none)
static void snap_tracker(SnapRec &r, const SlotKeypoints &K, const KltPyramids *c, int k) {
    r.trk = 1; r.n[0] = K.n; r.n[1] = K.prev_n;
    for (int j = 0; j < 2; ++j) {
        const int b = j ? 1 - K.cur : K.cur;
        r.kz[j] = K.z(b); r.kb[j] = K.birth(b); r.kp[j] = K.prev(b);
    }
    if (!c || k < 0) return;
    r.levels = c->levels; r.pyr = c->pyr[k].d;
    for (int l = 0; l < c->levels; ++l) { r.poff[l] = (int64_t)c->off[l]; r.lw[l] = c->lw[l]; r.lh[l] = c->lh[l]; }
}

// the pyramid of a tracker slot's newest frame in its cache, -1: none
static int snap_pyramid(const KltBatchState &B, int t) {
    if ((size_t)t >= B.slots.size()) return -1;
    for (int k = 0; k < 2; ++k)
        if (B.slots[t].pyr_id[k] == B.kps[t].frame_id && B.slots[t].pyr[k].d) return k;
    return -1;
}

// the kernels' record of blob H with sections o: window slot `slot` (-1: none), the tracker part when trk
static SnapRec snap_rec(const SnapHead &H, const SnapOff &o, int slot, int64_t base, int fac_off, int n_fac, int rows) {
    SnapRec r{};
    r.o = o; r.base = base; r.slot = slot; r.fac_off = fac_off;
    if (slot >= 0) {
        r.N = H.N; r.T = H.T; r.F = snap_factors(H); r.n_prior = H.n_prior; r.n_planes = H.n_planes;
        r.n_fac = n_fac; r.rows = rows;
    }
    return r;
}

// the slots of save or restore record R, each marked in its list: its window slot (-1: none) and tracker slot (-1: none),
// in range and not named by an earlier record; live: the window slot resident and the tracker slot live.  Null, or why
// the record is rejected.
static const char *snap_slots(const Handle *h, const pvio_b200_window_snapshot &R, bool live, std::vector<uint8_t> &wseen,
                              std::vector<uint8_t> &tseen) {
    if (R.slot < -1 || R.slot >= h->W || R.tracker_slot < -1 || R.tracker_slot > kMaxBatchSlot)
        return "slot or tracker slot out of range";
    if (R.slot < 0 && R.tracker_slot < 0) return "a record names neither a slot nor a tracker slot";
    if (R.slot >= 0) {
        if (live && !h->slots[R.slot].resident) return "slot not resident";
        if (wseen[R.slot]) return "a slot named twice";
        wseen[R.slot] = 1;
    }
    if (R.tracker_slot < 0) return nullptr;
    const std::vector<SlotKeypoints> &kps = h->kltb.kps;
    if (live && ((size_t)R.tracker_slot >= kps.size() || !kps[R.tracker_slot].live)) return "tracker slot not live";
    return take_slot(tseen, R.tracker_slot, "a tracker slot named twice");
}

}  // namespace pvio

using namespace pvio;

extern "C" {

int pvio_b200_batch_window_save(pvio_b200_handle hh, int n, pvio_b200_window_snapshot *records) {
    BwCall C(hh, "batch_window_save");
    if (!C.open(n, records, false)) return C.rc;
    Handle *h = C.h;
    // every record is checked and sized from the host mirrors before anything is staged
    const KltBatchState &B = h->kltb;
    std::vector<SnapHead> heads(n);
    std::vector<SnapOff> offs(n);
    std::vector<SnapRec> recs;
    std::vector<SnapFac> facs;
    std::vector<int> packed;                  // the records with data, in call order
    std::vector<uint8_t> wseen(h->W, 0), tseen;
    int64_t area = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        if (const char *why = snap_slots(h, R, true, wseen, tseen)) return C.bad(why);
        const SlotKeypoints *K = R.tracker_slot >= 0 ? &B.kps[R.tracker_slot] : nullptr;
        if (R.capacity < 0) return C.bad("negative capacity");
        SnapHead &H = heads[i];
        memset(&H, 0, sizeof(H));
        H.magic = PVIO_B200_SNAPSHOT_MAGIC; H.version = PVIO_B200_SNAPSHOT_VERSION;
        H.parts = (R.slot >= 0 ? kSnapWindow : 0) | (K ? kSnapTracker : 0);
        int n_fac = 0, rows = 0;
        if (R.slot >= 0) {
            const WinSlot &s = h->slots[R.slot];
            H.N = s.N; H.T = (int32_t)s.ids.size(); H.fixed = s.fixed; H.next_id = s.next_id; H.n_prior = s.n_prior;
            H.inertial = s.inertial; H.n_planes = s.n_planes; H.newest_kf = s.newest_kf; H.skipped = s.skipped;
            // the link, when it names the record's tracker slot, its current sequence and one of its two held
            // frames, with every row's keypoint index inside that frame's keypoints (otherwise: saved unlinked)
            const int held = !K || !s.link_frame ? -1 : s.link_frame == K->frame_id ? K->n
                                                     : s.link_frame == K->prev_frame_id ? K->prev_n : -1;
            H.linked = K && s.link && s.link_tracker == R.tracker_slot && s.link_gen == K->gen && s.link_kmax < held ? 1 : 0;
            H.link_frame = H.linked ? s.link_frame : 0;
            for (int k = 0; k < snap_factors(H); ++k)
                if (s.n_samples[k] > 0) { ++n_fac; rows += s.n_samples[k]; }
        }
        int pk = -1;
        if (K) {
            H.n[0] = K->n; H.n[1] = K->prev_n; H.frame_no = K->frame_no;
            H.frame_id = K->frame_id; H.prev_frame_id = K->prev_frame_id;
            H.K[0] = K->fx; H.K[1] = K->fy; H.K[2] = K->cx; H.K[3] = K->cy;
            pk = snap_pyramid(B, R.tracker_slot);
            if (pk >= 0) {
                const KltPyramids &c = B.slots[R.tracker_slot];
                H.w = c.w; H.h = c.h; H.levels = c.levels; H.clahe = c.pyr_clahe[pk];
            }
        }
        offs[i] = snap_layout(H, n_fac, rows);
        H.size = offs[i].size;
        if (!R.data) continue;
        if (R.capacity < H.size) return C.bad("capacity below the record's size");
        SnapRec r = snap_rec(H, offs[i], R.slot, area - offs[i].dev0, (int)facs.size(), n_fac, rows);
        r.link = H.linked;
        if (R.slot >= 0) {
            const WinSlot &s = h->slots[R.slot];
            int64_t at = offs[i].smp;
            for (int k = 0; k < snap_factors(H); ++k)
                if (s.n_samples[k] > 0) { facs.push_back(SnapFac{k, s.n_samples[k], at}); at += 56 * (int64_t)s.n_samples[k]; }
        }
        if (K) snap_tracker(r, *K, pk >= 0 ? &B.slots[R.tracker_slot] : nullptr, pk);
        recs.push_back(r);
        packed.push_back(i);
        area += H.size - offs[i].dev0;
    }
    if (!recs.empty()) {
        Stage S(h->bw.stage, &h->bw.scratch);
        const auto rc = S.up(recs);
        const auto fc = S.up(facs);
        const auto out = S.add<uint8_t>(Stage::kDown, (size_t)area);
        TRY(S.place(h, true));
        bw_save_kernel<<<(int)recs.size(), kSnapThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(fc), S.dev(out));
        TRY(launched(h, "bw_save_kernel"));
        TRY(S.download(h));
        CK(h, cudaStreamSynchronize(h->stream));
        for (size_t j = 0; j < packed.size(); ++j) {
            const int i = packed[j];
            const pvio_b200_window_snapshot &R = records[i];
            const SnapHead &H = heads[i];
            const SnapOff &o = offs[i];
            memset(R.data, 0, o.dev0);
            memcpy(R.data, &H, sizeof(H));
            if (R.slot >= 0) {
                const WinSlot &s = h->slots[R.slot];
                memcpy(R.data + o.ids, s.ids.data(), 4 * (size_t)H.T);
                memcpy(R.data + o.mask, s.mask.data(), 4 * (size_t)H.T);
                memcpy(R.data + o.role, s.role.data(), H.T);
                memcpy(R.data + o.nsmp, s.n_samples.data(), 4 * (size_t)snap_factors(H));
            }
            memcpy(R.data + o.dev0, S.host(out) + recs[j].base + o.dev0, H.size - o.dev0);
        }
    }
    for (int i = 0; i < n; ++i) records[i].size = heads[i].size;
    return 0;
}

int pvio_b200_batch_window_restore(pvio_b200_handle hh, int n, const pvio_b200_window_snapshot *records) {
    BwCall C(hh, "batch_window_restore");
    if (!C.open(n, records, false)) return C.rc;
    Handle *h = C.h;
    // every blob is checked completely before anything is staged
    std::vector<SnapHead> heads(n);
    std::vector<SnapOff> offs(n);
    std::vector<std::vector<int32_t>> nsmp(n);
    std::vector<int32_t> wslots;              // the window records' slots and their windows after the call
    std::vector<WinSlot> next;
    std::vector<uint8_t> wseen(h->W, 0), tseen;
    int smax = 0;
    bool inertial = false;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        if (const char *why = snap_slots(h, R, false, wseen, tseen)) return C.bad(why);
        if (!R.data || R.capacity < (int64_t)sizeof(SnapHead)) return C.bad("a blob shorter than its head");
        SnapHead &H = heads[i];
        memcpy(&H, R.data, sizeof(H));
        if (H.magic != PVIO_B200_SNAPSHOT_MAGIC || H.version != PVIO_B200_SNAPSHOT_VERSION) return C.bad("not a blob of this version");
        if (H.size != R.capacity) return C.bad("the declared size is not the byte count");
        if (H.parts < 1 || H.parts > 3) return C.bad("bad parts");
        const bool win = H.parts & kSnapWindow, trk = H.parts & kSnapTracker;
        if ((R.slot >= 0 && !win) || (R.tracker_slot >= 0 && !trk)) return C.bad("the record names a part the blob lacks");
        // counts, before the layout is computed from them
        if (win) {
            if (H.N < 0 || H.N > kMaxFrames || H.T < 0 || H.T > 65536 || H.n_planes < 0 || H.n_planes > h->Pcap ||
                H.n_prior < 0 || H.n_prior > H.N)
                return C.bad("window counts out of range");
            if ((H.inertial != 0 && H.inertial != 1) || (H.n_prior > 0 && !H.inertial)) return C.bad("a prior on a visual-only window");
            if ((H.newest_kf != 0 && H.newest_kf != 1) || H.skipped < 0 || H.next_id < 0 || (H.linked != 0 && H.linked != 1))
                return C.bad("bad keyframe flag, skipped-frame counter, next id or link flag");
            if (H.fixed < 0 || (H.fixed >> H.N) != 0) return C.bad("a fixed frame outside the window");
        }
        if (trk) {
            if (H.n[0] < 0 || H.n[1] < 0 || !H.frame_id || (!H.prev_frame_id && H.n[1] > 0))
                return C.bad("bad tracker counts or frame ids");
            if (!(H.K[0] != 0.0 && H.K[1] != 0.0) || !all_finite(H.K, 4)) return C.bad("bad K");
            if (H.levels != 0 &&
                (H.levels < 1 || H.levels > kMaxLevels || H.w < kKltMinFrame || H.h < kKltMinFrame || H.w > 32768 ||
                 H.h > 32768 || klt_levels(H.w, H.h, H.levels - 1) != H.levels || !std::isfinite(H.clahe) || H.clahe < 0.0))
                return C.bad("a pyramid shape the tracker does not build");
        }
        if (win && H.linked && (!trk || !H.link_frame || (H.link_frame != H.frame_id && H.link_frame != H.prev_frame_id)))
            return C.bad("a link to a frame the blob's tracker part does not hold");
        const int F = snap_factors(H);
        SnapOff o = snap_layout(H, 0, 0);
        if (R.capacity < o.dev0) return C.bad("the declared size is not the byte count");
        nsmp[i].resize(F);
        memcpy(nsmp[i].data(), R.data + o.nsmp, 4 * (size_t)F);
        int64_t rows = 0;
        int n_fac = 0, fmax = 0;
        for (int32_t c : nsmp[i]) {
            if (c < 0) return C.bad("a negative sample count");
            rows += c; n_fac += c > 0; fmax = std::max(fmax, (int)c);
        }
        if (rows > INT32_MAX) return C.bad("too many samples");
        offs[i] = o = snap_layout(H, n_fac, rows);
        if (o.size != H.size) return C.bad("the declared size is not the byte count");
        // contents
        auto rd = [&R](int64_t off, size_t k, auto *dst) { memcpy(dst, R.data + off, sizeof(*dst) * k); };
        std::vector<int32_t> kpn;                 // the tracker part's keypoints' prev_index, newest frame first
        if (trk) {
            kpn.resize((size_t)H.n[0] + H.n[1]);
            rd(o.kp, kpn.size(), kpn.data());
            for (size_t k = 0; k < kpn.size(); ++k)
                if (kpn[k] < -1 || (k < (size_t)H.n[0] && kpn[k] >= H.n[1])) return C.bad("a prev_index outside its keypoint count");
        }
        WinSlot s;
        if (win) {
            s.resident = true; s.N = H.N; s.n_prior = s.prior_resident = H.n_prior; s.fixed = H.fixed;
            s.inertial = H.inertial; s.n_planes = H.n_planes; s.next_id = H.next_id;
            s.ids.resize(H.T); s.mask.resize(H.T); s.role.resize(H.T);
            rd(o.ids, H.T, s.ids.data()); rd(o.mask, H.T, s.mask.data()); rd(o.role, H.T, s.role.data());
            for (int r = 0; r < H.T; ++r) {
                if (s.ids[r] < 0 || s.ids[r] >= H.next_id || (r > 0 && s.ids[r] <= s.ids[r - 1]))
                    return C.bad("track ids not increasing or not below the next id");
                if (s.mask[r] == 0u || (s.mask[r] >> H.N) != 0u) return C.bad("a frame mask 0 or outside the window");
                if (s.role[r] < -2 || s.role[r] >= H.n_planes) return C.bad("a role not -1, -2 or a plane of the blob");
            }
            std::vector<int32_t> tkp(H.T);
            rd(o.tkp, H.T, tkp.data());
            const int cnt = !H.linked ? 0 : H.link_frame == H.frame_id ? H.n[0] : H.n[1];
            for (int r = 0; r < H.T; ++r) {
                if (tkp[r] < -1 || tkp[r] >= cnt) return C.bad("a keypoint index outside its keypoint count");
                s.link_kmax = std::max(s.link_kmax, (int)tkp[r]);
            }
            s.newest_kf = H.newest_kf; s.skipped = H.skipped;
        }
        if (R.slot < 0) continue;
        // the target's capacities
        if (H.N > h->Ncap) return C.bad("more frames than max_frames");
        TRY(check_window(h, s));
        s.n_samples.assign(h->Ncap, 0);
        std::copy(nsmp[i].begin(), nsmp[i].end(), s.n_samples.begin());
        if (R.tracker_slot >= 0 && H.linked) {
            const KltBatchState &B = h->kltb;
            s.link = true; s.link_tracker = R.tracker_slot; s.link_frame = H.link_frame;
            s.link_gen = ((size_t)R.tracker_slot < B.kps.size() ? B.kps[R.tracker_slot].gen : 0u) + 1u;
        } else {
            s.link_kmax = -1;
        }
        smax = std::max(smax, fmax);
        inertial |= H.inertial != 0;
        wslots.push_back(R.slot);
        next.push_back(std::move(s));
    }

    // buffers, grown as the other calls grow them
    KltBatchState &B = h->kltb;
    if (!wslots.empty()) {
        TRY(ensure_bw(h));
        if (inertial) TRY(ensure_inertial(h));
        if (smax > 0) TRY(ensure_imu_store(h, smax));
        TRY(ensure_plane_tables(h, next));
    }
    if (tseen.size() > B.kps.size()) B.kps.resize(tseen.size());
    if (tseen.size() > B.slots.size()) B.slots.resize(tseen.size());
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        if (R.tracker_slot < 0) continue;
        SlotKeypoints &K = B.kps[R.tracker_slot];
        for (int b = 0; b < 2; ++b)
            if (K.cap[b] < (size_t)H.n[b]) {
                const size_t need = std::max<size_t>(H.n[b], 1024);
                TRY(alloc(h, K.buf[b], SlotKeypoints::bytes(need), kDevice));
                K.cap[b] = need;
            }
        K.cur = 0;
        KltPyramids &c = B.slots[R.tracker_slot];
        if (H.levels > 0) {
            if (c.w != H.w || c.h != H.h || c.levels != H.levels) {
                c = KltPyramids{};
                klt_layout(c, H.w, H.h, H.levels);
            }
            for (auto &p : c.pyr) TRY(reserve(h, p, c.off[c.levels], kDevice));
        }
    }

    // staging: upload the blobs (16-byte aligned, first) | records | factors | re-layout
    std::vector<SnapRec> recs(n);
    std::vector<SnapFac> facs;
    int64_t area = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        const SnapOff &o = offs[i];
        int n_fac = 0, rows = 0;
        if (R.slot >= 0) {
            int64_t at = o.smp;
            for (int k = 0; k < (int)nsmp[i].size(); ++k)
                if (nsmp[i][k] > 0) {
                    facs.push_back(SnapFac{k, nsmp[i][k], at});
                    at += 56 * (int64_t)nsmp[i][k]; ++n_fac; rows += nsmp[i][k];
                }
        }
        SnapRec &r = recs[i];
        r = snap_rec(H, o, R.slot, area, (int)facs.size() - n_fac, n_fac, rows);
        r.link = R.slot >= 0 && R.tracker_slot >= 0 && H.linked;
        if (R.tracker_slot >= 0)
            snap_tracker(r, B.kps[R.tracker_slot], H.levels > 0 ? &B.slots[R.tracker_slot] : nullptr, 0);
        r.n[0] = R.tracker_slot >= 0 ? H.n[0] : 0; r.n[1] = R.tracker_slot >= 0 ? H.n[1] : 0;
        area += H.size;
    }
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto blob = S.add<uint8_t>(Stage::kUp, (size_t)area);
    const auto rc = S.up(recs);
    const auto fc = S.up(facs);
    std::unique_ptr<Relayout> lay;
    if (!wslots.empty()) lay.reset(new Relayout(S, wslots.data(), next));
    TRY(S.place(h));
    for (int i = 0; i < n; ++i) memcpy(S.host(blob) + recs[i].base, records[i].data, heads[i].size);
    TRY(S.upload(h));
    bw_restore_kernel<<<n, kSnapThreads, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(fc), S.dev(blob));
    TRY(launched(h, "bw_restore_kernel"));
    if (lay) {
        TRY(lay->launch(h, S, true));
        bw_restore_origin_kernel<<<n, 32, 0, h->stream>>>(launch_args<BwArgs>(h), S.dev(rc), S.dev(blob));
        TRY(launched(h, "bw_restore_origin_kernel"));
    }
    CK(h, cudaStreamSynchronize(h->stream));

    // the host mirrors
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_snapshot &R = records[i];
        const SnapHead &H = heads[i];
        if (R.slot >= 0) memcpy(&h->cst.h[R.slot], R.data + offs[i].cst, sizeof(WinConst));
        if (R.tracker_slot < 0) continue;
        SlotKeypoints &K = B.kps[R.tracker_slot];
        K.n = H.n[0]; K.prev_n = H.n[1]; K.live = true; K.frame_no = H.frame_no;
        K.frame_id = H.frame_id; K.prev_frame_id = H.prev_frame_id; ++K.gen;
        K.fx = H.K[0]; K.fy = H.K[1]; K.cx = H.K[2]; K.cy = H.K[3];
        KltPyramids &c = B.slots[R.tracker_slot];
        c.pyr_id[0] = H.levels > 0 ? H.frame_id : 0; c.pyr_clahe[0] = H.clahe;
        c.pyr_id[1] = 0; c.pyr_clahe[1] = 0.0;
    }
    commit(h, wslots.data(), next);
    return 0;
}

}  // extern "C"
