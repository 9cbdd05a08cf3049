// pvio_b200_batch_feature_track: the per-frame step of FeatureTracker::work (feature_tracker.cpp:77-99) for many
// sequences, with each slot's newest keypoints kept on the device (KltBatchState::kps).
//
//   ft_guess_kernel   one thread per keypoint: the LK input apply_k(z) and the initial guess
//                     apply_k(hnormalized(q [z; 1])) of frame.cpp:90-103, in fp64 without contraction, as floats
//   (klt.cu)          the batched tracker's stages: pyramids, LK + border, F-RANSAC schedules, hypotheses, the host
//                     replay, the winners' masks
//   ft_thin_kernel    one CTA per sequence: the F-RANSAC mask applied, the track-length-ordered Poisson-disk thinning
//                     of frame.cpp:108-130 (std::sort restated in introsort.cuh, PoissonDiskFilter::insert from
//                     detect.cuh), the survivors compacted in previous-frame order
//   (detect.cu)       Harris, NMS, the segmented sort and the select kernel on the new frame's cached level 0, with the
//                     survivors as the existing keypoints (frame.cpp:72-86)
//   ft_commit_kernel  one warp per sequence: the detections appended
// Compiled with -fmad=false: the reference's fp64 arithmetic is not contracted.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "detect.cuh"
#include "introsort.cuh"
#include "klt_border.cuh"
#include "quat.cuh"

namespace pvio {
namespace {

constexpr int kThinThreads = 128;
constexpr int kMaxFeatureFrames = 32767;      // the batched tracker's pair limit

// one sequence of a call as the kernels read it (uploaded before the tracker's stages)
struct FtSeq {
    const double2 *z_prev;                    // the slot's newest keypoints (normalised) and their births
    const int *birth_prev;
    double2 *z_next;                          // the slot's other buffer: this frame's keypoints
    int *birth_next;
    double2 *pre;                             // [n_prev] scratch: the survivors in pixels, the detector's presets
    double2 *out_z;                           // [out_cap] download staging: keypoints, prev_index
    int *out_prev;
    int *head;                                // [6] download staging: n, counts[4], survivors (the presets' count)
    uint8_t *work;                            // the thinning's working area in global memory, or nullptr: on chip
    double kp[4], kn[4];                      // fx, fy, cx, cy of the previous and the new frame
    double q[4];                              // delta_key_q (use_q)
    double gs, r2;                            // Poisson cell size r / sqrt(2), r^2
    int use_q, n_prev, first, prev_no;        // first: its first point in the tracker's arrays; prev_no: the previous
    int map_frames, out_cap, hbits, w;        //   frame's number (births count in these)
    int *prev_next;                           // the slot's other buffer: this frame's prev_index
};

// the F-RANSAC outcome of one sequence (uploaded after the replay)
struct FtFm {
    const unsigned *mask;                     // the winner's mask words (bit k: the k-th point LK kept), or nullptr
    int clear, pad;                           // RANSAC ran and kept nothing
};

// the thinning's working area: the (index, track length) pairs, the status, the hash table of the Poisson filter
inline size_t thin_work_bytes(int n, int hbits) {
    auto a16 = [](size_t x) { return (x + 15) & ~(size_t)15; };
    return a16(sizeof(int2) * n) + a16((size_t)n) + 12 * ((size_t)1 << hbits);
}

__global__ void ft_guess_kernel(const FtSeq *seqs, const int *pair_of, float *prev_pts, float *next_pts, int n_pts) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_pts) return;
    const FtSeq &s = seqs[pair_of[p]];
    const double2 z = s.z_prev[p - s.first];
    const float px = (float)(z.x * s.kp[0] + s.kp[2]), py = (float)(z.y * s.kp[1] + s.kp[3]);
    prev_pts[2 * p] = px; prev_pts[2 * p + 1] = py;
    if (s.use_q) {
        const double v[3] = {z.x, z.y, 1.0};
        double y[3];
        bw_qrot(s.q, v, y);
        const double hx = y[0] / y[2], hy = y[1] / y[2];
        next_pts[2 * p] = (float)(hx * s.kn[0] + s.kn[2]);
        next_pts[2 * p + 1] = (float)(hy * s.kn[1] + s.kn[3]);
    } else {                                  // opencv_image.cpp:91-96: the guess is the current position
        next_pts[2 * p] = px; next_pts[2 * p + 1] = py;
    }
}

// std::sort's comparator of frame.cpp:116-118: longer tracks first
struct LongerTrack {
    __host__ __device__ bool operator()(const int2 &a, const int2 &b) const { return a.y > b.y; }
};

// frame.cpp:105-137 after LK, the border test and F-RANSAC, for sequence blockIdx.x.  Warp 0 applies the mask and lists
// the keypoints that take part in the thinning (status set and a track: born before the previous frame) with their
// track lengths; thread 0 sorts them; warp 0 runs the Poisson filter in that order on the tracked pixel positions and
// compacts the survivors in previous-frame order.
__global__ void __launch_bounds__(kThinThreads) ft_thin_kernel(const FtSeq *seqs, const FtFm *fms, const float *next_pts,
                                                               const uint8_t *status) {
    extern __shared__ __align__(16) uint8_t smem[];
    const FtSeq &s = seqs[blockIdx.x];
    const FtFm fm = fms[blockIdx.x];
    const int n = s.n_prev, tid = threadIdx.x, lane = tid & 31;
    uint8_t *work = s.work ? s.work : smem;
    int2 *list = reinterpret_cast<int2 *>(work);
    uint8_t *st = work + ((sizeof(int2) * n + 15) & ~(size_t)15);
    unsigned long long *hk = reinterpret_cast<unsigned long long *>(st + ((n + 15) & ~15));
    const unsigned long long hcap = 1ull << s.hbits;
    int *hv = reinterpret_cast<int *>(hk + hcap);
    for (unsigned long long i = tid; i < hcap; i += kThinThreads) { hk[i] = kHashEmpty; hv[i] = -1; }
    for (int k = tid; k < n; k += kThinThreads) st[k] = status[s.first + k] != 0;
    __syncthreads();
    if (tid >= 32) return;
    const float *pos = next_pts + 2 * (size_t)s.first;

    // the F-RANSAC mask (bit r: the r-th point LK kept), then the list of the thinning
    int c_lk = 0, c_fm = 0, m = 0;
    for (int base = 0; base < n; base += 32) {
        const int k = base + lane;
        bool on = k < n && st[k];
        const unsigned kept = __ballot_sync(0xffffffffu, on);
        if (on) {
            const int r = c_lk + __popc(kept & ((1u << lane) - 1u));
            if (fm.clear || (fm.mask && !((fm.mask[r >> 5] >> (r & 31)) & 1u))) on = false;
            st[k] = on;
        }
        c_lk += __popc(kept);
        const int birth = k < n ? s.birth_prev[k] : 0;
        const bool tracked = on && birth < s.prev_no;
        const unsigned in = __ballot_sync(0xffffffffu, tracked);
        if (tracked) list[m + __popc(in & ((1u << lane) - 1u))] = make_int2(k, min(s.prev_no - birth + 1, s.map_frames));
        c_fm += __popc(__ballot_sync(0xffffffffu, on));
        m += __popc(in);
    }
    __syncwarp();
    if (lane == 0) gcc_sort(list, m, LongerTrack());
    __syncwarp();
    auto point = [pos](int v) { return make_double2((double)pos[2 * v], (double)pos[2 * v + 1]); };
    for (int j = 0; j < m; ++j) {
        const int k = list[j].x;
        const double2 p = point(k);
        const bool take = poisson_insert(hk, hv, s.hbits, s.gs, s.r2, p.x, p.y, k, point);
        if (lane == 0 && !take) st[k] = 0;
        __syncwarp();
    }

    // the survivors in previous-frame order: remove_k in the new frame's K, the presets apply_k of that
    int ns = 0;
    for (int base = 0; base < n; base += 32) {
        const int k = base + lane;
        const bool on = k < n && st[k];
        const unsigned kept = __ballot_sync(0xffffffffu, on);
        if (on) {
            const int j = ns + __popc(kept & ((1u << lane) - 1u));
            const double x = (double)pos[2 * k], y = (double)pos[2 * k + 1];
            const double2 z = make_double2((x - s.kn[2]) / s.kn[0], (y - s.kn[3]) / s.kn[1]);
            s.pre[j] = make_double2(z.x * s.kn[0] + s.kn[2], z.y * s.kn[1] + s.kn[3]);
            if (j < s.out_cap) {                  // always, by the capacity bound; the host reports a breach
                s.z_next[j] = z; s.birth_next[j] = s.birth_prev[k]; s.prev_next[j] = k;
                s.out_z[j] = z; s.out_prev[j] = k;
            }
        }
        ns += __popc(kept);
    }
    if (lane == 0) { s.head[1] = c_lk; s.head[2] = c_fm; s.head[3] = ns; s.head[5] = ns; }
}

// Frame::detect_keypoints' append (frame.cpp:78-85): the detector's keypoints after the survivors, for sequence
// blockIdx.x (one warp)
__global__ void ft_commit_kernel(const FtSeq *seqs, const DetectResult *res) {
    const FtSeq &s = seqs[blockIdx.x];
    const DetectResult &R = res[blockIdx.x];
    const int lane = threadIdx.x, ns = s.head[5], ng = R.n_gftt;
    int m = 0;
    for (int base = 0; base < ng; base += 32) {
        const int j = base + lane;
        const bool on = j < ng && ((R.mask[j >> 5] >> (j & 31)) & 1u);
        const unsigned kept = __ballot_sync(0xffffffffu, on);
        if (on) {
            const int i = ns + m + __popc(kept & ((1u << lane) - 1u));
            const unsigned idx = R.corner[j], y = idx / (unsigned)s.w, x = idx - y * (unsigned)s.w;
            const double2 z = make_double2(((double)x - s.kn[2]) / s.kn[0], ((double)y - s.kn[3]) / s.kn[1]);
            if (i < s.out_cap) {
                s.z_next[i] = z; s.birth_next[i] = s.prev_no + 1; s.prev_next[i] = -1;
                s.out_z[i] = z; s.out_prev[i] = -1;
            }
        }
        m += __popc(kept);
    }
    if (lane == 0) { s.head[0] = ns + m; s.head[4] = m; }
}

// track_camera's prediction: delta_key_q of frame.cpp:98, (cam_q^* imu_q dq imu_q^* cam_q)^* with the extrinsics of the
// sequence's window slot and dq of its step-1 IMU record, each product eigen_qmul (uncontracted: this unit is built
// with -fmad=false), written into the staged FtSeq before ft_guess_kernel reads it
__global__ void ft_predict_kernel(FtSeq *seqs, int n, FtPredict p) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const WinConst &c = p.cst[p.slot[(size_t)i * p.slot_stride]];
    const double *dq = p.rec + (size_t)i * kImuStride + 1;
    const double cq[4] = {-c.cam_q[0], -c.cam_q[1], -c.cam_q[2], c.cam_q[3]};
    const double iq[4] = {-c.imu_q[0], -c.imu_q[1], -c.imu_q[2], c.imu_q[3]};
    double u[4], v[4];
    eigen_qmul(cq, c.imu_q, u);
    eigen_qmul(u, dq, v);
    eigen_qmul(v, iq, u);
    eigen_qmul(u, c.cam_q, v);
    const double q[4] = {-v[0], -v[1], -v[2], v[3]};
    for (int k = 0; k < 4; ++k) { seqs[i].q[k] = q[k]; p.q_out[4 * (size_t)i + k] = q[k]; }
    seqs[i].use_q = 1;
}

}  // namespace

// Every request is checked, and each gets its previous frame's keypoint count and its output bound.  outputs: the
// keypoints, prev_index and n_keypoints arrays are required.
int ft_check(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
             double keypoint_distance, bool outputs, FtRun &run) {
    if (n < 1 || n > kMaxFeatureFrames) return fail(h, PVIO_B200_EINVAL, "batch_feature_track: bad frame count");
    if (!frames || !(keypoint_distance > 0.0) || !std::isfinite(keypoint_distance))
        return fail(h, PVIO_B200_EINVAL, "batch_feature_track: bad arguments");
    KltBatchState &B = h->kltb;
    const double gs = keypoint_distance / std::sqrt(2.0);
    std::vector<uint8_t> taken;
    std::vector<int> &n_prev = run.n_prev;
    n_prev.assign(n, 0);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        TRY(take_slot(h, taken, a.slot, "batch_feature_track"));
        if (a.width < kKltMinFrame || a.height < kKltMinFrame || a.stride < a.width || !a.frame_id || !a.image ||
            a.map_frames < 0 || (outputs && (!a.keypoints || !a.prev_index || !a.n_keypoints)))
            return fail(h, PVIO_B200_EINVAL, "batch_feature_track: bad shape, stride, frame id, pixels or outputs");
        if (!(a.fx != 0.0 && a.fy != 0.0 && std::isfinite(a.fx) && std::isfinite(a.fy) && std::isfinite(a.cx) &&
              std::isfinite(a.cy)))
            return fail(h, PVIO_B200_EINVAL, "batch_feature_track: bad K");
        const double cells = (std::floor(a.width / gs) + 1.0) * (std::floor(a.height / gs) + 1.0);
        if ((double)a.max_keypoints < cells + 2.0 * kMaxCorners)
            return fail(h, PVIO_B200_EINVAL, "batch_feature_track: max_keypoints below cells + 2000");
        if (a.map_frames == 0) continue;
        const SlotKeypoints *K = (size_t)a.slot < B.kps.size() ? &B.kps[a.slot] : nullptr;
        const KltPyramids *c = (size_t)a.slot < B.slots.size() ? &B.slots[a.slot] : nullptr;
        bool cached = false;
        if (K && K->live && c && c->w == a.width && c->h == a.height)
            for (int k = 0; k < 2; ++k) cached |= c->pyr_id[k] == K->frame_id && c->pyr_clahe[k] == opt.clahe_clip;
        if (!cached) return fail(h, PVIO_B200_EINVAL, "batch_feature_track: the slot's newest frame is not in its cache");
        if (K->frame_id == a.frame_id) return fail(h, PVIO_B200_EINVAL, "batch_feature_track: the frame id is the slot's newest");
        n_prev[i] = K->n;
    }
    if (taken.size() > B.kps.size()) B.kps.resize(taken.size());
    run.out_cap.resize(n);
    for (int i = 0; i < n; ++i)
        run.out_cap[i] = (int)std::min<long long>(frames[i].max_keypoints, (long long)n_prev[i] + kMaxCorners);
    return 0;
}

// The tracker's stages (klt_batch_track) with the points written by ft_guess_kernel right after its upload (pred, when
// given: after ft_predict_kernel has written each sequence's delta_key_q); after its replay one H2D copy (masks'
// outcome, detector descriptors, zeroed counters), ft_thin_kernel, the detector's 4 launches, ft_commit_kernel, one D2H
// copy of every output, a synchronise.  No slot's keypoints change.
int ft_run(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
           double keypoint_distance, const FtPredict *pred, FtRun &run) {
    KltBatchState &B = h->kltb;
    const double gs = keypoint_distance / std::sqrt(2.0);
    const std::vector<int> &n_prev = run.n_prev;

    // the tracker's pairs: a new sequence has no previous frame and no points
    std::vector<KltBatchItem> items(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        const uint64_t prev_id = a.map_frames > 0 ? B.kps[a.slot].frame_id : 0;
        items[i] = KltBatchItem{a.slot, a.width, a.height, a.stride, n_prev[i], prev_id, a.frame_id, nullptr, a.image,
                                nullptr, nullptr};
    }

    // sizes.  Per sequence: outputs of at most n_prev + 1000 keypoints (survivors and detections), the thinning's
    // working area, the detector's plan with at most n_prev presets.
    struct Plan {
        DetectPlan det;
        int out_cap, hbits, key_off;
        size_t work, work_off, out_off, resp_off;
    };
    std::vector<Plan> plan(n);
    size_t out_bytes = 0, n_keys = 0, resp_bytes = 0, det_work = 0, thin_work = 0, det_smem = 0, thin_smem = 0, n_pre = 0;
    int max_w = 0, max_h = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        Plan &P = plan[i];
        P.out_cap = run.out_cap[i];
        P.out_off = out_bytes;
        out_bytes += align256((sizeof(double2) + sizeof(int)) * (size_t)P.out_cap);
        P.hbits = 1;
        while (((size_t)1 << P.hbits) < 2 * (size_t)std::max(n_prev[i], 1)) ++P.hbits;
        P.work = thin_work_bytes(n_prev[i], P.hbits);
        if (P.work <= kSelectSmem) thin_smem = std::max(thin_smem, P.work);
        P.det = detect_plan(a.width, a.height, keypoint_distance, n_prev[i]);
        if (P.det.work <= kSelectSmem) det_smem = std::max(det_smem, P.det.work);
        P.key_off = (int)n_keys;
        n_keys += P.det.cap;
        P.resp_off = resp_bytes;
        resp_bytes += align256(sizeof(float) * a.width * a.height);
        n_pre += n_prev[i];
        max_w = std::max(max_w, a.width); max_h = std::max(max_h, a.height);
    }
    if (n_keys > (size_t)INT_MAX) return fail(h, PVIO_B200_EINVAL, "batch_feature_track: too many pixels in one call");
    for (auto &P : plan) {
        P.work_off = 0;
        if (P.work > thin_smem) { P.work_off = thin_work; thin_work += P.work; }
    }
    for (auto &P : plan)
        if (P.det.work > det_smem) det_work += P.det.work;
    size_t sort_bytes = 0;
    TRY(detect_sort_bytes(h, n, n_keys, sort_bytes));

    // staging: sequences (uploaded first) | F-RANSAC outcomes, detector descriptors, counters (uploaded after the replay) |
    // heads, outputs (downloaded); device scratch: presets | thinning areas | responses | keys | sorted keys | select
    // areas | sort temporaries | results
    Stage stage(B.fstage, &B.fscratch);
    const auto sSeq = stage.add<FtSeq>(Stage::kUp, n);
    const auto sFm = stage.add<FtFm>(Stage::kUp, n);
    const auto sDet = stage.add<DetectBatchFrame>(Stage::kUp, n);
    const auto sCnt = stage.add<int>(Stage::kUp, 2 * n);
    const auto sHead = stage.add<int>(Stage::kDown, 8 * n);
    const auto sOut = stage.add<uint8_t>(Stage::kDown, out_bytes);
    const auto sPre = stage.add<double2>(Stage::kScratch, n_pre);
    const auto sThin = stage.add<uint8_t>(Stage::kScratch, thin_work);
    const auto sResp = stage.add<uint8_t>(Stage::kScratch, resp_bytes);
    const auto sKeys = stage.add<unsigned long long>(Stage::kScratch, n_keys);
    const auto sSorted = stage.add<unsigned long long>(Stage::kScratch, n_keys);
    const auto sWork = stage.add<uint8_t>(Stage::kScratch, det_work);
    const auto sSort = stage.add<uint8_t>(Stage::kScratch, sort_bytes);
    const auto sRes = stage.add<DetectResult>(Stage::kScratch, n);
    TRY(stage.place(h));
    // each slot's other buffer holds this frame's keypoints
    for (int i = 0; i < n; ++i) {
        SlotKeypoints &K = B.kps[frames[i].slot];
        const int b = run.staged ? 2 : 1 - K.cur;
        // the staged buffer rotates through all three: sized for the stated bound, so each is allocated once
        const size_t need = std::max<size_t>(run.staged ? frames[i].max_keypoints : plan[i].out_cap, 1024);
        if (K.cap[b] < (size_t)plan[i].out_cap) {
            TRY(alloc(h, K.buf[b], SlotKeypoints::bytes(need), kDevice));
            K.cap[b] = need;
        }
    }

    FtSeq *seq = stage.host(sSeq);
    size_t pre = 0, dwork = 0;                // pre: the call's points
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        const Plan &P = plan[i];
        const SlotKeypoints &K = B.kps[a.slot];
        FtSeq &S = seq[i];
        memset(&S, 0, sizeof(S));
        const int cb = K.cur, nb = run.staged ? 2 : 1 - K.cur;
        S.z_prev = K.z(cb);
        S.birth_prev = K.birth(cb);
        S.z_next = K.z(nb);
        S.birth_next = K.birth(nb);
        S.prev_next = K.prev(nb);
        S.pre = stage.dev(sPre) + pre;
        S.out_z = reinterpret_cast<double2 *>(stage.dev(sOut) + P.out_off);
        S.out_prev = reinterpret_cast<int *>(stage.dev(sOut) + P.out_off + sizeof(double2) * P.out_cap);
        S.head = stage.dev(sHead) + 8 * i;
        S.work = P.work > thin_smem ? stage.dev(sThin) + P.work_off : nullptr;
        S.kp[0] = K.fx; S.kp[1] = K.fy; S.kp[2] = K.cx; S.kp[3] = K.cy;
        S.kn[0] = a.fx; S.kn[1] = a.fy; S.kn[2] = a.cx; S.kn[3] = a.cy;
        S.use_q = a.predict_q != nullptr;
        if (a.predict_q) memcpy(S.q, a.predict_q, sizeof(S.q));
        S.gs = gs; S.r2 = keypoint_distance * keypoint_distance;
        S.n_prev = n_prev[i];
        S.prev_no = a.map_frames > 0 ? K.frame_no : K.frame_no + 1;   // a new sequence: nothing is older than its frame
        S.map_frames = a.map_frames;
        S.out_cap = P.out_cap; S.hbits = P.hbits; S.w = a.width;
        S.first = (int)pre;                   // the tracker's points are the sequences' in order
        pre += n_prev[i];
    }

    cudaStream_t st = h->stream;
    const FtSeq *d_seq = stage.dev(sSeq);
    TRY(stage.upload(h, sSeq));
    if (pred) {
        ft_predict_kernel<<<(n + 127) / 128, 128, 0, st>>>(stage.dev(sSeq), n, *pred);
        ++h->launches;
        CK(h, cudaGetLastError());
    }
    KltDevicePoints dev;
    dev.write_points = [&](Handle *hh, float *prev_pts, float *next_pts, const int *pair_of) -> int {
        ft_guess_kernel<<<(unsigned)((pre + 255) / 256), 256, 0, st>>>(d_seq, pair_of, prev_pts, next_pts, (int)pre);
        ++hh->launches;
        return 0;
    };
    KltBatchResults &r = run.r;
    TRY(klt_batch_track(h, n, items.data(), opt, &dev, r));

    // after the replay: each sequence's F-RANSAC outcome and detector descriptor, on the frame just cached
    FtFm *fm = stage.host(sFm);
    DetectBatchFrame *det = stage.host(sDet);
    memset(stage.host(sCnt), 0, sizeof(int) * 2 * n);
    dwork = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        const Plan &P = plan[i];
        fm[i] = FtFm{r.mask[i], r.clear[i], 0};
        const KltPyramids &s = B.slots[a.slot];
        const uint8_t *img = nullptr;
        for (int k = 0; k < 2; ++k)
            if (s.pyr_id[k] == a.frame_id && s.pyr_clahe[k] == opt.clahe_clip) img = s.pyr[k].d;
        DetectBatchFrame &F = det[i];
        memset(&F, 0, sizeof(F));
        F.img = img;
        F.resp = reinterpret_cast<float *>(stage.dev(sResp) + P.resp_off);
        F.keys = stage.dev(sKeys) + P.key_off;
        F.sorted = stage.dev(sSorted) + P.key_off;
        F.counters = stage.dev(sCnt) + 2 * i;
        F.pre = seq[i].pre;
        F.pre_count = seq[i].head + 5;
        F.work = P.det.work > det_smem ? stage.dev(sWork) + dwork : nullptr;
        if (P.det.work > det_smem) dwork += P.det.work;
        F.res = stage.dev(sRes) + i;
        detect_apply_plan(P.det, a.width, a.height, keypoint_distance, F);
        F.key_off = P.key_off;
    }
    TRY(stage.upload(h, sFm, sCnt));
    if (thin_smem > 48 * 1024)
        CK(h, cudaFuncSetAttribute(ft_thin_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)thin_smem));
    ft_thin_kernel<<<n, kThinThreads, thin_smem, st>>>(d_seq, stage.dev(sFm), r.next, r.status);
    ++h->launches;
    TRY(detect_run(h, stage.dev(sDet), n, max_w, max_h, stage.dev(sKeys), stage.dev(sSorted), n_keys, stage.dev(sSort),
                   sort_bytes, det_smem));
    ft_commit_kernel<<<n, 32, 0, st>>>(d_seq, stage.dev(sRes));
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(stage.download(h));
    CK(h, cudaStreamSynchronize(st));
    run.count.resize(n);
    run.out_off.resize(n);
    run.prev_no.resize(n);
    run.head = reinterpret_cast<const uint8_t *>(stage.host(sHead));
    run.out = stage.host(sOut);
    for (int i = 0; i < n; ++i) {
        run.count[i] = stage.host(sHead)[8 * i];
        run.out_off[i] = plan[i].out_off;
        run.prev_no[i] = seq[i].prev_no;
    }
    return 0;
}

// The outputs (keypoints and prev_index where given), and each slot's newest frame is now this one
int ft_finish(Handle *h, int n, const pvio_b200_feature_frame *frames, const FtRun &run) {
    KltBatchState &B = h->kltb;
    bool overflow = false;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_feature_frame &a = frames[i];
        const int *hd = reinterpret_cast<const int *>(run.head) + 8 * i;
        const int m = hd[0], cap = run.out_cap[i];
        overflow |= m > cap;
        const int w = std::min(m, cap);
        if (a.keypoints) memcpy(a.keypoints, run.out + run.out_off[i], sizeof(double2) * w);
        if (a.prev_index) memcpy(a.prev_index, run.out + run.out_off[i] + sizeof(double2) * cap, sizeof(int) * w);
        *a.n_keypoints = m;
        if (a.counts) memcpy(a.counts, hd + 1, sizeof(int32_t) * 4);
        if (a.info) memcpy(a.info, &run.r.info[4 * (size_t)i], sizeof(int32_t) * 4);
        SlotKeypoints &K = B.kps[a.slot];
        K.prev_frame_id = a.map_frames > 0 ? K.frame_id : 0;     // map_frames == 0: the link to the previous frame goes
        K.prev_n = a.map_frames > 0 ? K.n : 0;
        if (a.map_frames == 0) ++K.gen;
        if (run.staged) {
            std::swap(K.buf[1 - K.cur], K.buf[2]);
            std::swap(K.cap[1 - K.cur], K.cap[2]);
        }
        K.cur = 1 - K.cur;
        K.n = w;
        K.live = true;
        K.frame_no = run.prev_no[i] + 1;
        K.frame_id = a.frame_id;
        K.fx = a.fx; K.fy = a.fy; K.cx = a.cx; K.cy = a.cy;
    }
    return overflow ? fail(h, PVIO_B200_EINVAL, "batch_feature_track: more keypoints than the stated bound") : 0;
}

int batch_feature_track_impl(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
                             double keypoint_distance) {
    if (n == 0) return 0;
    FtRun run;
    TRY(ft_check(h, n, frames, opt, keypoint_distance, true, run));
    TRY(ft_run(h, n, frames, opt, keypoint_distance, nullptr, run));
    return ft_finish(h, n, frames, run);
}

}  // namespace pvio
