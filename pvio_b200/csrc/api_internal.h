// Internal handle of libpvio_b200 (host side).  Not part of the ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <cstring>
#include <functional>
#include <map>
#include <string>
#include <tuple>
#include <utility>
#include <vector>
#include "../../include/pvio_b200.h"
#include "ba_types.h"

namespace pvio {

// Owner of one array in device memory, pinned host memory or both (the same element count on each side); move-only,
// freed with its owner.  Allocated only by alloc / reserve (below), which also record its capacity and slot stride.
template <typename T>
struct DevBuf {
    T *d = nullptr;      // device
    T *h = nullptr;      // pinned host
    size_t n = 0;        // capacity in elements: 0 until an allocation has fully succeeded
    size_t per = 0;      // arrays indexed by window slot: elements per slot
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : d(o.d), h(o.h), n(o.n), per(o.per) { o.d = o.h = nullptr; o.n = o.per = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        DevBuf t(std::move(o));
        std::swap(d, t.d); std::swap(h, t.h); std::swap(n, t.n); std::swap(per, t.per);
        return *this;
    }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() {
        if (d) cudaFree(d);
        if (h) cudaFreeHost(h);
    }
    T *slot(size_t i) const { return h + i * per; }      // pinned staging of window slot i
    T *dslot(size_t i) const { return d + i * per; }     // device array of window slot i
};
enum MemSides { kDevice = 1, kPinned = 2, kBoth = 3 };

// klt.cu: the pyramid cache of one sequence -- the finished pyramids of its last two frames.  Rebuilt (which drops the
// image cache) when the image shape or the level count changes.
constexpr int kMaxLevels = 8;
struct KltPyramids {
    int w = 0, h = 0, levels = 0;
    DevBuf<uint8_t> pyr[2];                   // both pyramids, levels packed back to back
    size_t off[kMaxLevels + 1] = {};
    int lw[kMaxLevels] = {}, lh[kMaxLevels] = {};
    // image cache: pyr[i] holds the finished pyramid of the frame with id pyr_id[i] (0: none) built with pyr_clahe[i];
    // the tracker calls with prev = the previous call's next (feature_tracker.cpp:92), so half the uploads and
    // pyramid builds of a steady-state call are skipped
    uint64_t pyr_id[2] = {0, 0};
    double pyr_clahe[2] = {0.0, 0.0};
};

// the single-call tracker: one sequence's pyramids and the staging of one frame pair.  Also rebuilt when the point
// capacity changes.
struct KltState : KltPyramids {
    int cap_pts = 0;
    DevBuf<uint8_t> stage;                    // both sides, grown: descriptors and points | positions, errors, status
    DevBuf<uint8_t> raw[2];                   // pre-CLAHE level-0 images (raw entry point only)
    DevBuf<uint8_t> lut;                      // [tiles][256] CLAHE look-up tables
    DevBuf<uint8_t> img;                      // pinned staging for both level-0 images
};

// one frame the tracker or the detector undistorts, equalises or downsamples on the device (klt.cu, detect.cu,
// undistort.cu), as the remap, CLAHE and pyrDown kernels read it: with a lens the uploaded pixels remapped into raw,
// then CLAHE from raw into level 0 of `pyr`, then pyrDown level by level
struct KltBatchFrame {
    const uint8_t *lens_src;                  // with a lens: the uploaded frame, remapped into raw through m1 / m2
    const short2 *m1;                         //   (its slot's map, SlotLens); nullptr: no lens
    const uint16_t *m2;
    uint8_t *raw;                             // level-0 pixels before CLAHE: as uploaded, or the remap's output
    uint8_t *lut;                             // [tiles][256] its CLAHE tables
    uint8_t *pyr;                             // its pyramid (the detector and clahe_impl: level 0 only)
    int levels, tw, th, clip;
    float lut_scale;
    int w[kMaxLevels], h[kMaxLevels];
    size_t off[kMaxLevels];
};
constexpr int kMaxBatchSlot = 65535;          // the sequence slots of the batched calls: 0 .. kMaxBatchSlot

// undistort.cu: the lens of one sequence slot (pvio_b200_batch_set_lens) -- OpenCV's CV_16SC2 map pair, 6 bytes per pixel
// on the device: [h][w] short2 integer source pixel, then [h][w] uint16 fraction index.  Kept apart from the slot's
// pyramids, so the tracker's shape-change rebuild of a slot leaves its lens alone.
struct SlotLens {
    int w = 0, h = 0, model = 0;              // model 0: no lens
    DevBuf<uint8_t> map;
    const short2 *m1() const { return reinterpret_cast<const short2 *>(map.d); }
    const uint16_t *m2() const { return reinterpret_cast<const uint16_t *>(map.d + (size_t)4 * w * h); }
};

// feature_track.cu: the keypoints of a slot's newest frame (pvio_b200_batch_feature_track), double-buffered so that a
// call reads buf[cur] and writes buf[1 - cur].  Each buffer: [cap] double2 normalised keypoint, then [cap] int32 birth
// (the number of the frame that detected it), then [cap] int32 prev_index (the keypoint of the frame before that it
// continues, or -1).  Right after a call buf[1 - cur] still holds the previous frame's keypoints: the link that
// pvio_b200_batch_window_mirror_frame reads (bw_frame.cu).
struct SlotKeypoints {
    DevBuf<uint8_t> buf[3];                   // buf[2]: pvio_b200_batch_window_track_camera writes the new frame here and
                                              // swaps it with buf[1 - cur] when the call commits, so that a rejected
                                              // call leaves the previous frame's keypoints as they were
    size_t cap[3] = {0, 0, 0};                // keypoints each buffer holds
    int cur = 0, n = 0;                       // newest buffer, its keypoint count
    bool live = false;                        // a sequence was started in this slot (map_frames == 0)
    int frame_no = 0;                         // the number of the newest frame (births count in these)
    uint64_t frame_id = 0;                    // its id in the slot's pyramid cache
    uint64_t prev_frame_id = 0;               // the previous frame's id, 0: none (the newest frame started the sequence)
    uint32_t gen = 0;                         // sequences started in the slot (map_frames == 0): a window link names one
    int prev_n = 0;                           // the previous frame's keypoint count (in buf[1 - cur])
    double fx = 0, fy = 0, cx = 0, cy = 0;    // its K
    static size_t bytes(size_t cap) { return (sizeof(double2) + 2 * sizeof(int)) * cap; }
    double2 *z(int b) const { return reinterpret_cast<double2 *>(buf[b].d); }
    int *birth(int b) const { return reinterpret_cast<int *>(buf[b].d + sizeof(double2) * cap[b]); }
    int *prev(int b) const { return birth(b) + cap[b]; }
};

// the batched tracker (pvio_b200_batch_track_keypoints): one pyramid cache per sequence slot, grown on demand, and
// the buffers of one call, grown to the largest call seen
struct KltBatchState {
    std::vector<KltPyramids> slots;
    std::vector<SlotKeypoints> kps;           // per slot, grown on demand by pvio_b200_batch_feature_track
    std::vector<SlotLens> lens;               // per slot, grown on demand by pvio_b200_batch_set_lens
    DevBuf<uint8_t> ustage;                   // both sides: pvio_b200_batch_undistort's descriptors and frames
    DevBuf<uint8_t> stage;                    // both sides: uploaded descriptors, frames and points | downloaded results |
                                              // winners' masks | the mask jobs the device reads in place (klt.cu)
    DevBuf<uint8_t> scratch;                  // device: CLAHE tables, RANSAC matches, schedules, models, masks (and the
                                              // LK arrays of points written on the device)
    DevBuf<uint8_t> fstage;                   // feature_track.cu, both sides: descriptors (uploaded) | outputs (downloaded)
    DevBuf<uint8_t> fscratch;                 // feature_track.cu, device: thinning, detection and commit working areas
};

// detect.cu: per-image-shape buffers of the corner detector
struct DetectState {
    int w = 0, h = 0;
    int cap = 0;                              // candidate capacity
    size_t cub_bytes = 0;
    DevBuf<uint8_t> img;                      // own copy of the image when the frame is not in the KLT cache; .h: its staging
    DevBuf<uint8_t> raw, lut;
    DevBuf<float> resp;
    DevBuf<unsigned long long> keys;
    DevBuf<unsigned long long> keys_sorted;   // both sides
    DevBuf<uint8_t> stage;                    // both sides: the frame's descriptors and counters (detect.cu: DetectStage)
    DevBuf<uint8_t> cub_tmp;
};

// detect.cu: the batched detector (pvio_b200_batch_detect_keypoints); both grown to the largest call seen
struct DetectBatchState {
    DevBuf<uint8_t> stage;                    // both sides: descriptors, counters, existing points, uploaded pixels |
                                              // per-request results
    DevBuf<uint8_t> scratch;                  // device: responses, keys, sorted keys, equalised frames, CLAHE tables,
                                              // sort temporaries, select working areas that do not fit on chip
};

// fmat.cu: the buffers of the single F-matrix RANSAC call, grown to powers of two
struct FmState {
    DevBuf<uint8_t> stage;                    // both sides: problem, matches, schedule | counts, the winner and its mask |
                                              // the mask job the device reads in place
    DevBuf<uint8_t> scratch;                  // device: the models and masks of every iteration
};

// twoview.cu: the buffers of pvio_b200_batch_two_view, grown to the largest call seen
struct TwoViewState {
    DevBuf<uint8_t> stage;                    // both sides: problems, keypoints (uploaded) | sample schedules and
                                              // per-iteration inlier counts of both RANSACs, results (downloaded)
    DevBuf<uint8_t> scratch;                  // device: lots, models of every iteration, parallax, candidate scores
};

// imu_stream.cu: the IMU stream slots (pvio_b200_batch_imu_stream).  The device keeps each slot's queues ([slot][Qcap]
// rows, live at [head, head + n) and moved to the front at the start of every call) and its ImuStreamSlot header; the
// host keeps what checking a record needs: the queue sizes after the last call, the last reading time of each stream,
// whether the slot has a latest state, and the newest frame released without one.
struct ImuStreamHost {
    bool set = false;                 // reset at least once
    bool has_state = false;
    double last_g = 0, last_a = 0;    // last gyroscope / accelerometer time (valid once n_g / n_a readings were seen)
    bool seen_g = false, seen_a = false;
    double t_drop = 0;                // newest frame time released without a state (samples up to it are dropped)
    bool dropped = false;
    int64_t g = 0, a = 0, s = 0, f = 0, k = 0;   // queue sizes: gyroscope, accelerometer, unreleased samples, pending
                                                 // frames, kept samples
};
// The latest state's covariance seed of one stream slot (pvio_b200_batch_imu_stream_set_covariance).  gen counts the
// changes of the slot's latest state (SET and CLEAR records, reset, restore); the seed holds while seed_gen == gen.
struct ImuStreamCovHost {
    int64_t gen = 0, seed_gen = -1;
    double state_t = 0;               // the latest state's time (while ImuStreamHost::has_state)
};
struct ImuStreams {
    int slots = 0;                    // slots allocated on the device
    int qcap = 0;                     // rows per queue per slot
    std::vector<ImuStreamHost> host;
    std::vector<ImuStreamCovHost> cov_host;   // sized with host
    DevBuf<uint8_t> hdr;              // [slots] ImuStreamSlot (imu_stream.cu)
    DevBuf<double> g, a, s, f, k;     // [slots][qcap][4 / 4 / 7 / 1 / 7]
    DevBuf<double> cov;               // [slots][kStreamCovStride] the seeded covariance, noise_cov and state time
    DevBuf<uint8_t> stage;            // both sides: records and events (uploaded) | outputs (downloaded)
};

// The host record of one window slot.  Its frame and landmark counts are those of the slot's host header (Handle::hdr).
// A slot holds either a window packed from the caller's arrays (api.cu: pack_window) or a resident window
// (batch_window.cu; slot 0 is also the window of pvio_b200_window_*).  Of a resident window the host keeps integers only:
// the frame count, the prior's frame count, the fixed mask, the plane count, and for every live track (rows in id order)
// its id, frame mask and role; the device keeps the track table (frame mask, role, inverse depth, fp64 keypoint per
// window frame, post-pass flags), the plane parameters and the packed window.  Of the IMU factors whose samples stay on
// the device (pvio_b200_batch_window_set_imu) the host keeps the sample count only.
// Role of a row: -1 a landmark; -2 a landmark that stays out of the marginaliser's victim set (a plane track of a plane
// with fewer than 20 tracks); p >= 0 a plane track of plane p: one plane-distance factor over all its observations.
struct WinSlot {
    bool resident = false;            // the slot changes through pvio_b200_batch_window_* (and window_*) only
    int N = 0, n_prior = 0, fixed = 0, inertial = 0, n_planes = 0;
    int32_t next_id = 0;
    std::vector<int32_t> ids;         // live tracks, increasing: row r of the device table holds track ids[r]
    std::vector<uint32_t> mask;       // frame mask of each row
    std::vector<int8_t> role;         // role of each row
    std::vector<int32_t> perm;        // packed landmark -> caller landmark; empty: the identity (always, when resident)
    int prior_resident = 0;           // frame count of the prior (S, e, x0) the marginaliser wrote on the device (0: none);
                                      // a pack naming it with prior_S == NULL keeps it, a host prior clears it
    std::vector<int32_t> n_samples;   // resident: [Ncap] per IMU factor k (frames k, k + 1) the samples it holds on the
                                      // device, 0: none (it keeps the record its edit gave it)
    // the link of the newest frame to a tracker slot (pvio_b200_batch_window_set_keypoints / mirror_frame); the device
    // keeps each row's keypoint index in that frame (BatchWindows::tkp)
    bool link = false;
    int link_tracker = -1;            // the tracker slot
    uint64_t link_frame = 0;          // the tracker's frame id of the newest frame
    uint32_t link_gen = 0;            // the tracker slot's sequence (SlotKeypoints::gen): frame ids restart with it
    int link_kmax = -1;               // the largest keypoint index a row holds, -1: none
    int newest_kf = 1;                // the newest frame is a keyframe
    int skipped = 0;                  // the tracker's skipped-frame counter (sliding_window_tracker.cpp:286)
};
struct BatchWindows {
    DevBuf<int32_t> tid;                         // [W][Mcap] track id of each row
    DevBuf<uint32_t> tmask;                      // [W][Mcap] frames observing it (0: free row)
    DevBuf<double> trho;                         // [W][Mcap] inverse depth in its anchor (lowest) frame
    DevBuf<double2> tz;                          // [W][Mcap][Ncap] fp64 keypoint per window frame
    DevBuf<uint8_t> tvalid;                      // [W][Mcap] post-pass result of the last solve
    DevBuf<double> tqual;                        // [W][Mcap]
    DevBuf<int8_t> trole;                        // [W][Mcap] role of each row (WinSlot::role)
    DevBuf<double> tplane;                       // [W][Pcap][4] plane parameters (normal, distance)
    DevBuf<int32_t> lm_row;                      // [W][Mcap] packed landmark -> row
    DevBuf<int32_t> tkp;                         // [W][Mcap] keypoint index of each row in the newest frame, -1: none
                                                 // (meaningful while the slot's link is set, WinSlot::link)
    DevBuf<uint8_t> stage;                       // both sides, grown: every call's staging (Stage)
    DevBuf<uint8_t> scratch;                     // device, grown: every call's scratch sections
    // IMU samples of the factors named by set_imu, indexed like imu_data (factor k couples frames k, k + 1); allocated
    // with the first set_imu, imu_s grown to the longest sample list seen
    int Scap = 0;                                // samples per factor in imu_s
    DevBuf<double> imu_s;                        // [W][Ncap][Scap][7] t, w xyz, a xyz
    DevBuf<double> imu_aux;                      // [W][Ncap][37] t_end, then noise [4][9] cov_w, cov_a, cov_bg, cov_ba
};

// the plane tables of the solve (api.cu: for_each_staged), allocated with the first window that has plane tracks and
// grown by ensure_planes
struct PlaneTables {
    DevBuf<double> plane_param;
    DevBuf<int32_t> pt_plane, pt_begin, pt_frame;
    DevBuf<float> pt_z;
};

struct Handle {
    int device = 0;
    int W = 1, Ncap = 0, Mcap = 0, Kcap = 0;
    int Pcap = 4, Tcap = 0, Ocap = 0;            // planes / plane tracks / plane observations per window
    cudaStream_t stream = nullptr;
    cudaStream_t stream_up = nullptr, stream_down = nullptr;   // copy streams of the pipelined host path
    std::vector<cudaStream_t> stream_c;                        // compute streams of the pipelined host path
    cudaEvent_t ev_fork = nullptr;
    cudaStream_t stream_aux = nullptr;                         // second branch of the captured single-window solve (api.cu: iteration_body)
    cudaEvent_t ev_aux_fork = nullptr, ev_aux_join = nullptr;  //   and the second stream of the split batched step
    cudaStream_t stream_mark = nullptr;                        // stage-time events of the split batched step (api.cu:
    cudaEvent_t ev_stage[2] = {nullptr, nullptr};              //   run_gn_step_split), recorded once both streams are done
    int step_parts = 0;                                        // batch_gn_step's sub-batches: 0 chosen from the batch (api.cu:
                                                               //   gn_step_parts); > 0 forced by the internal entry point
    std::vector<cudaEvent_t> ev_up, ev_done, ev_down;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    std::string err;
    int64_t launches = 0;
    std::vector<WinSlot> slots;                   // [W]
    DetectState detect;                           // detect.cu
    DetectBatchState detectb;                     // detect.cu: the batched detector, independent of detect
    size_t sys_set = 0;                           // elements between the two buffer sets of the reduced-system arrays (LinBufs)
    int sm_count = 132;                           // set from the device at create
    int smem_lim = 0;                             // dynamic shared memory the large-layout kernels opt in to (create)
    std::map<std::tuple<int, int, int>, bool> lin_part;   // (sizeof(real), N, Mp) -> the linearise sweep keeps its
                                                          // per-landmark sums in shared memory (api.cu: lin_part_fits)

    // vision (always allocated)
    DevBuf<WinHdr> hdr;
    DevBuf<WinConst> cst;
    DevBuf<ObsRec> obs;                          // landmark-major table as the shim gathers it (uploaded)
    DevBuf<float2> fz;                           // frame-major table, built on the device after every upload: keypoints
    DevBuf<FLm> flm;                             //   and landmark indices
    DevBuf<int32_t> seg;                         // [W][kSegTab]
    DevBuf<LmRec> lms;
    DevBuf<double> rho, frames;
    DevBuf<WinCtrl> ctrl;
    DevBuf<double> rho_cand, frames_cand, lm_scale, dx_lm, lm_v, dx_pose, pose_scale, v_pose;
    DevBuf<LmAux> lm_aux;
    DevBuf<unsigned char> hs;                    // [W][Ncap][Mcap][6] float (visual-only windows) or double (inertial):
    DevBuf<unsigned char> jr;                    //   unscaled h records / [W][Ncap][Mcap][2] (j.j, j.r), linearise -> Schur / update
    DevBuf<unsigned char> lm_w;                  // [W][Mcap][2] real: pivot w_l, w_l g_l
    DevBuf<int32_t> lm_msk;                      // [W][Mcap] frame mask of each landmark
    bool hs_double = false;
    DevBuf<double> frames_out, rho_out;          // pinned landing area of downloaded states (the upload staging stays intact)
    DevBuf<double> Hred;                         // reduced-system outputs of the linearise sweep, Hdd, gdir, gred and
                                                 // cost_vis included, both buffer sets (api.cu: refresh_arrays)
    DevBuf<double> acc, aux_cost;
    DevBuf<double> Hfull, gfull;                 // debug dump (single window only)
    DevBuf<uint8_t> valid;                       // post-pass results
    DevBuf<double> quality;
    // inertial / prior / planes (allocated on first use)
    bool have_inertial = false;
    DevBuf<int32_t> imu_idx, prior_frames;
    DevBuf<double> imu_data, prior_S, prior_L, prior_e, prior_x0;
    bool have_planes = false;
    PlaneTables planes;
    DevBuf<double> pt_J;                          // [W][Tcap][6 Ncap + 2] scratch of the plane block of solve_kernel
    int n_uploaded = 0;
    // ring of event triples around the linearise + Schur launches (roofline timing without host syncs)
    std::vector<cudaEvent_t> kev;
    int kev_count = 0;
    // CUDA graphs of the latency path (few windows): the whole trust-region solve / one GN iteration as ONE launch.
    // Key: (kind, n, max_iter, flags) -- no floating-point values; all scalars the kernels need live in WinCtrl.
    // Launch shapes use the handle's capacities, so a graph survives window-shape changes between keyframes.
    // Cleared whenever a device buffer is reallocated (pointers are baked into the nodes).
    typedef std::tuple<int, int, int, int> GraphKey;
    std::map<GraphKey, std::pair<cudaGraphExec_t, int>> graphs;
    bool capturing = false;
    BatchArrays arrays;                           // the device arrays above as the kernels see them (api.cu: refresh_arrays)
    KltState klt;
    KltBatchState kltb;                           // klt.cu: the batched tracker, independent of klt
    DevBuf<double> marg;                          // ba_marg.cu: scratch blocks of the marginaliser's dense kernels
    FmState fm;
    DevBuf<uint8_t> pnp;                          // pnp.cu's own staging: both sides, grown to powers of two
    BatchWindows bw;                              // batch_window.cu (empty until the first pvio_b200_batch_window_reset)
    TwoViewState tv;                              // twoview.cu
    ImuStreams imus;                              // imu_stream.cu
};

int fail(Handle *h, int code, const char *what, cudaError_t e = cudaSuccess);

// argument struct of a bundle-adjustment kernel (ba_*.cuh): the handle's array view, every per-launch field zero
template <typename Args>
Args launch_args(const Handle *h) {
    Args a{};
    static_cast<BatchArrays &>(a) = h->arrays;
    return a;
}

// pvio_b200_options with its defaults (opt may be NULL): 10 iterations, initial trust-region radius 1e4 unless a positive
// one is given, alias_bias 1, no time limit
struct SolveOptions {
    int max_iter = 10;
    double radius0 = 1e4;
    int alias_bias = 1;
    double max_time = 0.0;
};
inline SolveOptions solve_options(const pvio_b200_options *opt) {
    SolveOptions o;
    if (opt) {
        o.max_iter = opt->max_iterations;
        if (opt->initial_trust_region_radius > 0) o.radius0 = opt->initial_trust_region_radius;
        o.alias_bias = opt->alias_bias;
        o.max_time = opt->max_time;
    }
    return o;
}

#define CK(h, call)                                                        \
    do {                                                                   \
        cudaError_t e__ = (call);                                          \
        if (e__ != cudaSuccess) return fail((h), PVIO_B200_ECUDA, #call, e__); \
    } while (0)

#define TRY(x) do { int rc__ = (x); if (rc__ != 0) return rc__; } while (0)

// right after a launch of `kernel`: counts it (Handle::launches), then 0, or PVIO_B200_ECUDA with the message
// "launch of <kernel>: <error>" when the launch failed
inline int launched(Handle *h, const char *kernel) {
    ++h->launches;
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : fail(h, PVIO_B200_ECUDA, (std::string("launch of ") + kernel).c_str(), e);
}

// The one allocation routine of the library.  n elements on the given sides (MemSides), per elements per window slot.
// A buffer being replaced may still be in use by queued work, so the handle's stream is synchronised before it is freed.
// Every allocation is zeroed: device memory in stream order on the handle's stream (which every kernel of the handle
// follows), pinned memory here.  The capacity is recorded last, so a failed step leaves an empty buffer that the next
// alloc / reserve allocates again instead of a half-built one.
template <typename T>
int alloc(Handle *h, DevBuf<T> &b, size_t n, int sides, size_t per = 0) {
    if (b.d || b.h) CK(h, cudaStreamSynchronize(h->stream));
    b = DevBuf<T>();
    if (n == 0) return 0;
    const size_t bytes = n * sizeof(T);
    if (sides & kDevice) {
        CK(h, cudaMalloc(&b.d, bytes));
        CK(h, cudaMemsetAsync(b.d, 0, bytes, h->stream));
    }
    if (sides & kPinned) {
        CK(h, cudaMallocHost(&b.h, bytes));
        memset(b.h, 0, bytes);
    }
    b.n = n; b.per = per;
    return 0;
}

// grow-only: allocates only when n exceeds the capacity
template <typename T>
int reserve(Handle *h, DevBuf<T> &b, size_t n, int sides) {
    return n <= b.n ? 0 : alloc(h, b, n, sides);
}

// x rounded up to the 256-byte boundary every staging section starts on; also for sub-blocks inside a section (per-frame
// pixel blocks and the like)
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

// One batched call's staging.  Sections are declared by kind and size, then laid out kind after kind in the order of Kind,
// each on a 256-byte boundary (the largest alignment a kernel needs of one).  Upload, in/out, download and mapped sections
// go to the staging buffer (both sides), in that order, so that the call copies upload + in/out to the device in one copy
// and in/out + download back in one copy; the device reads mapped sections in place from pinned memory (unified
// addressing), and nothing copies them.  Scratch sections go to the scratch buffer (device only), which a call that
// declares none may leave out.
struct Stage {
    enum Kind { kUp, kInOut, kDown, kMapped, kScratch, kKinds };
    template <typename T>
    struct Sec { int i; };
    struct Entry { Kind kind; size_t bytes; const void *src; size_t off; };
    DevBuf<uint8_t> *buf, *scratch;
    std::vector<Entry> secs;
    size_t end[kKinds] = {};                  // after place: the end of each kind's sections in its buffer
    uint8_t *hp = nullptr, *dp = nullptr, *sp = nullptr;
    bool pow2 = false;                        // grow the buffers to powers of two (sizes that vary per call)

    explicit Stage(DevBuf<uint8_t> &stage, DevBuf<uint8_t> *scratch_buf = nullptr) : buf(&stage), scratch(scratch_buf) {}

    // n elements of kind k; src (n elements, or null): what place copies into the section
    template <typename T>
    Sec<T> add(Kind k, size_t n, const T *src = nullptr) {
        secs.push_back(Entry{k, sizeof(T) * n, src, 0});
        return Sec<T>{(int)secs.size() - 1};
    }
    template <typename T>
    Sec<T> up(const std::vector<T> &v) { return add(kUp, v.size(), v.data()); }
    template <typename T>
    T *host(Sec<T> s) const { return reinterpret_cast<T *>(hp + secs[s.i].off); }
    template <typename T>
    T *dev(Sec<T> s) const { return reinterpret_cast<T *>((secs[s.i].kind == kScratch ? sp : dp) + secs[s.i].off); }

    // lays the sections out, grows the buffers to them and copies the sources into the staging's host side; upload_now:
    // then uploads (a call that fills host sections itself uploads after that)
    int place(Handle *h, bool upload_now = false) {
        size_t o = 0;
        for (int k = 0; k < kKinds; ++k) {
            if (k == kScratch) o = 0;
            for (Entry &e : secs)
                if (e.kind == k) { e.off = o; o += align256(e.bytes); }
            end[k] = o;
        }
        if (end[kScratch] > 0 && !scratch) return fail(h, PVIO_B200_EINVAL, "internal error: scratch without a buffer");
        TRY(reserve(h, *buf, grown(end[kMapped]), kBoth));
        if (scratch) TRY(reserve(h, *scratch, grown(end[kScratch]), kDevice));
        hp = buf->h; dp = buf->d; sp = scratch ? scratch->d : nullptr;
        for (const Entry &e : secs)
            if (e.src && e.bytes) memcpy(hp + e.off, e.src, e.bytes);
        return upload_now ? upload(h) : 0;
    }
    int upload(Handle *h) const { return copy(h, 0, end[kInOut], true); }
    int download(Handle *h) const { return copy(h, end[kUp], end[kDown], false); }
    // sections a .. b (a laid out first, both in the staging buffer) in one copy: to the device after the host has
    // rewritten them, or back to the host
    template <typename A, typename B>
    int upload(Handle *h, Sec<A> a, Sec<B> b) const { return copy(h, secs[a.i].off, last(b), true); }
    template <typename A>
    int upload(Handle *h, Sec<A> a) const { return upload(h, a, a); }
    template <typename A, typename B>
    int download(Handle *h, Sec<A> a, Sec<B> b) const { return copy(h, secs[a.i].off, last(b), false); }

  private:
    size_t grown(size_t n) const {
        size_t w = n;
        if (pow2 && n > 0)
            for (w = 4096; w < n; w <<= 1) {}
        return w;
    }
    template <typename B>
    size_t last(Sec<B> b) const { return secs[b.i].off + secs[b.i].bytes; }
    // bytes [o, e) of the staging buffer to the device (up) or back to the host
    int copy(Handle *h, size_t o, size_t e, bool up) const {
        if (e > o) CK(h, up ? cudaMemcpyAsync(dp + o, hp + o, e - o, cudaMemcpyHostToDevice, h->stream)
                            : cudaMemcpyAsync(hp + o, dp + o, e - o, cudaMemcpyDeviceToHost, h->stream));
        return 0;
    }
};

// Slot s of a batched call whose slots must be distinct sequence slots (0 .. kMaxBatchSlot), marked in taken (grown to
// it); null, or why it cannot be taken: out of range, or named before (the text `twice`)
inline const char *take_slot(std::vector<uint8_t> &taken, int s, const char *twice = "a slot appears twice") {
    if (s < 0 || s > kMaxBatchSlot) return "slot out of range";
    if ((size_t)s >= taken.size()) taken.resize(s + 1, 0);
    if (taken[s]) return twice;
    taken[s] = 1;
    return nullptr;
}
// the same for call `call`: 0, or PVIO_B200_EINVAL with the message "<call>: <why>"
inline int take_slot(Handle *h, std::vector<uint8_t> &taken, int s, const char *call) {
    const char *why = take_slot(taken, s);
    return why ? fail(h, PVIO_B200_EINVAL, (std::string(call) + ": " + why).c_str()) : 0;
}

// api.cu: pack window into slot 0, copy it to the device, build the frame-major table
int pack_and_upload(Handle *h, const pvio_b200_window *w, const pvio_b200_state *s);
// api.cu: the constants of window w as the kernels read them, origin 0
WinConst win_const(const pvio_b200_window *w);
// api.cu: the summary of a solve from its window's WinCtrl (solve_seconds 0)
void fill_summary(const WinCtrl &c, pvio_b200_summary *sm);
// api.cu: linearise + Schur of the uploaded windows [0, n) with the fp64 pipeline, no loss (the marginaliser's reprojection part)
// h_slots / d_slots (may be NULL): host / device copies of a list of the n windows, instead of [0, n)
int run_marg_vision(Handle *h, int n, const int32_t *h_slots = nullptr, const int32_t *d_slots = nullptr);
// api.cu: the covariance of the n windows of a slot list (host / device copies h_slots / d_slots): the solve's
// linearise + Schur sweeps at the state with mu = 0, then cov_kernel and cov_lm_kernel (ba_cov.cuh) on the staged records.
// Four launches whatever n is.
struct CovLaunch {
    const CovRec *recs;
    const int32_t *frames;
    const CovLm *lms;
    int n_lm;
    double *cov, *var;
    int32_t *status;
    double *sig, *sig_xi;
};
int run_covariance(Handle *h, int n, const int32_t *h_slots, const int32_t *d_slots, const CovLaunch &L);
// the first three of those launches: Sigma_xi of every frame pair in L.sig_xi and each record's status, for a landmark
// kernel of the caller's (bw_query.cu: pvio_b200_batch_window_landmarks)
int run_cov_system(Handle *h, int n, const int32_t *h_slots, const int32_t *d_slots, const CovLaunch &L);
size_t cov_smem_bytes(const WinHdr &H);   // dynamic shared memory of cov_kernel for a window of this header
void drop_graphs(Handle *h);
// api.cu, for the resident batched windows (batch_window.cu)
int ensure_inertial(Handle *h);
// plane-table capacity of at least T plane tracks and O plane observations per window; growth keeps every slot's tables,
// the pinned staging and the device arrays
int ensure_planes(Handle *h, int T, int O);
// the trust-region solve of windows [0, n); named (device, [n], may be NULL): only windows with named[w] != 0 are solved,
// the others are marked finished before the first body and cost no iteration; named_h: the same on the host (the
// launches are shaped for the named windows only)
int run_named_solve(Handle *h, const pvio_b200_options *opt, int n, const uint8_t *named, const uint8_t *named_h);
int run_postpass_slots(Handle *h, int n, const int32_t *slots);   // post-pass of the n windows of a device list
// the frame-major table of the n windows slots[0 .. n) (device list), and Lambda = S^T S of their priors when prior
int launch_layout_tail(Handle *h, const int32_t *slots, int n, bool prior);
// ba_marg.cu: the marginaliser of windows [0, n) or of the list h_slots / d_slots (host / device copies of one list);
// to_slots: each new prior into its window's prior arrays
int run_marg(Handle *h, int n, int index, bool eig, bool to_slots, const int32_t *h_slots = nullptr,
             const int32_t *d_slots = nullptr);
bool marg_eig_fits(int dk);
// klt.cu
int klt_track_impl(Handle *h, const uint8_t *prev, const uint8_t *next, int width, int height, int stride,
                   const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                   int max_level, int max_iter, double eps, double clahe_clip = 0.0, int tiles_x = 0, int tiles_y = 0,
                   uint8_t *prev_eq = nullptr, uint8_t *next_eq = nullptr, uint64_t prev_id = 0, uint64_t next_id = 0, int border = 0);
int clahe_impl(Handle *h, const uint8_t *src, int width, int height, int stride, double clip, int tiles_x, int tiles_y, uint8_t *dst);
// pnp.cu: one problem's record of the PnP kernel, staged in device memory (pointers into the same staging buffer)
struct PnpArgs {
    const double *pts;      // [n][3]
    const double *z;        // [n][2]
    int n, inertial, max_iter;
    double radius0;
    WinConst wc;            // extrinsics, sqrt_inv_cov, cauchy_a
    double last[16];
    const double *imu_rec;  // [288] device (null without inertial)
    double *frame;          // [16] in/out (device)
    double *out;            // [8] iterations, accepted, termination, usable, initial_cost, final_cost, radius, mu
};
static_assert(sizeof(PnpArgs) % sizeof(double) == 0, "records are staged as whole 8-byte words");
// the PnP kernel on n records already on the device, between the events ev0 / ev1: 256 threads for n == 1, otherwise 128
int launch_pnp(Handle *h, int n, const PnpArgs *d_recs);
// the summary of one problem from the kernel's 8 words PnpArgs::out, with the launch's time ms
void pnp_summary(const double *out, float ms, pvio_b200_summary *s);
int pnp_solve_impl(Handle *h, const pvio_b200_pnp_problem *pb, double *frame, const pvio_b200_options *opt,
                   pvio_b200_summary *summary);
int batch_pnp_solve_impl(Handle *h, int n, const pvio_b200_pnp_problem *pbs, double *frames, int64_t frames_stride,
                         const pvio_b200_options *opt, pvio_b200_summary *summaries);
// klt.cu: the level count of a width x height frame's pyramid for maxLevel max_level; the level sizes and offsets of an
// empty cache for w x hgt frames with `levels` levels
int klt_levels(int width, int height, int max_level);
void klt_layout(KltPyramids &k, int w, int hgt, int levels);
// klt.cu / detect.cu
const uint8_t *klt_cached_level0(Handle *h, uint64_t frame_id, int width, int height, double clahe_clip);
// klt.cu, used by detect.cu: cv::CLAHE's per-tile constants of a w x h frame, and CLAHE of n_frames frames (frames in
// device memory; each equalises raw into level 0 of pyr) as 2 launches whose grids cover max_w x max_h
void klt_clahe_params(int w, int hgt, double clip_limit, int tiles_x, int tiles_y, int &tw, int &th, int &clip, float &lut_scale);
void klt_batch_clahe(Handle *h, const KltBatchFrame *frames, int n_frames, int tiles_x, int tiles_y, int max_w, int max_h);
// undistort.cu: the map of one lens (pvio_b200_undistort_map); the lens of a slot, or nullptr; the remap of n_frames
// frames (descriptors in device memory, each with lens_src, m1, m2, raw and w[0] x h[0]) as 1 launch covering max_w x max_h
int undistort_map_host(int model, int width, int height, const double *p, const double *c, int16_t *m1, uint16_t *m2);
const SlotLens *slot_lens(const KltBatchState &B, int slot);
void undistort_frames(Handle *h, const KltBatchFrame *frames, int n_frames, int max_w, int max_h);
// detect.cu: pvio_b200_batch_detect_keypoints
int batch_detect_impl(Handle *h, int n, const pvio_b200_detect_request *reqs, double clahe_clip, int tiles_x, int tiles_y);
// ba_marg.cu
int marginalize_impl(Handle *h, const pvio_b200_window *w, const pvio_b200_state *s, int index,
                     double *S_out, double *e_out, double *H_out, double *b_out);
int batch_marginalize_impl(Handle *h, int n, double *S_out, int64_t S_stride, double *e_out, int64_t e_stride);
int selftest_eig_impl(Handle *h, int n, const int32_t *dk, const double *A, const double *b, double *S_out, double *e_out);
int marg_opt_in(Handle *h);        // the eigen-solver's dynamic shared memory, for the current device (pvio_b200_create)
// klt.cu: pvio_b200_batch_track_keypoints
int batch_track_impl(Handle *h, int n, const pvio_b200_klt_pair *pairs, int max_level, int max_iter, double eps,
                     double clahe_clip, int tiles_x, int tiles_y, int border, double ransac_threshold,
                     double ransac_confidence);
// klt.cu: the stages of a batched tracker call, shared by pvio_b200_batch_track_keypoints and
// pvio_b200_batch_feature_track.  One pair of such a call:
struct KltBatchItem {
    int slot, width, height, stride, n_points;
    uint64_t prev_id, next_id;                // prev_id 0: no previous frame and no points; the next frame is only cached
    const uint8_t *prev, *next;
    const float *prev_pts, *next_pts;         // host [n_points][2]; unused when the points are written on the device
};
struct KltBatchOptions {
    int max_level, max_iter;
    double eps, clahe_clip;
    int tiles_x, tiles_y, border;
    double ransac_threshold, ransac_confidence;
};
// points written on the device: called once the staging is uploaded, with the call's device arrays of LK inputs and
// initial guesses ([n][2], pair i's points from KltBatchResults::first[i]) and the pair of each point
struct KltDevicePoints {
    std::function<int(Handle *, float *prev_pts, float *next_pts, const int *pair_of)> write_points;
};
// what the stages leave: LK + border results (host copies, or device arrays when the points were written on the
// device), and per pair its F-RANSAC outcome: mask = the winner's mask words on the device (fm_batch_masks has been
// launched; bit k: the k-th point with a nonzero status), clear = RANSAC ran and kept nothing, info as
// pvio_b200_klt_pair::info
struct KltBatchResults {
    const float *next = nullptr, *err = nullptr;
    const uint8_t *status = nullptr;
    std::vector<size_t> first;
    std::vector<const unsigned *> mask;
    std::vector<uint8_t> clear;
    std::vector<int32_t> info;
    unsigned *mw = nullptr;                   // the mask words (`words` of them) in KltBatchState::stage: host side,
    const unsigned *d_mw = nullptr;           //   device side
    size_t words = 0;
};
// Checks every pair, then uploads, builds the pyramids, runs LK, the schedules and the hypotheses, synchronises once,
// replays each pair on the host and launches the winners' masks.  dev == nullptr: the points come from the items.
int klt_batch_track(Handle *h, int n, const KltBatchItem *pairs, const KltBatchOptions &opt, const KltDevicePoints *dev,
                    KltBatchResults &res);
// feature_track.cu: pvio_b200_batch_feature_track, and its stages, which pvio_b200_batch_window_track_camera shares:
// ft_check checks every request (outputs: keypoints, prev_index and n_keypoints must be given); ft_run stages,
// launches and synchronises without changing any slot's keypoints; ft_finish writes the outputs and makes each slot's
// newest frame the new one.
int batch_feature_track_impl(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
                             double keypoint_distance);
// the device inputs of delta_key_q (frame.cpp:98), composed before the initial guesses: sequence i's step-1 IMU record
// (delta q at +1) and the constants of its window slot
struct FtPredict {
    const double *rec;                        // [n][kImuStride]
    const WinConst *cst;                      // the handle's window constants
    const int32_t *slot;                      // sequence i's window slot at slot[i * slot_stride]
    int slot_stride;
    double *q_out;                            // [n][4] the delta_key_q written
};
struct FtRun {
    std::vector<int> n_prev, out_cap;         // ft_check: keypoints of the previous frame, the output bound
    std::vector<int> count, prev_no;          // ft_run: the new frame's keypoints, the previous frame's number
    std::vector<size_t> out_off;
    const uint8_t *head = nullptr, *out = nullptr;   // the downloaded counts and outputs
    bool staged = false;                      // the new frames go to each slot's buf[2] (SlotKeypoints), not buf[1 - cur]
    KltBatchResults r;
};
int ft_check(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
             double keypoint_distance, bool outputs, FtRun &run);
int ft_run(Handle *h, int n, const pvio_b200_feature_frame *frames, const KltBatchOptions &opt,
           double keypoint_distance, const FtPredict *pred, FtRun &run);
int ft_finish(Handle *h, int n, const pvio_b200_feature_frame *frames, const FtRun &run);
// fmat.cu
int fm_ransac_impl(Handle *h, int n, const float *p, const float *q, double threshold, double confidence, int max_iters,
                   const int32_t *schedule, int n_schedule, uint8_t *mask, double *F_out, int32_t *info);
int fm_cv_schedule(int n, const float *p, const float *q, int iters, int32_t *schedule);
// fmat.cu, the F-matrix rejection of a batched tracker call: one problem per frame pair, every pointer on the device
struct FmBatchProblem {
    const float *prev_pts, *next_pts;         // [n_pts][2] the pair's LK input and output
    const uint8_t *status;                    // [n_pts] LK + border status
    float2 *p, *q;                            // [n_pts] room for the survivors, compacted in order
    int *sched, *counts;                      // [budget][7], [budget][4] (as fm_hypotheses_kernel writes them)
    double *F;                                // [budget][3][9]
    unsigned *masks;                          // [budget][3][words of n_pts]
    int *surv;                                // [2] written on the device: survivors, iterations that have a subset
    int n_pts, budget;                        // tracked points; iterations reserved (0: fewer than 8 points)
};
struct FmMaskJob {                            // the mask of one pair's winning model (n == 0: none)
    const float2 *p, *q;
    const double *F;                          // LMedS: the model, tested against thr2
    const unsigned *src;                      // RANSAC: the mask as fm_hypotheses_kernel stored it
    unsigned *out;
    float thr2;
    int n;
};
void fm_options(double &threshold, double &confidence, int &max_iters);
int fm_lmeds_iters(double confidence, int max_iters);
float fm_replay(const int *counts, int n, int have, int max_iters, double confidence, int *info);
void fm_batch_schedule(Handle *h, const FmBatchProblem *probs, int n, int max_iters, int lmeds_iters);
void fm_batch_hypotheses(Handle *h, const FmBatchProblem *probs, int n, int max_budget, float thr2);
void fm_batch_masks(Handle *h, const FmMaskJob *jobs, int n, int max_words);
// twoview.cu: pvio_b200_batch_two_view
int batch_two_view_impl(Handle *h, int n, const pvio_b200_two_view *recs);
// selftest.cu
int selftest_lie_impl(Handle *h, int n, const double *w_in, double *out);
int selftest_chol_opt_in(Handle *h);
int selftest_chol_impl(Handle *h, int n, int mode, const int32_t *Ds, const double *A, const double *b, double *x_out,
                       int32_t *ok_out);

}  // namespace pvio
