// Plane detection of many sequences on their resident slots (pvio_b200_batch_window_plane_ransac):
// PlaneExtractor::work (plane_extractor.cpp:40-81) and Plane::update_parameter(true) (plane.cpp:64-114), each a
// Ransac<3, PlaneState, PlaneSolver, PlaneEvaluator> (utility/ransac.h) over points built from the slot's own track
// table, followed by the inliers' centroid, covariance and normal.  All fp64.
//
// The RANSAC is the one pvio_b200_batch_two_view runs (ransac.cuh, DESIGN 4.7c): every iteration is evaluated
// speculatively, and the serial acceptance rule is replayed on the host over the counts.
//   device  pr_gather_kernel: one CTA per record: per candidate track (the caller's order) enough_baseline over the
//           body positions of its observing frames, its point -- get_landmark_point() for an extraction,
//           try_triangulate over its window views for a refit -- and the used points compacted in candidate order;
//           thread 0 then draws the record's sample schedule (a LotBox of the used points, seed 0, 3 draws)
//   device  pr_hypothesis_kernel: one warp per (record, iteration): PlaneSolver on the 3 drawn points, the lanes count
//           the points within the threshold with ballot and popc
//   host    the replay of Ransac::solve's loop over the counts (ransac_replay)
//   device  pr_finish_kernel: one CTA per record: the winner's mask, the inliers' centroid and covariance summed
//           serially in point order, the covariance's eigenvector of smallest eigenvalue (Jacobi), the results
//
// Two deviations from the reference (DESIGN 4.7g): the refined normal's sign is fixed (d >= 0, the component of largest
// magnitude positive at d == 0) where Eigen's QR iterations decide it; a refit track whose triangulation fails is left
// out, where plane.cpp:69-72 pushes an uninitialised point.
//
// Compiled with -fmad=false: the host arithmetic of the reference is not contracted, so the counts equal the oracle's.
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"
#include "batch_window.cuh"
#include "ransac.cuh"
#include "tri.cuh"

namespace pvio {
namespace {

constexpr int kIters = 1000;                  // Ransac's max_iteration
constexpr double kConfidence = 0.999;
constexpr int kMinInliers = 31;               // accepted on more than 30 inliers
constexpr int kMaxRecords = 65535;            // records are the grid's y dimension in the hypothesis kernel

// one record as the kernels read it: its candidates' rows at off, its iteration rows at blockIdx * kIters; best_it and
// inliers are the replay's, set before the finish
struct PrRec { int32_t slot, mode, n, off, N, best_it, inliers, pad; };
static_assert(sizeof(PrRec) % sizeof(double) == 0, "records are staged as whole 8-byte words");

struct PrArgs {
    const PrRec *rec;        // [n]
    const int32_t *row;      // [C] track-table row of each candidate
    int *n_used;             // [n] points that enter the RANSAC
    int *sched, *cnt;        // [n][kIters][3], [n][kIters]
    double *pts;             // [C][3] the used points, compacted in candidate order at each record's off
    int *lots;               // [C]
    int *cidx;               // [C] compacted index of each candidate, -1: not used
    uint8_t *cmask;          // [C] the winner's mask over the compacted points
    uint8_t *used, *inl;     // [C] results per candidate
    double *cpt;             // [C][3] the point of each candidate, NaN where it is left out
    double *plane;           // [n][8] normal, distance, reference point
};

__device__ __forceinline__ double pr_threshold(int mode) { return mode == PVIO_B200_PLANE_EXTRACT ? 0.03 : 0.05; }
__device__ __forceinline__ int pr_min_points(int mode) { return mode == PVIO_B200_PLANE_EXTRACT ? 3 : 50; }
__device__ __forceinline__ double pr_dot(const double *a, const double *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }

// PlaneSolver: n = (p2 - p0) x (p1 - p0), Eigen's stableNormalize (w = max |n_i|, z = |n / w|^2, n / (sqrt(z) w) when
// z > 0, so a zero cross product stays zero and every point is then an inlier), d = p0 . n
__device__ __forceinline__ void plane_solve(const double *p0, const double *p1, const double *p2, double *n, double &d) {
    const double a[3] = {p2[0] - p0[0], p2[1] - p0[1], p2[2] - p0[2]}, b[3] = {p1[0] - p0[0], p1[1] - p0[1], p1[2] - p0[2]};
    n[0] = a[1] * b[2] - a[2] * b[1]; n[1] = a[2] * b[0] - a[0] * b[2]; n[2] = a[0] * b[1] - a[1] * b[0];
    const double w = fmax(fmax(fabs(n[0]), fabs(n[1])), fabs(n[2]));
    const double u[3] = {n[0] / w, n[1] / w, n[2] / w};
    const double z = pr_dot(u, u);
    if (z > 0) {
        const double s = sqrt(z) * w;
        for (int k = 0; k < 3; ++k) n[k] /= s;
    }
    d = pr_dot(p0, n);
}

// PlaneEvaluator within the threshold
__device__ __forceinline__ bool plane_inlier(const double *p, const double *n, double d, double thr) {
    return fabs(pr_dot(p, n) - d) <= thr;
}

struct RowViews {                             // the window views of one track: its observing frames' camera matrices and keypoints
    const double (*Pm)[12];
    const int8_t *f;
    const double2 *zs;
    __device__ const double *P(int o) const { return Pm[f[o]]; }
    __device__ const double *z(int o) const { return reinterpret_cast<const double *>(zs + f[o]); }
};

__global__ void __launch_bounds__(kBwThreads) pr_gather_kernel(BwArgs a, PrArgs A) {
    __shared__ double sP[kMaxFrames][12];
    __shared__ int sh[kBwWarps + 1];
    const PrRec r = A.rec[blockIdx.x];
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    if (r.mode == PVIO_B200_PLANE_REFIT && threadIdx.x < r.N) {    // [R | T], R = q_cam^*, T = -R p_cam (track.cpp:61-81)
        double qc[4], pc[3];
        bw_cam_pose(fr + threadIdx.x * kFrameStride, c, qc, pc);
        loc_camera_matrix(qc, pc, sP[threadIdx.x]);
    }
    __syncthreads();
    int carry = 0;
    for (int c0 = 0; c0 < r.n; c0 += kBwThreads) {
        const int i = c0 + threadIdx.x;
        bool ok = false;
        double x[3] = {NAN, NAN, NAN};
        if (i < r.n) {
            const size_t R = base + A.row[r.off + i];
            const uint32_t m = a.tmask[R];
            double bl = 0.0;                  // Track::compute_baseline over the observing frames' body positions
            int8_t f[kMaxFrames];
            int nv = 0;
            for (uint32_t b = m; b; b &= b - 1) {
                const int g = __ffs(b) - 1;
                if (nv > 0) {
                    const double *p = fr + f[nv - 1] * kFrameStride + 4, *q = fr + g * kFrameStride + 4;
                    const double d[3] = {p[0] - q[0], p[1] - q[1], p[2] - q[2]};
                    bl += sqrt(pr_dot(d, d));
                }
                f[nv++] = (int8_t)g;
            }
            const double rho = a.trho[R];     // PlaneExtractor::enough_baseline
            ok = bl > 0.5 || (rho < 1 / 0.2 && bl * rho > 0.5);
            if (ok && r.mode == PVIO_B200_PLANE_EXTRACT) {
                bw_landmark_point(a, R, fr, c, x);
            } else if (ok) {
                double score;
                ok = nv >= 2 && tri_point_scored(RowViews{sP, f, a.tz + R * a.Ncap}, 0, nv, x, score);
                if (!ok) x[0] = x[1] = x[2] = NAN;
            }
        }
        int tot;
        const int pos = carry + bw_block_scan(ok ? 1 : 0, sh, tot);
        if (i < r.n) {
            const size_t k = (size_t)r.off + i;
            A.used[k] = ok;
            A.cidx[k] = ok ? pos : -1;
            for (int j = 0; j < 3; ++j) A.cpt[3 * k + j] = x[j];
            if (ok)
                for (int j = 0; j < 3; ++j) A.pts[3 * ((size_t)r.off + pos) + j] = x[j];
        }
        carry += tot;
    }
    if (threadIdx.x == 0) {
        A.n_used[blockIdx.x] = carry;
        if (carry >= pr_min_points(r.mode))
            lotbox_schedule(carry, 0, 3, kIters, A.lots + r.off, A.sched + (size_t)blockIdx.x * kIters * 3);
    }
}

constexpr int kPrWarps = 4;

__global__ void __launch_bounds__(32 * kPrWarps) pr_hypothesis_kernel(PrArgs A) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int it = blockIdx.x * kPrWarps + warp, k = blockIdx.y;
    const PrRec &r = A.rec[k];
    const int nu = A.n_used[k];
    if (it >= kIters || nu < pr_min_points(r.mode)) return;
    const size_t row = (size_t)k * kIters + it;
    const double *P = A.pts + 3 * (size_t)r.off;
    const int *s = A.sched + 3 * row;
    double n[3], d;
    plane_solve(P + 3 * s[0], P + 3 * s[1], P + 3 * s[2], n, d);
    const double thr = pr_threshold(r.mode);
    int good = 0;
    for (int b = 0; b < nu; b += 32) {
        const int i = b + lane;
        const bool in = i < nu && plane_inlier(P + 3 * i, n, d, thr);
        good += __popc(__ballot_sync(0xffffffffu, in));
    }
    if (lane == 0) A.cnt[row] = good;
}

__global__ void __launch_bounds__(kBwThreads) pr_finish_kernel(PrArgs A) {
    __shared__ double sM[4];
    const int k = blockIdx.x;
    const PrRec r = A.rec[k];
    const int nu = A.n_used[k];
    const double *P = A.pts + 3 * (size_t)r.off;
    const double thr = pr_threshold(r.mode);
    if (threadIdx.x == 0) {
        if (r.best_it >= 0) {
            const int *s = A.sched + 3 * ((size_t)k * kIters + r.best_it);
            plane_solve(P + 3 * s[0], P + 3 * s[1], P + 3 * s[2], sM, sM[3]);
        } else {
            sM[0] = sM[1] = sM[2] = sM[3] = NAN;
        }
    }
    __syncthreads();
    const double n[3] = {sM[0], sM[1], sM[2]}, d = sM[3];
    for (int j = threadIdx.x; j < nu; j += kBwThreads) A.cmask[r.off + j] = r.best_it >= 0 && plane_inlier(P + 3 * j, n, d, thr);
    __syncthreads();
    for (int i = threadIdx.x; i < r.n; i += kBwThreads) {
        const int j = A.cidx[r.off + i];
        A.inl[r.off + i] = j >= 0 ? A.cmask[r.off + j] : 0;
    }
    if (threadIdx.x != 0) return;
    double *out = A.plane + 8 * (size_t)k;
    for (int j = 0; j < 8; ++j) out[j] = NAN;
    if (r.inliers >= kMinInliers) {           // plane_extractor.cpp:58-77, plane.cpp:78-97
        const uint8_t *msk = A.cmask + r.off;
        double cog[3] = {0, 0, 0};
        for (int j = 0; j < nu; ++j)
            if (msk[j])
                for (int t = 0; t < 3; ++t) cog[t] += P[3 * j + t];
        for (int t = 0; t < 3; ++t) cog[t] /= (double)r.inliers;
        double G[16] = {};
        for (int j = 0; j < nu; ++j)
            if (msk[j]) {
                const double dx[3] = {P[3 * j] - cog[0], P[3 * j + 1] - cog[1], P[3 * j + 2] - cog[2]};
                for (int u = 0; u < 3; ++u)
                    for (int v = 0; v < 3; ++v) G[4 * u + v] += dx[u] * dx[v];
            }
        // the 3 x 3 covariance in a 4 x 4 whose fourth eigenvalue (above the trace) is never the smallest
        G[15] = ((G[0] + G[5]) + G[10]) + 1.0;
        double q[4];
        jacobi_eig4_smallest(G, q);
        double nn[3] = {q[0], q[1], q[2]};
        int big = 0;
        for (int t = 1; t < 3; ++t)
            if (fabs(nn[t]) > fabs(nn[big])) big = t;
        const double d0 = pr_dot(nn, cog);
        if (d0 < 0 || (d0 == 0 && nn[big] < 0))
            for (int t = 0; t < 3; ++t) nn[t] = -nn[t];
        for (int t = 0; t < 3; ++t) { out[t] = nn[t]; out[4 + t] = cog[t]; }
        out[3] = pr_dot(nn, cog);
    } else if (r.mode == PVIO_B200_PLANE_REFIT && nu >= pr_min_points(r.mode)) {   // plane.cpp:77: the raw model
        for (int t = 0; t < 4; ++t) out[t] = sM[t];
    }
}

// checks every record against its slot's host mirror and collects the candidates' rows
int pr_plan(Handle *h, int n, const pvio_b200_window_plane_ransac *recs, std::vector<PrRec> &P, std::vector<int32_t> &rows) {
    const char *what = "batch_window_plane_ransac";
    auto bad = [&](const char *why) { return fail(h, PVIO_B200_EINVAL, (std::string(what) + ": " + why).c_str()); };
    if (n < 0 || (n > 0 && !recs)) return bad("bad record list");
    if (n > kMaxRecords) return bad("more than 65535 records");
    for (int k = 0; k < n; ++k) {
        const pvio_b200_window_plane_ransac &R = recs[k];
        if (R.slot < 0 || R.slot >= h->W || !h->slots[R.slot].resident) return bad("slot out of range or not resident");
        if (R.mode != PVIO_B200_PLANE_EXTRACT && R.mode != PVIO_B200_PLANE_REFIT) return bad("unknown mode");
        if (R.n_tracks < 0 || (R.n_tracks > 0 && (!R.tracks || !R.used || !R.inlier)) || !R.info || !R.plane)
            return bad("null array");
        const WinSlot &s = h->slots[R.slot];
        if ((int64_t)rows.size() + R.n_tracks > INT32_MAX) return bad("more than 2^31 - 1 candidates in one call");
        P.push_back(PrRec{R.slot, R.mode, R.n_tracks, (int32_t)rows.size(), s.N, -1, 0, 0});
        std::vector<uint8_t> named(s.ids.size(), 0);
        for (int i = 0; i < R.n_tracks; ++i) {
            const int r = find_row(s, R.tracks[i]);
            if (r < 0) return bad("unknown or dead track");
            if (named[r]) return bad("a track named twice");
            named[r] = 1;
            rows.push_back(r);
        }
    }
    return 0;
}

int batch_window_plane_ransac_impl(Handle *h, int n, const pvio_b200_window_plane_ransac *recs) {
    std::vector<PrRec> plan;
    std::vector<int32_t> rows;
    TRY(pr_plan(h, n, recs, plan, rows));
    if (n == 0) return 0;
    cudaSetDevice(h->device);
    bool want_sched = false;
    for (int k = 0; k < n; ++k) want_sched |= recs[k].schedule != nullptr;
    const size_t C = rows.size(), I = (size_t)n * kIters;
    // upload records | rows; download (after the hypotheses) points used | counts | schedules, (after the finish)
    // used | inlier | candidate points | planes; device only the compacted points, lots, compacted indices and mask
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto sRec = S.up(plan);
    const auto sRow = S.up(rows);
    const auto sNu = S.add<int>(Stage::kDown, n);
    const auto sCnt = S.add<int>(Stage::kDown, I);
    const auto sSch = S.add<int>(Stage::kDown, 3 * I);
    const auto sUsed = S.add<uint8_t>(Stage::kDown, C);
    const auto sInl = S.add<uint8_t>(Stage::kDown, C);
    const auto sCpt = S.add<double>(Stage::kDown, 3 * C);
    const auto sPl = S.add<double>(Stage::kDown, 8 * (size_t)n);
    const auto sPts = S.add<double>(Stage::kScratch, 3 * C);
    const auto sLots = S.add<int>(Stage::kScratch, C);
    const auto sCidx = S.add<int>(Stage::kScratch, C);
    const auto sMask = S.add<uint8_t>(Stage::kScratch, C);
    TRY(S.place(h, true));
    PrArgs A;
    A.rec = S.dev(sRec); A.row = S.dev(sRow); A.n_used = S.dev(sNu); A.sched = S.dev(sSch); A.cnt = S.dev(sCnt);
    A.pts = S.dev(sPts); A.lots = S.dev(sLots); A.cidx = S.dev(sCidx); A.cmask = S.dev(sMask);
    A.used = S.dev(sUsed); A.inl = S.dev(sInl); A.cpt = S.dev(sCpt); A.plane = S.dev(sPl);
    cudaStream_t st = h->stream;
    pr_gather_kernel<<<n, kBwThreads, 0, st>>>(launch_args<BwArgs>(h), A);
    pr_hypothesis_kernel<<<dim3((kIters + kPrWarps - 1) / kPrWarps, n), 32 * kPrWarps, 0, st>>>(A);
    h->launches += 2;
    CK(h, cudaGetLastError());
    TRY(S.download(h, sNu, want_sched ? sSch : sCnt));
    CK(h, cudaStreamSynchronize(st));

    std::vector<int> res(4 * (size_t)n);
    const int *nu = S.host(sNu), *cnt = S.host(sCnt);
    for (int k = 0; k < n; ++k) {
        int *rk = &res[4 * (size_t)k];
        rk[0] = rk[1] = 0; rk[2] = rk[3] = -1;
        const int min_pts = plan[k].mode == PVIO_B200_PLANE_EXTRACT ? 3 : 50;
        if (nu[k] >= min_pts) ransac_replay(cnt + (size_t)k * kIters, 1, true, nu[k], kIters, kConfidence, rk);
        PrRec &R = S.host(sRec)[k];
        R.best_it = rk[2]; R.inliers = rk[0];
    }
    TRY(S.upload(h, sRec));
    pr_finish_kernel<<<n, kBwThreads, 0, st>>>(A);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(S.download(h, sUsed, sPl));
    CK(h, cudaStreamSynchronize(st));

    for (int k = 0; k < n; ++k) {
        const pvio_b200_window_plane_ransac &R = recs[k];
        const PrRec &p = plan[k];
        const int *rk = &res[4 * (size_t)k];
        const int min_pts = p.mode == PVIO_B200_PLANE_EXTRACT ? 3 : 50;
        const int status = nu[k] < min_pts ? PVIO_B200_PLANE_FEW_POINTS
                           : rk[0] >= kMinInliers ? PVIO_B200_PLANE_ACCEPTED : PVIO_B200_PLANE_REJECTED;
        const int32_t info[5] = {status, nu[k], rk[0], rk[1], rk[2]};
        std::memcpy(R.info, info, sizeof(info));
        std::memcpy(R.plane, S.host(sPl) + 8 * (size_t)k, sizeof(double) * 7);
        if (p.n) {
            std::memcpy(R.used, S.host(sUsed) + p.off, p.n);
            std::memcpy(R.inlier, S.host(sInl) + p.off, p.n);
            if (R.points) std::memcpy(R.points, S.host(sCpt) + 3 * (size_t)p.off, sizeof(double) * 3 * p.n);
        }
        const bool ran = nu[k] >= min_pts;
        if (R.schedule) {
            if (ran) std::memcpy(R.schedule, S.host(sSch) + 3 * (size_t)k * kIters, sizeof(int) * 3 * kIters);
            else std::fill(R.schedule, R.schedule + 3 * kIters, -1);
        }
        if (R.counts) {
            if (ran) std::memcpy(R.counts, cnt + (size_t)k * kIters, sizeof(int) * kIters);
            else std::fill(R.counts, R.counts + kIters, -1);
        }
    }
    return 0;
}

}  // namespace
}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_batch_window_plane_ransac(pvio_b200_handle hh, int n, const pvio_b200_window_plane_ransac *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_window_plane_ransac_impl(h, n, records);
}
