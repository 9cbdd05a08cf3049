// Queries on the resident slots at their current state: the joint covariance of window frames with the landmarks'
// inverse-depth variances (pvio_b200_batch_window_covariance), every landmark's world point with its covariance
// (pvio_b200_batch_window_landmarks), and the state at any time inside the window (pvio_b200_batch_window_trajectory).
#include <cmath>
#include <vector>

#include <math_constants.h>

#include "ba_cov_lm.cuh"
#include "batch_window.cuh"
#include "imu.cuh"
#include "imu_factor_cov.cuh"

namespace pvio {

// ---- pvio_b200_batch_window_landmarks: every row's world point, and for the rows the solve treats as landmarks the
// point's covariance from the covariance call's Sigma_xi and the landmark's Schur records
struct BwLmk {
    int32_t slot, n_rows, T;      // rows written; live rows of the slot
    int32_t rows_off;             // ints into the call's row list; -1: rows [0, n_rows) of the slot (every live track)
    int32_t out_off;              // rows into the call's points
    int32_t cov, cov_off, pad;    // index among the records with a covariance (-1: none); rows into its outputs
};
struct LmkArgs {
    const BwLmk *rec;             // [n]
    const int32_t *rows;          // the named rows of every record
    const int32_t *cov_rec;       // [n_cov] the record of each covariance record
    double *pts;                  // out: [rows][3]
    int32_t *role;                // out: [rows]
    int32_t *lm_of;               // scratch: [n_cov][Mcap] the packed landmark of each row of the slot, -1: none
    const int32_t *status;        // [n_cov] cov_kernel's status
    const double *sig_xi;         // [n_cov][Ncap][Ncap][36] Sigma_xi of every frame pair (cov_kernel)
    double *pcov, *var;           // out: [cov rows][9], [cov rows]
};
constexpr int kLmkWarps = 4;

// One CTA per record: Track::get_landmark_point() of every row; for a record with a covariance, the packed landmark of
// every row of its slot (bw_layout_kernel's lm_row inverted) for bw_landmark_cov_kernel
__global__ void __launch_bounds__(kBwThreads) bw_landmark_point_kernel(BwArgs a, LmkArgs L) {
    const BwLmk r = L.rec[blockIdx.x];
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const double *fr = a.frames + (size_t)w * a.Ncap * kFrameStride;
    const WinConst &c = a.cst[w];
    for (int k = threadIdx.x; k < r.n_rows; k += kBwThreads) {
        const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
        bw_landmark_point(a, base + row, fr, c, L.pts + 3 * ((size_t)r.out_off + k));
        L.role[r.out_off + k] = a.trole[base + row];
    }
    if (r.cov < 0) return;
    int32_t *lm = L.lm_of + (size_t)r.cov * a.Mcap;
    for (int q = threadIdx.x; q < r.T; q += kBwThreads) lm[q] = -1;
    __syncthreads();
    for (int lp = threadIdx.x; lp < a.hdr[w].M; lp += kBwThreads) lm[a.lm_row[base + lp]] = lp;
}

// row i of X_l = [[x]x, I]
__device__ __forceinline__ void lmk_xrow(const double *x, int i, double *o) {
    o[0] = i == 1 ? x[2] : (i == 2 ? -x[1] : 0.0);
    o[1] = i == 0 ? -x[2] : (i == 2 ? x[0] : 0.0);
    o[2] = i == 0 ? x[1] : (i == 1 ? -x[0] : 0.0);
    o[3] = i == 0 ? 1.0 : 0.0; o[4] = i == 1 ? 1.0 : 0.0; o[5] = i == 2 ? 1.0 : 0.0;
}

// One warp per row of a record with a covariance (grid: covariance records x row blocks).  Var(rho) as cov_lm_kernel
// forms it (ba_cov_lm.cuh), C = Cov(xi_a, rho) = -(Sigma_xi h_l)_a / H_ll from the same products, then
//   Sigma_x = X Sigma_aa X^T - X C c^T - c C^T X^T + c c^T Var(rho),  X = [[x - o]x, I], c = -(x - c_a) / rho,
// o the window's origin, about which frame_T takes xi,
// the upper triangle on six lanes, mirrored (exactly symmetric).  NaN for a row that is not a landmark of the solve and
// for every row of a record whose factorisation failed.
template <typename real>
__global__ void __launch_bounds__(32 * kLmkWarps) bw_landmark_cov_kernel(BwArgs a, LmkArgs L) {
    __shared__ double u_sm[kLmkWarps][6 * kMaxFrames];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const int crec = blockIdx.x;                     // the covariance record
    const BwLmk r = L.rec[L.cov_rec[crec]];
    const int k = blockIdx.y * kLmkWarps + wv;
    if (k >= r.n_rows) return;
    const int w = r.slot;
    const size_t base = (size_t)w * a.Mcap;
    const int row = r.rows_off < 0 ? k : L.rows[r.rows_off + k];
    const int lm = L.lm_of[(size_t)crec * a.Mcap + row];
    double *P = L.pcov + 9 * ((size_t)r.cov_off + k);
    double *V = L.var + r.cov_off + k;
    if (lm < 0 || L.status[crec] != PVIO_B200_OK) {
        if (lane < 9) P[lane] = CUDART_NAN;
        if (lane == 0) *V = CUDART_NAN;
        return;
    }
    const int N = a.hdr[w].N;
    const unsigned fixed = (unsigned)a.hdr[w].fixed_mask & ((1u << N) - 1u);
    const real *hs = reinterpret_cast<const real *>(a.hs) + (size_t)w * a.Ncap * a.Mcap * 6;
    double *u = u_sm[wv];
    cov_lm_h(hs, a.Mcap, lm, N, fixed, lane, u);
    __syncwarp();
    const double *X = L.sig_xi + (size_t)crec * a.Ncap * a.Ncap * 36;
    const int an = __ffs(a.tmask[base + row]) - 1;
    double srow = 0.0;
    const double q = cov_lm_quad<true>(u, X, N, lane, an, srow);
    const double hll = a.lm_aux[base + lm].hll;
    const double var = cov_lm_var(hll, q);
    double C[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) C[i] = -__shfl_sync(0xffffffffu, srow, (6 * an + i) & 31) / hll;
    const double2 z = a.tz[(base + row) * a.Ncap + an];
    const double rho = a.trho[base + row];
    double qc[4], pc[3], x[3];
    bw_cam_pose(a.frames + ((size_t)w * a.Ncap + an) * kFrameStride, a.cst[w], qc, pc);
    bw_world_point(qc, pc, z.x, z.y, rho, x);
    const double cl[3] = {-(x[0] - pc[0]) / rho, -(x[1] - pc[1]) / rho, -(x[2] - pc[2]) / rho};
    const double *o = a.cst[w].origin;                  // xi is taken about the window's origin (frame_T)
    const double xo[3] = {x[0] - o[0], x[1] - o[1], x[2] - o[2]};
    if (lane < 6) {
        const int i = lane < 3 ? 0 : (lane < 5 ? 1 : 2), j = lane < 3 ? lane : (lane < 5 ? lane - 2 : 2);
        double Xi[6], Xj[6];
        lmk_xrow(xo, i, Xi);
        lmk_xrow(xo, j, Xj);
        const double *S = X + ((size_t)an * N + an) * 36;
        double s = 0.0, bi = 0.0, bj = 0.0;
#pragma unroll
        for (int m = 0; m < 6; ++m) {
            double t = 0.0;
#pragma unroll
            for (int n = 0; n < 6; ++n) t += S[m * 6 + n] * Xj[n];
            s += Xi[m] * t;
            bi += Xi[m] * C[m];
            bj += Xj[m] * C[m];
        }
        const double cli = i == 0 ? cl[0] : (i == 1 ? cl[1] : cl[2]), clj = j == 0 ? cl[0] : (j == 1 ? cl[1] : cl[2]);
        const double v = s - bi * clj - cli * bj + cli * clj * var;
        P[3 * i + j] = v;
        P[3 * j + i] = v;
    }
    if (lane == 0) *V = var;
}

// ---- pvio_b200_batch_window_trajectory: the state at any time inside the window, forward from the preceding frame
// through the part of its IMU factor's kept samples up to that time, and its covariance
struct BwTraj {
    int32_t slot, N, n_times, cov;    // cov: index among the records with a covariance (-1: none asked; -2: asked, but
                                      // no factor holds samples)
    int64_t t_off;                    // rows into the call's times, states and frames
    int64_t cov_off;                  // doubles into the covariance scratch: the joint block of the frames that own a
                                      // factor with samples (CovRec::cov_off)
    int64_t scov_off;                 // rows into the call's state covariances
    int32_t ns[kMaxFrames];           // samples of factor k (frames k, k + 1), 0: none
};
static_assert(sizeof(BwTraj) % sizeof(double) == 0, "records are staged as whole 8-byte words");
struct TrajArgs {
    const BwTraj *rec;                // [n]
    const double *times;              // [rows]
    double *states;                   // out: [rows][16]
    int32_t *frame;                   // out: [rows]
    double *scov;                     // out: [cov rows][225]
    const double *jcov;               // cov_kernel's joint blocks (scratch)
    const int32_t *status;            // [n_cov] cov_kernel's status
    int covs;                         // 1: the per-warp covariance scratch is laid out
};
// per warp of bw_trajectory_kernel: the chain, the emitted copy, then (with covariances) four 15 x 15 matrices
__host__ __device__ constexpr size_t traj_warp_bytes(bool covs) { return 2 * sizeof(ImuWarpSm) + (covs ? 4 * 225 * 8 : 0); }

// the first of the n sorted times t[i] that is >= x (upper: > x)
__device__ __forceinline__ int traj_bound(const double *t, int n, double x, bool upper) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int m = (lo + hi) >> 1;
        if (upper ? t[m] <= x : t[m] < x) lo = m + 1;
        else hi = m;
    }
    return lo;
}

// queries [q0, q1) of record r, which no factor takes: frame -1, a zero state, a NaN covariance.  One warp.
__device__ __forceinline__ void none_rows(const TrajArgs &T, const BwTraj &r, int lane, int q0, int q1, bool cov) {
    for (int q = q0; q < q1; ++q) {
        const size_t row = r.t_off + q;
        if (lane < 16) T.states[16 * row + lane] = 0.0;
        if (lane == 0) T.frame[row] = -1;
        if (cov)
            for (int e = lane; e < 225; e += 32) T.scov[225 * ((size_t)r.scov_off + q) + e] = CUDART_NAN;
    }
}

// One CTA per record, one warp per factor k with samples (warp k).  The warp's queries are the times t >= s_0.t of its
// factor and below s_0.t of the next factor with samples (so k is the largest such factor whose s_0.t <= t), found by
// binary search; it takes those at most its t_end, or all of them when factor k + 1 holds samples.  It walks its
// samples once, as imu_integrate_warp does (imu_step_warp), and emits each query as the walk passes it: the increment
// of the last sample at or before t, over t - s_j.t, goes onto a copy of the chain, which is what imu_integrate_warp
// gives for the samples at or before t with t_end = t.  Then PreIntegrator::predict from frame k's state, and with a
// covariance Phi Sigma_k Phi^T + Psi Sigma_delta Psi^T (imu_factor_propagate), Sigma_delta the partial increment's
// covariance itself.  Times no warp takes (before the first sample, past a factor's t_end, over a factor without
// samples) get frame -1, a zero state and a NaN covariance: warp 0 writes those before the earliest s_0.t, each warp
// those past its t_end.
__global__ void __launch_bounds__(32 * (kMaxFrames - 1)) bw_trajectory_kernel(BwArgs a, TrajArgs T) {
    extern __shared__ __align__(16) unsigned char traj_sm[];
    const int lane = threadIdx.x & 31, wv = threadIdx.x >> 5;
    const BwTraj &r = T.rec[blockIdx.x];
    const int nf = r.N - 1, nq = r.n_times;
    const double *tq = T.times + r.t_off;
    const size_t F0 = (size_t)r.slot * a.Ncap;
    auto s0 = [&](int k) { return a.imu_s[(F0 + k) * a.Scap * 7]; };
    const bool cov = r.cov != -1;                           // -2: covariances asked, no factor holds samples
    const bool cov_ok = r.cov >= 0 && T.status[r.cov] == PVIO_B200_OK;
    if (wv == 0) {
        double lo = CUDART_INF;
        for (int j = 0; j < nf; ++j)
            if (r.ns[j] > 0) lo = fmin(lo, s0(j));
        none_rows(T, r, lane, 0, traj_bound(tq, nq, lo, false), cov);
    }
    const int k = wv;
    if (k >= nf || r.ns[k] == 0) return;
    const size_t F = F0 + k;
    const double lo = s0(k);
    double hi = CUDART_INF;
    for (int j = k + 1; j < nf; ++j)
        if (r.ns[j] > 0) hi = fmin(hi, s0(j));
    const double *aux = a.imu_aux + F * kImuAux, t_end = aux[0];
    const int q0 = traj_bound(tq, nq, lo, false), q1 = max(q0, traj_bound(tq, nq, hi, false));
    const int q2 = (k + 1 < nf && r.ns[k + 1] > 0) ? q1 : min(q1, max(q0, traj_bound(tq, nq, t_end, true)));
    none_rows(T, r, lane, q2, q1, cov);
    if (q0 >= q2) return;
    unsigned char *base = traj_sm + (size_t)wv * traj_warp_bytes(T.covs);
    ImuWarpSm &S = *reinterpret_cast<ImuWarpSm *>(base), &E = *reinterpret_cast<ImuWarpSm *>(base + sizeof(ImuWarpSm));
    double *A = reinterpret_cast<double *>(base + 2 * sizeof(ImuWarpSm)), *B = A + 225, *C = B + 225, *D = C + 225;
    const double *x = a.frames + F * kFrameStride;
    const double bg[3] = {x[10], x[11], x[12]}, ba[3] = {x[13], x[14], x[15]};
    const double *smp = a.imu_s + F * a.Scap * 7, *noise = aux + 1;
    const int m = r.ns[k];
    // Sigma_k: frame k's diagonal block of the joint covariance of the frames that own a factor with samples
    unsigned has = 0;
    for (int j = 0; j < nf; ++j) has |= (r.ns[j] > 0 ? 1u : 0u) << j;
    const int K15 = 15 * __popc(has), p15 = 15 * __popc(has & ((1u << k) - 1u));
    const double *Sk = T.jcov + r.cov_off + (size_t)p15 * K15 + p15;
    imu_reset_warp(S, lane);
    int q = q0;
    for (int j = 0; j < m && q < q2; ++j) {
        const double *d = smp + (size_t)j * 7;
        const bool last = j + 1 == m;
        const double t_next = last ? t_end : smp[(size_t)(j + 1) * 7];
        for (; q < q2 && (last || tq[q] < t_next); ++q) {   // the queries whose last sample is s_j
            imu_copy_warp(S, E, lane);
            imu_step_warp(E, lane, d, tq[q] - d[0], bg, ba, noise);
            const size_t row = r.t_off + q;
            if (lane == 0) {
                bw_imu_predict(x, E.tsum, E.q, E.p, E.v, T.states + 16 * row);
                T.frame[row] = k;
            }
            if (!cov) continue;
            double *out = T.scov + 225 * (size_t)(r.scov_off + q);
            if (!cov_ok) {
                for (int e = lane; e < 225; e += 32) out[e] = CUDART_NAN;
                continue;
            }
            for (int e = lane; e < 225; e += 32) {
                const int i = e / 15, c = e % 15;
                A[e] = 0.5 * (Sk[(size_t)i * K15 + c] + Sk[(size_t)c * K15 + i]);
                D[e] = (i < 9 && c < 9) ? E.C[i * 9 + c]
                     : (i >= 9 && i < 12 && c >= 9 && c < 12) ? E.cbg[(i - 9) * 3 + c - 9]
                     : (i >= 12 && c >= 12) ? E.cba[(i - 12) * 3 + c - 12] : 0.0;
            }
            __syncwarp();
            double Rs[9], dR[9];
            quat_to_mat(x, Rs);
            quat_to_mat(E.q, dR);
            const ImuFactorJac f{E.tsum, E.p, E.v, E.dq_dbg, E.dp_dbg, E.dp_dba, E.dv_dbg, E.dv_dba};
            imu_factor_propagate(A, B, C, D, f, Rs, dR, lane);
            for (int e = lane; e < 225; e += 32) {
                const int i = e / 15, c = e % 15;
                out[e] = 0.5 * ((A[e] + D[e]) + (A[c * 15 + i] + D[c * 15 + i]));
            }
            __syncwarp();
        }
        if (!last && q < q2) imu_step_warp(S, lane, d, t_next - d[0], bg, ba, noise);
    }
}

// the landmark index of every row of a slot in its packed window (rows of role < 0 with >= 2 observations, stably by
// anchor, as bw_layout_kernel orders them), -1 for the other rows
static std::vector<int32_t> landmark_of_rows(const WinSlot &s) {
    const int T = (int)s.ids.size();
    std::vector<int32_t> lm(T, -1);
    int k = 0;
    for (int a = 0; a < kMaxFrames; ++a)
        for (int r = 0; r < T; ++r)
            if (s.role[r] < 0 && __builtin_popcount(s.mask[r]) >= 2 && __builtin_ctz(s.mask[r]) == a) lm[r] = k++;
    return lm;
}

// The covariance systems a call solves: one CovRec per slot whose Sigma_xi it needs, the frames of each record's joint
// block, the Sigma_delta scratch.  stage declares their sections (the joint blocks of kind `blocks`), run launches the
// systems (with_lms: and the covariance call's landmark variances).
struct CovPlan {
    std::vector<CovRec> recs;
    std::vector<int32_t> slots, frames;
    int64_t cov_n = 0, sig_n = 0;
    Stage::Sec<CovRec> rec;
    Stage::Sec<int32_t> fr, sl, st;
    Stage::Sec<double> cov, sig, sxi;

    // a record of slot `slot` with the joint block of frames f[0 .. nf): its index, -1 when the slot's reduced system is
    // too large for cov_kernel's shared memory
    int add(const Handle *h, int slot, int nf = 0, const int32_t *f = nullptr) {
        if (cov_smem_bytes(h->hdr.h[slot]) > 220 * 1024) return -1;
        const WinSlot &s = h->slots[slot];
        const int64_t D = (s.inertial ? 15 : 6) * (int64_t)s.N;
        recs.push_back(CovRec{slot, nf, (int32_t)frames.size(), 0, cov_n, sig_n});
        slots.push_back(slot);
        frames.insert(frames.end(), f, f + nf);
        cov_n += 225 * (int64_t)nf * nf;
        sig_n += D * D;
        return (int)recs.size() - 1;
    }
    void stage(Stage &S, const Handle *h, Stage::Kind blocks) {
        const size_t n = recs.size();
        rec = S.up(recs); fr = S.up(frames); sl = S.up(slots);
        cov = S.add<double>(blocks, (size_t)cov_n); st = S.add<int32_t>(Stage::kDown, n);
        sig = S.add<double>(Stage::kScratch, (size_t)sig_n); sxi = S.add<double>(Stage::kScratch, n * h->Ncap * h->Ncap * 36);
    }
    int run(Handle *h, const Stage &S, bool with_lms = false, const CovLm *lms = nullptr, int n_lm = 0, double *var = nullptr) const {
        const int n = (int)recs.size();
        const CovLaunch L{S.dev(rec), S.dev(fr), lms, n_lm, S.dev(cov), var, S.dev(st), S.dev(sig), S.dev(sxi)};
        if (n == 0) return 0;
        return with_lms ? run_covariance(h, n, slots.data(), S.dev(sl), L) : run_cov_system(h, n, slots.data(), S.dev(sl), L);
    }
};

}  // namespace pvio

using namespace pvio;

extern "C" {

int pvio_b200_batch_window_covariance(pvio_b200_handle hh, int n, pvio_b200_window_covariance *records) {
    BwCall C(hh, "batch_window_covariance");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked against its slot's host mirror before anything is staged
    CovPlan P;
    std::vector<CovLm> lms;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_covariance &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (s.N < 1) return C.bad("a window without frames");
        if (R.n_frames < 0 || R.n_frames > s.N || R.n_tracks < 0 || R.n_tracks > (int)s.ids.size())
            return C.bad("a frame or track count out of range");
        if (R.n_frames == 0 && R.n_tracks == 0) return C.bad("a record asking for nothing");
        if (R.n_frames > 0 && (!R.frames || !R.cov)) return C.bad("frames or cov missing");
        if (R.n_tracks > 0 && (!R.tracks || !R.inv_depth_var)) return C.bad("tracks or inv_depth_var missing");
        uint32_t seen = 0;
        for (int k = 0; k < R.n_frames; ++k) {
            const int f = R.frames[k];
            if (f < 0 || f >= s.N) return C.bad("a frame out of range");
            if ((seen >> f) & 1u) return C.bad("a frame named twice");
            seen |= 1u << f;
        }
        if (P.add(h, R.slot, R.n_frames, R.frames) < 0) return C.bad("reduced system too large for shared memory");
        const std::vector<int32_t> lm = R.n_tracks > 0 ? landmark_of_rows(s) : std::vector<int32_t>();
        std::vector<uint8_t> taken(s.ids.size(), 0);
        for (int k = 0; k < R.n_tracks; ++k) {
            const int r = find_row(s, R.tracks[k]);
            if (r < 0) return C.bad("a track that is not live in its slot");
            if (taken[r]) return C.bad("a track named twice");
            taken[r] = 1;
            lms.push_back(CovLm{i, R.slot, lm[r], 0});
        }
    }
    const int n_lm = (int)lms.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    P.stage(S, h, Stage::kDown);
    const auto lmv = S.up(lms);
    const auto var = S.add<double>(Stage::kDown, (size_t)n_lm);
    TRY(S.place(h, true));
    TRY(P.run(h, S, true, S.dev(lmv), n_lm, S.dev(var)));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0, t = 0; i < n; ++i) {
        pvio_b200_window_covariance &R = records[i];
        if (R.n_frames > 0) memcpy(R.cov, S.host(P.cov) + P.recs[i].cov_off, sizeof(double) * 225 * R.n_frames * R.n_frames);
        if (R.n_tracks > 0) memcpy(R.inv_depth_var, S.host(var) + t, sizeof(double) * R.n_tracks);
        t += R.n_tracks;
        R.status = S.host(P.st)[i];
    }
    return 0;
}

int pvio_b200_batch_window_landmarks(pvio_b200_handle hh, int n, pvio_b200_window_landmarks *records) {
    BwCall C(hh, "batch_window_landmarks");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked against its slot's host mirror before anything is staged; the all-tracks mode takes its rows
    // from the mirror's size, with no per-track work
    std::vector<BwLmk> recs(n);
    std::vector<int32_t> rows, cov_rec;
    CovPlan P;
    int32_t n_pts = 0, n_cov_rows = 0, max_cov_rows = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_landmarks &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        const int T = (int)s.ids.size();
        if (s.N < 1) return C.bad("a window without frames");
        if (R.n_tracks < -1 || R.n_tracks > T) return C.bad("a track count out of range");
        const bool all = R.n_tracks == -1;
        const int nr = all ? T : R.n_tracks;
        if (all && R.capacity < T) return C.bad("capacity smaller than the slot's live tracks");
        if (!all && nr > 0 && !R.tracks) return C.bad("tracks missing");
        if (nr > 0 && !R.point) return C.bad("point missing");
        if (R.inv_depth_var && !R.point_cov) return C.bad("inv_depth_var without point_cov");
        const bool cov = R.point_cov != nullptr;
        const int c = cov ? P.add(h, R.slot) : -1;
        if (cov && c < 0) return C.bad("reduced system too large for shared memory");
        BwLmk &L = recs[i];
        L = BwLmk{R.slot, nr, T, all ? -1 : (int32_t)rows.size(), n_pts, c, n_cov_rows, 0};
        if (!all) {
            std::vector<uint8_t> taken(T, 0);
            for (int k = 0; k < nr; ++k) {
                const int r = find_row(s, R.tracks[k]);
                if (r < 0) return C.bad("a track that is not live in its slot");
                if (taken[r]) return C.bad("a track named twice");
                taken[r] = 1;
                rows.push_back(r);
            }
        }
        n_pts += nr;
        if (cov) {
            cov_rec.push_back(i);
            n_cov_rows += nr;
            max_cov_rows = std::max(max_cov_rows, nr);
        }
    }
    const int n_cov = (int)cov_rec.size();
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto rw = S.up(rows);
    const auto crc = S.up(cov_rec);
    P.stage(S, h, Stage::kScratch);
    const auto pts = S.add<double>(Stage::kDown, 3 * (size_t)n_pts);
    const auto rol = S.add<int32_t>(Stage::kDown, (size_t)n_pts);
    const auto pcov = S.add<double>(Stage::kDown, 9 * (size_t)n_cov_rows), var = S.add<double>(Stage::kDown, (size_t)n_cov_rows);
    const auto lmo = S.add<int32_t>(Stage::kScratch, (size_t)n_cov * h->Mcap);
    TRY(S.place(h, true));
    const LmkArgs L{S.dev(rec), S.dev(rw), S.dev(crc), S.dev(pts), S.dev(rol), S.dev(lmo), S.dev(P.st), S.dev(P.sxi), S.dev(pcov), S.dev(var)};
    const BwArgs a = launch_args<BwArgs>(h);
    bw_landmark_point_kernel<<<n, kBwThreads, 0, h->stream>>>(a, L);
    TRY(launched(h, "bw_landmark_point_kernel"));
    if (n_cov > 0) {
        TRY(P.run(h, S));
        const dim3 grid(n_cov, std::max(1, (max_cov_rows + kLmkWarps - 1) / kLmkWarps));
        if (h->hs_double) bw_landmark_cov_kernel<double><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        else bw_landmark_cov_kernel<float><<<grid, 32 * kLmkWarps, 0, h->stream>>>(a, L);
        TRY(launched(h, "bw_landmark_cov_kernel"));
    }
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_landmarks &R = records[i];
        const BwLmk &L = recs[i];
        const WinSlot &s = h->slots[R.slot];
        const size_t nr = L.n_rows;
        if (nr > 0) memcpy(R.point, S.host(pts) + 3 * (size_t)L.out_off, sizeof(double) * 3 * nr);
        if (R.role && nr > 0) memcpy(R.role, S.host(rol) + L.out_off, sizeof(int32_t) * nr);
        if (R.track_id && nr > 0) {
            if (L.rows_off < 0) memcpy(R.track_id, s.ids.data(), sizeof(int32_t) * nr);
            else memcpy(R.track_id, records[i].tracks, sizeof(int32_t) * nr);
        }
        R.status = PVIO_B200_OK;
        if (L.cov >= 0) {
            if (nr > 0) memcpy(R.point_cov, S.host(pcov) + 9 * (size_t)L.cov_off, sizeof(double) * 9 * nr);
            if (R.inv_depth_var && nr > 0) memcpy(R.inv_depth_var, S.host(var) + L.cov_off, sizeof(double) * nr);
            R.status = S.host(P.st)[L.cov];
        }
        R.n_rows = (int32_t)nr;
    }
    return 0;
}

int pvio_b200_batch_window_trajectory(pvio_b200_handle hh, int n, pvio_b200_window_trajectory *records) {
    BwCall C(hh, "batch_window_trajectory");
    if (!C.open(n, records)) return C.rc;
    Handle *h = C.h;
    // every record checked before anything is staged
    std::vector<BwTraj> recs(n);
    std::vector<double> times;
    CovPlan P;
    int64_t rows = 0, cov_rows = 0;
    int warps = 1;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_window_trajectory &R = records[i];
        const WinSlot &s = h->slots[R.slot];
        if (!s.inertial) return C.bad("a visual-only slot");
        if (R.n_times < 0) return C.bad("a negative time count");
        if (R.n_times > 0 && (!R.times || !R.states || !R.frame)) return C.bad("times, states or frame missing");
        for (int q = 0; q < R.n_times; ++q) {
            if (!std::isfinite(R.times[q])) return C.bad("a time that is not finite");
            if (q > 0 && R.times[q] < R.times[q - 1]) return C.bad("times that decrease");
        }
        BwTraj &T = recs[i];
        T = BwTraj{};
        T.slot = R.slot; T.N = s.N; T.n_times = R.n_times; T.cov = -1; T.t_off = rows; T.scov_off = cov_rows;
        std::vector<int32_t> owners;
        for (int k = 0; k + 1 < s.N; ++k) {
            T.ns[k] = s.n_samples.empty() ? 0 : s.n_samples[k];
            if (T.ns[k] > 0) owners.push_back(k);
        }
        warps = std::max(warps, s.N - 1);
        if (R.state_cov && !owners.empty()) {        // Sigma_k of the frames that own a factor with samples
            T.cov_off = P.cov_n;
            T.cov = P.add(h, R.slot, (int)owners.size(), owners.data());
            if (T.cov < 0) return C.bad("reduced system too large for shared memory");
        }
        if (R.state_cov) {
            if (T.cov < 0) T.cov = -2;               // NaN rows only: no factor holds samples
            cov_rows += R.n_times;
        }
        times.insert(times.end(), R.times, R.times + R.n_times);
        rows += R.n_times;
    }
    const bool any_cov = cov_rows > 0;
    Stage S(h->bw.stage, &h->bw.scratch);
    const auto rec = S.up(recs);
    const auto tm = S.up(times);
    P.stage(S, h, Stage::kScratch);
    const auto sto = S.add<double>(Stage::kDown, 16 * (size_t)rows);
    const auto fro = S.add<int32_t>(Stage::kDown, (size_t)rows);
    const auto sco = S.add<double>(Stage::kDown, 225 * (size_t)cov_rows);
    TRY(S.place(h, true));
    TRY(P.run(h, S));
    const TrajArgs T{S.dev(rec), S.dev(tm), S.dev(sto), S.dev(fro), S.dev(sco), S.dev(P.cov), S.dev(P.st), any_cov ? 1 : 0};
    const size_t smem = warps * traj_warp_bytes(any_cov);
    if (smem > 48 * 1024)
        CK(h, cudaFuncSetAttribute(bw_trajectory_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    bw_trajectory_kernel<<<n, 32 * warps, smem, h->stream>>>(launch_args<BwArgs>(h), T);
    TRY(launched(h, "bw_trajectory_kernel"));
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(h->stream));
    for (int i = 0; i < n; ++i) {
        pvio_b200_window_trajectory &R = records[i];
        const BwTraj &T = recs[i];
        const size_t nq = R.n_times;
        if (nq > 0) {
            memcpy(R.states, S.host(sto) + 16 * (size_t)T.t_off, sizeof(double) * 16 * nq);
            memcpy(R.frame, S.host(fro) + T.t_off, sizeof(int32_t) * nq);
            if (R.state_cov) memcpy(R.state_cov, S.host(sco) + 225 * (size_t)T.scov_off, sizeof(double) * 225 * nq);
        }
        R.status = T.cov >= 0 ? S.host(P.st)[T.cov] : PVIO_B200_OK;
    }
    return 0;
}

}  // extern "C"
