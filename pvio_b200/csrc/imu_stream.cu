// IMU stream slots (pvio_b200_batch_imu_stream): the IMU side of PVIO::Core for many sequences -- gyroscope and
// accelerometer synchronisation (core.cpp:59-107), the sorting of samples into pending camera frames (:129-141), the
// prepend rule of each released frame's sample list (feature_tracker.cpp:78-84) and the IMU-rate pose (:143-164 with
// propagate_state :32-39).  One thread per record: a sequence's events are a serial state machine.
//
// A sequence's poses are prefixes of one propagation chain from its latest state over its kept samples, which are in
// time order (the gyroscope and accelerometer times are checked to be non-decreasing, so the samples' accelerometer
// times are too).  So the chain is extended event by event instead of recomputed from the state per event, as
// predict_pose does; an event earlier than the chain's last sample restarts it from the state.  Both are the same
// operations in the same order, so the same bits.  Compiled with -fmad=false: the arithmetic is Eigen's scalar
// evaluation order without contraction (DESIGN 4.7h).
#include <cmath>
#include "api_internal.h"
#include "ba_math.cuh"
#include "imu_factor_cov.cuh"
#include "quat.cuh"

namespace pvio {

namespace {

constexpr double kGravityNominal = 9.80665;           // PVIO_GRAVITY_NOMINAL, common.h:62
constexpr int kMinQcap = 16;
constexpr int kStreamCovStride = 264;                 // ImuStreams::cov per slot: P [225], noise_cov [36], state time, pad

// one stream slot on the device: output extrinsic, latest state, the previously released frame's last row, and where
// each queue's live rows are in the slot's part of ImuStreams::g / a / s / f / k
struct ImuStreamSlot {
    double q_ob[4], p_ob[3];
    double state_t, state[16];
    double prev_t, prev_row[6];       // the previously released frame: its time, its list's last row (w xyz, a xyz)
    int32_t has_state, has_prev, prev_nonempty;
    int32_t drop_pending;             // a state was set and no pose has read it yet: the kept samples up to its time go at
                                      // the next pose, as predict_pose pops them (core.cpp:149-151)
    int32_t g0, gn, a0, an, s0, sn, nfront, f0, fn, k0, kn, pad2;   // head and size of each queue; nfront: the leading
                                                                     // unreleased samples given to the front frame
};

struct ImuStreamRec {                 // one record as staged
    int32_t slot, n_events, state_op, pad;
    double state_t, state[16];
    int64_t ev, pose, frame, row;     // first event / pose row / frame / sample row of the record in the call's arrays
    int32_t frame_cap, row_cap;       // the record's room for frames and rows (need_frames / need_rows)
};

struct ImuStreamOut {                 // one record's results, downloaded
    int32_t n_consumed, n_frames, n_rows, overflow;
    int32_t g, a, s, f, k, pad[3];    // queue sizes after the call
};

struct ImuStreamArgs {
    ImuStreamSlot *hdr;
    double *g, *a, *s, *f, *k;
    int qcap;
    const ImuStreamRec *recs;
    const double *events;             // [*][5]
    ImuStreamOut *outs;
    double *poses, *frame_t, *rows;   // [*][7], [*], [*][7]
    int32_t *frame_rows;
    int n;
};

__device__ inline void copy_rows(double *q, int w, int from, int n) {
    for (int j = 0; j < n * w; ++j) q[j] = q[from * w + j];
}

__global__ void __launch_bounds__(128) imu_stream_kernel(ImuStreamArgs A) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= A.n) return;
    const ImuStreamRec &R = A.recs[i];
    ImuStreamSlot &S = A.hdr[R.slot];
    const size_t qb = (size_t)R.slot * A.qcap;
    double *G = A.g + qb * 4, *Ac = A.a + qb * 4, *Sm = A.s + qb * 7, *F = A.f + qb, *K = A.k + qb * 7;
    // each queue's live rows to the front: the call's growth bound then fits in qcap
    copy_rows(G, 4, S.g0, S.gn);
    copy_rows(Ac, 4, S.a0, S.an);
    copy_rows(Sm, 7, S.s0, S.sn);
    copy_rows(F, 1, S.f0, S.fn);
    copy_rows(K, 7, S.k0, S.kn);
    int g0 = 0, gn = S.gn, a0 = 0, an = S.an, s0 = 0, sn = S.sn, nfront = S.nfront, f0 = 0, fn = S.fn, k0 = 0, kn = S.kn;

    if (R.state_op == PVIO_B200_IMU_STREAM_SET) {
        S.has_state = 1;
        S.state_t = R.state_t;
        for (int j = 0; j < 16; ++j) S.state[j] = R.state[j];
        S.drop_pending = 1;
    } else if (R.state_op == PVIO_B200_IMU_STREAM_CLEAR) {
        S.has_state = 0;
        S.drop_pending = 0;
    }
    const bool has_state = S.has_state != 0;
    const double state_t = S.state_t;

    ImuStreamOut &O = A.outs[i];
    double *ft = A.frame_t + R.frame, *rows = A.rows + R.row * 7;
    int32_t *frows = A.frame_rows + R.frame;
    int nf = 0, nr = 0, overflow = 0;

    // the propagation chain: c kept samples (from k0) applied to the latest state
    int c = 0;
    bool chain = false;
    double ct = 0, cq[4], cp[3], cv[3];

    // Core::track_imu: keep the sample for predict_pose, queue it, give queued samples to the front frame and release
    // frames that a later sample has passed
    auto track_imu = [&](double t, const double *w, const double *acc) -> bool {
        if (!(has_state && t <= state_t)) {            // the event's pose pops it before any use (:149-151)
            double *r = K + (k0 + kn) * 7;
            r[0] = t;
            for (int j = 0; j < 3; ++j) { r[1 + j] = w[j]; r[4 + j] = acc[j]; }
            ++kn;
        }
        double *r = Sm + (s0 + sn) * 7;
        r[0] = t;
        for (int j = 0; j < 3; ++j) { r[1 + j] = w[j]; r[4 + j] = acc[j]; }
        ++sn;
        bool released = false;
        while (sn > nfront && fn > 0) {
            const double tf = F[f0];
            if (Sm[(s0 + nfront) * 7] <= tf) { ++nfront; continue; }
            // release the front frame: its samples, with the prepend rule against the previous frame's list
            const bool prepend = S.has_prev && S.prev_nonempty && (nfront == 0 || Sm[s0 * 7] - S.prev_t > 1.0e-5);
            const int cnt = nfront + (prepend ? 1 : 0);
            if (nf >= R.frame_cap || nr + cnt > R.row_cap) { overflow = 1; return released; }
            double *o = rows + (size_t)nr * 7;
            if (prepend) {
                o[0] = S.prev_t;
                for (int j = 0; j < 6; ++j) o[1 + j] = S.prev_row[j];
                o += 7;
            }
            for (int j = 0; j < nfront * 7; ++j) o[j] = Sm[s0 * 7 + j];
            if (cnt > 0) {
                const double *last = rows + (size_t)(nr + cnt - 1) * 7;
                for (int j = 0; j < 6; ++j) S.prev_row[j] = last[1 + j];
            }
            S.has_prev = 1;
            S.prev_nonempty = cnt > 0;
            S.prev_t = tf;
            ft[nf] = tf;
            frows[nf] = cnt;
            ++nf;
            nr += cnt;
            s0 += nfront; sn -= nfront; nfront = 0;
            ++f0; --fn;
            if (!has_state) {                          // the next state is this frame's or a later one's
                while (kn > 0 && K[k0 * 7] <= tf) { ++k0; --kn; }
                chain = false;
            }
            released = true;
        }
        return released;
    };

    auto restart = [&]() {
        c = 0;
        ct = state_t;
        for (int j = 0; j < 4; ++j) cq[j] = S.state[j];
        for (int j = 0; j < 3; ++j) { cp[j] = S.state[4 + j]; cv[j] = S.state[7 + j]; }
        chain = true;
    };

    // Core::predict_pose at t, into pose row o
    auto predict = [&](double t, double *o) {
        if (!has_state) {
            for (int j = 0; j < 7; ++j) o[j] = 0.0;
            return;
        }
        if (S.drop_pending) {                            // predict_pose :149-151
            while (kn > 0 && K[k0 * 7] <= state_t) { ++k0; --kn; }
            S.drop_pending = 0;
            chain = false;
        }
        if (!chain || (c > 0 && K[(k0 + c - 1) * 7] > t)) restart();
        const double *bg = S.state + 10, *ba = S.state + 13;
        for (; c < kn && K[(k0 + c) * 7] <= t; ++c) {   // propagate_state, core.cpp:32-39
            const double *r = K + (k0 + c) * 7;
            const double dt = r[0] - ct;
            const double d[3] = {r[4] - ba[0], r[5] - ba[1], r[6] - ba[2]};
            double ra[3];
            bw_qrot(cq, d, ra);
            const double acc[3] = {0.0 + ra[0], 0.0 + ra[1], -kGravityNominal + ra[2]};
            const double hdt = 0.5 * dt * dt;
            for (int j = 0; j < 3; ++j) {
                cp[j] = cp[j] + dt * cv[j] + hdt * acc[j];
                cv[j] = cv[j] + dt * acc[j];
            }
            const double u[3] = {(r[1] - bg[0]) * dt, (r[2] - bg[1]) * dt, (r[3] - bg[2]) * dt};
            double e[4], qn[4];
            expmap(u, e);
            eigen_qmul(cq, e, qn);
            const double nrm = sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
            for (int j = 0; j < 4; ++j) cq[j] = qn[j] / nrm;
            ct = r[0];
        }
        double q[4], rp[3];
        eigen_qmul(cq, S.q_ob, q);                       // :158-159
        bw_qrot(cq, S.p_ob, rp);
        for (int j = 0; j < 4; ++j) o[j] = q[j];
        for (int j = 0; j < 3; ++j) o[4 + j] = cp[j] + rp[j];
    };

    int consumed = 0;
    for (int e = 0; e < R.n_events; ++e) {
        const double *ev = A.events + (size_t)(R.ev + e) * 5;
        const int kind = (int)ev[0];
        const double t = ev[1], v[3] = {ev[2], ev[3], ev[4]};
        bool released = false;
        if (kind == PVIO_B200_IMU_EVENT_GYROSCOPE) {                // Core::track_gyroscope
            if (an > 0) {
                if (t < Ac[a0 * 4]) {
                    g0 = 0; gn = 0;
                } else {
                    while (an > 0 && t >= Ac[a0 * 4]) {
                        const double *ac = Ac + a0 * 4, *g = G + g0 * 4;
                        const double lambda = (ac[0] - g[0]) / (t - g[0]);
                        const double w[3] = {g[1] + lambda * (v[0] - g[1]), g[2] + lambda * (v[1] - g[2]),
                                             g[3] + lambda * (v[2] - g[3])};
                        released |= track_imu(ac[0], w, ac + 1);
                        ++a0; --an;
                    }
                    if (an > 0)
                        while (gn > 0 && G[g0 * 4] < t) { ++g0; --gn; }
                }
            }
            double *g = G + (g0 + gn) * 4;
            g[0] = t; g[1] = v[0]; g[2] = v[1]; g[3] = v[2];
            ++gn;
        } else if (kind == PVIO_B200_IMU_EVENT_ACCELEROMETER) {     // Core::track_accelerometer
            if (gn > 0 && t >= G[g0 * 4]) {
                const double tb = G[(g0 + gn - 1) * 4];
                if (t > tb) {
                    g0 += gn - 1; gn = 1;
                    double *a = Ac + (a0 + an) * 4;
                    a[0] = t; a[1] = v[0]; a[2] = v[1]; a[3] = v[2];
                    ++an;
                } else if (t == tb) {
                    g0 += gn - 1; gn = 1;
                    released = track_imu(t, G + g0 * 4 + 1, v);
                } else {
                    while (t >= G[(g0 + 1) * 4]) { ++g0; --gn; }
                    const double *g = G + g0 * 4, *g1 = g + 4;
                    const double lambda = (t - g[0]) / (g1[0] - g[0]);
                    const double w[3] = {g[1] + lambda * (g1[1] - g[1]), g[2] + lambda * (g1[2] - g[2]),
                                         g[3] + lambda * (g1[3] - g[3])};
                    released = track_imu(t, w, v);
                }
            }
        } else {                                                    // Core::track_camera: the frame waits for samples
            F[f0 + fn] = t;
            ++fn;
        }
        predict(t, A.poses + (size_t)(R.pose + e) * 7);
        consumed = e + 1;
        if (released || overflow) break;
    }

    S.g0 = g0; S.gn = gn; S.a0 = a0; S.an = an; S.s0 = s0; S.sn = sn; S.nfront = nfront;
    S.f0 = f0; S.fn = fn; S.k0 = k0; S.kn = kn;
    O.n_consumed = consumed; O.n_frames = nf; O.n_rows = nr; O.overflow = overflow;
    O.g = gn; O.a = an; O.s = sn; O.f = fn; O.k = kn;
}

// reset: slot list and headers staged back to back
__global__ void imu_stream_reset_kernel(int n, const int32_t *slots, const ImuStreamSlot *src, ImuStreamSlot *hdr) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) hdr[slots[i]] = src[i];
}

// device queues for `slots` slots of at least `qcap` rows each; growth keeps every slot's queues and header
int ensure_streams(Handle *h, int slots, int qcap) {
    ImuStreams &M = h->imus;
    if (slots <= M.slots && qcap <= M.qcap) return 0;
    const int ns = slots <= M.slots ? M.slots : std::max(slots, std::min(std::max(2 * M.slots, 64), kMaxBatchSlot + 1));
    int nq = std::max(M.qcap, kMinQcap);
    while (nq < qcap) nq *= 2;
    CK(h, cudaStreamSynchronize(h->stream));
    DevBuf<uint8_t> hdr;
    TRY(alloc(h, hdr, sizeof(ImuStreamSlot) * ns, kDevice));
    if (M.slots) CK(h, cudaMemcpyAsync(hdr.d, M.hdr.d, sizeof(ImuStreamSlot) * M.slots, cudaMemcpyDeviceToDevice, h->stream));
    DevBuf<double> cov;
    if (ns > M.slots) {
        TRY(alloc(h, cov, (size_t)ns * kStreamCovStride, kDevice));
        if (M.slots)
            CK(h, cudaMemcpyAsync(cov.d, M.cov.d, sizeof(double) * kStreamCovStride * M.slots, cudaMemcpyDeviceToDevice,
                                  h->stream));
    }
    DevBuf<double> *qs[5] = {&M.g, &M.a, &M.s, &M.f, &M.k};
    const int width[5] = {4, 4, 7, 1, 7};
    DevBuf<double> grown[5];
    for (int q = 0; q < 5; ++q) {
        TRY(alloc(h, grown[q], (size_t)ns * nq * width[q], kDevice));
        if (M.slots)
            CK(h, cudaMemcpy2DAsync(grown[q].d, sizeof(double) * nq * width[q], qs[q]->d, sizeof(double) * M.qcap * width[q],
                                    sizeof(double) * M.qcap * width[q], M.slots, cudaMemcpyDeviceToDevice, h->stream));
    }
    CK(h, cudaStreamSynchronize(h->stream));
    M.hdr = std::move(hdr);
    if (ns > M.slots) M.cov = std::move(cov);
    for (int q = 0; q < 5; ++q) *qs[q] = std::move(grown[q]);
    M.slots = ns;
    M.qcap = nq;
    return 0;
}

bool finite_all(const double *v, int n) {
    for (int j = 0; j < n; ++j)
        if (!std::isfinite(v[j])) return false;
    return true;
}

int stream_reset_impl(Handle *h, int n, const int32_t *slots, const double *oq, const double *op) {
    if (n < 0) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_reset: bad slot count");
    if (n == 0) return 0;
    if (!slots || !oq || !op) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_reset: bad arguments");
    std::vector<uint8_t> taken;
    int top = 0;
    for (int i = 0; i < n; ++i) {
        const int s = slots[i];
        TRY(take_slot(h, taken, s, "batch_imu_stream_reset"));
        if (!finite_all(oq + 4 * i, 4) || !finite_all(op + 3 * i, 3))
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_reset: an extrinsic value is not finite");
        top = std::max(top, s + 1);
    }
    ImuStreams &M = h->imus;
    TRY(ensure_streams(h, top, kMinQcap));
    Stage S(M.stage);
    const auto sl = S.add(Stage::kUp, n, slots);
    const auto hdr = S.add<ImuStreamSlot>(Stage::kUp, n);
    TRY(S.place(h));
    ImuStreamSlot *hs = S.host(hdr);
    for (int i = 0; i < n; ++i) {
        ImuStreamSlot z{};
        for (int j = 0; j < 4; ++j) z.q_ob[j] = oq[4 * i + j];
        for (int j = 0; j < 3; ++j) z.p_ob[j] = op[3 * i + j];
        hs[i] = z;
    }
    cudaStream_t st = h->stream;
    TRY(S.upload(h));
    imu_stream_reset_kernel<<<(n + 127) / 128, 128, 0, st>>>(n, S.dev(sl), S.dev(hdr), reinterpret_cast<ImuStreamSlot *>(M.hdr.d));
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(st));
    if ((size_t)top > M.host.size()) M.host.resize(top);
    M.cov_host.resize(M.host.size());
    for (int i = 0; i < n; ++i) {
        M.host[slots[i]] = ImuStreamHost{};
        M.host[slots[i]].set = true;
        ++M.cov_host[slots[i]].gen;
    }
    return 0;
}

// what checking a record finds: its queue bounds and its room
struct StreamNeed {
    int64_t frames = 0, rows = 0, queue = 0;
};

int stream_impl(Handle *h, int n, pvio_b200_imu_stream_record *recs) {
    if (n < 0) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: bad record count");
    if (n == 0) return 0;
    if (!recs) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: bad arguments");
    ImuStreams &M = h->imus;
    std::vector<uint8_t> taken;
    std::vector<StreamNeed> need(n);
    bool query = false;
    int64_t total_ev = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_record &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_imu_stream"));
        if ((size_t)r.slot >= M.host.size() || !M.host[r.slot].set)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: the slot was never reset");
        const ImuStreamHost &S = M.host[r.slot];
        if (r.n_events < 0 || (r.n_events > 0 && (!r.events || !r.poses)))
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: bad event count or pointer");
        if (r.state_op < PVIO_B200_IMU_STREAM_KEEP || r.state_op > PVIO_B200_IMU_STREAM_CLEAR)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: unknown state_op");
        if (r.state_op == PVIO_B200_IMU_STREAM_SET) {
            if (!r.state || !std::isfinite(r.state_time) || !finite_all(r.state, 16))
                return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: a SET state is missing or not finite");
            if (S.dropped && r.state_time < S.t_drop)
                return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: the state is older than a frame released without one");
        }
        int64_t ng = 0, na = 0, nc = 0;
        bool seen_g = S.seen_g, seen_a = S.seen_a;
        double last_g = S.last_g, last_a = S.last_a;
        for (int e = 0; e < r.n_events; ++e) {
            const double *ev = r.events + (size_t)e * 5;
            if (!finite_all(ev, 5)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: an event value is not finite");
            const double t = ev[1];
            if (ev[0] == PVIO_B200_IMU_EVENT_GYROSCOPE) {
                if (seen_g && t < last_g) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: a gyroscope time decreases");
                seen_g = true; last_g = t; ++ng;
            } else if (ev[0] == PVIO_B200_IMU_EVENT_ACCELEROMETER) {
                if (seen_a && t < last_a) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: an accelerometer time decreases");
                seen_a = true; last_a = t; ++na;
            } else if (ev[0] == PVIO_B200_IMU_EVENT_CAMERA) {
                ++nc;
            } else {
                return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: unknown event kind");
            }
        }
        StreamNeed &d = need[i];
        d.frames = S.f + nc;
        d.rows = S.s + S.a + na + d.frames;
        d.queue = std::max({S.g + ng, S.a + na, S.s + S.a + na, S.f + nc, S.k + S.a + na});
        if (d.queue > PVIO_B200_IMU_STREAM_MAX_QUEUE)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: a queue could exceed PVIO_B200_IMU_STREAM_MAX_QUEUE");
        if (!r.rows) query = true;
        total_ev += r.n_events;
    }
    if (query) {
        for (int i = 0; i < n; ++i) { recs[i].need_frames = (int32_t)need[i].frames; recs[i].need_rows = need[i].rows; }
        return 0;
    }
    int64_t total_f = 0, total_r = 0, qcap = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_record &r = recs[i];
        if (r.max_frames < need[i].frames || r.max_rows < need[i].rows || (need[i].frames > 0 && (!r.frame_t || !r.frame_rows)))
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream: max_frames / max_rows below need_frames / need_rows");
        total_f += need[i].frames;
        total_r += need[i].rows;
        qcap = std::max(qcap, need[i].queue);
    }
    TRY(ensure_streams(h, M.slots, (int)qcap));

    // staging: records | events (uploaded) || outputs | poses | frame times | rows | frame row counts (downloaded)
    Stage stage(M.stage);
    const auto rec = stage.add<ImuStreamRec>(Stage::kUp, n);
    const auto evs = stage.add<double>(Stage::kUp, 5 * total_ev);
    const auto out = stage.add<ImuStreamOut>(Stage::kDown, n);
    const auto pose = stage.add<double>(Stage::kDown, 7 * total_ev);
    const auto ft = stage.add<double>(Stage::kDown, total_f);
    const auto rws = stage.add<double>(Stage::kDown, 7 * total_r);
    const auto frw = stage.add<int32_t>(Stage::kDown, total_f);
    TRY(stage.place(h));
    ImuStreamRec *hr = stage.host(rec);
    double *hev = stage.host(evs);
    int64_t ev = 0, fr = 0, row = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_record &r = recs[i];
        ImuStreamRec R{};
        R.slot = r.slot; R.n_events = r.n_events; R.state_op = r.state_op;
        if (r.state_op == PVIO_B200_IMU_STREAM_SET) {
            R.state_t = r.state_time;
            memcpy(R.state, r.state, sizeof(R.state));
        }
        R.ev = ev; R.pose = ev; R.frame = fr; R.row = row;
        R.frame_cap = (int32_t)need[i].frames; R.row_cap = (int32_t)need[i].rows;
        hr[i] = R;
        if (r.n_events) memcpy(hev + ev * 5, r.events, sizeof(double) * 5 * r.n_events);
        ev += r.n_events; fr += need[i].frames; row += need[i].rows;
    }
    ImuStreamArgs A;
    A.hdr = reinterpret_cast<ImuStreamSlot *>(M.hdr.d);
    A.g = M.g.d; A.a = M.a.d; A.s = M.s.d; A.f = M.f.d; A.k = M.k.d;
    A.qcap = M.qcap;
    A.recs = stage.dev(rec);
    A.events = stage.dev(evs);
    A.outs = stage.dev(out);
    A.poses = stage.dev(pose);
    A.frame_t = stage.dev(ft);
    A.rows = stage.dev(rws);
    A.frame_rows = stage.dev(frw);
    A.n = n;
    cudaStream_t st = h->stream;
    TRY(stage.upload(h));
    imu_stream_kernel<<<(n + 127) / 128, 128, 0, st>>>(A);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(stage.download(h));
    CK(h, cudaStreamSynchronize(st));

    // Internal invariant: the host bounds (need_frames / need_rows) hold every release, so overflow is never set.  Were
    // it set, the kernel would already have changed the call's slots without the host's record of them following, so
    // every slot of the call is marked unset: later calls on them are rejected until they are reset.
    const ImuStreamOut *outs = stage.host(out);
    for (int i = 0; i < n; ++i)
        if (outs[i].overflow) {
            for (int j = 0; j < n; ++j) M.host[recs[j].slot].set = false;
            return fail(h, PVIO_B200_ECUDA, "batch_imu_stream: a record's releases exceeded its bound (internal "
                                            "error); the call's slots must be reset");
        }
    for (int i = 0; i < n; ++i) {
        pvio_b200_imu_stream_record &r = recs[i];
        const ImuStreamRec &R = hr[i];
        const ImuStreamOut &O = outs[i];
        memcpy(r.poses, stage.host(pose) + 7 * R.pose, sizeof(double) * 7 * O.n_consumed);
        const double *ftr = stage.host(ft) + R.frame;
        if (O.n_frames) {
            memcpy(r.frame_t, ftr, sizeof(double) * O.n_frames);
            memcpy(r.frame_rows, stage.host(frw) + R.frame, sizeof(int32_t) * O.n_frames);
        }
        if (O.n_rows) memcpy(r.rows, stage.host(rws) + 7 * R.row, sizeof(double) * 7 * O.n_rows);
        r.n_consumed = O.n_consumed;
        r.n_frames = O.n_frames;
        r.need_frames = (int32_t)need[i].frames;
        r.need_rows = need[i].rows;
        ImuStreamHost &S = M.host[r.slot];
        if (r.state_op == PVIO_B200_IMU_STREAM_SET) S.has_state = true;
        if (r.state_op == PVIO_B200_IMU_STREAM_CLEAR) S.has_state = false;
        if (r.state_op != PVIO_B200_IMU_STREAM_KEEP) {       // the seed of the previous state no longer holds
            ++M.cov_host[r.slot].gen;
            M.cov_host[r.slot].state_t = r.state_time;
        }
        for (int e = 0; e < O.n_consumed; ++e) {
            const double *evr = r.events + (size_t)e * 5;
            if (evr[0] == PVIO_B200_IMU_EVENT_GYROSCOPE) { S.seen_g = true; S.last_g = evr[1]; }
            if (evr[0] == PVIO_B200_IMU_EVENT_ACCELEROMETER) { S.seen_a = true; S.last_a = evr[1]; }
        }
        if (!S.has_state)
            for (int k = 0; k < O.n_frames; ++k) {
                S.t_drop = S.dropped ? std::max(S.t_drop, ftr[k]) : ftr[k];
                S.dropped = true;
            }
        S.g = O.g; S.a = O.a; S.s = O.s; S.f = O.f; S.k = O.k;
    }
    return 0;
}

// ------------------------------------------------------------ snapshots (pvio_b200_batch_imu_stream_save / restore)
// A blob: StreamSnapHead, then the live rows of the five queues back to back in queue order (gyroscope [n0][4],
// accelerometer [n1][4], unreleased samples [n2][7], pending frame stamps [n3], kept samples [n4][7]), oldest first.
// The head's first part is the host record (written by the host), `dev` the slot's device header (written by the pack
// kernel).  No slot, head offset, Qcap or pointer, so save -> restore -> save gives the same bytes in any stream slot.
struct StreamSnapDev {
    double q_ob[4], p_ob[3];
    double state_t, state[16];
    double prev_t, prev_row[6];
    int32_t has_state, drop_pending, has_prev, prev_nonempty, nfront, pad;
};
struct StreamSnapHead {
    uint32_t magic, version;
    int64_t size;                     // bytes of the blob
    int32_t n[5];                     // rows of each queue
    int32_t seen_g, seen_a, dropped;  // ImuStreamHost
    double last_g, last_a, t_drop;
    StreamSnapDev dev;
};
static_assert(sizeof(StreamSnapHead) == 344 && offsetof(StreamSnapHead, dev) == 72 && sizeof(StreamSnapDev) == 272,
              "the head has no implicit padding; the queue sections start 8-byte aligned");
constexpr int kSnapThreads = 128;

// row width of queue q (g, a, s, f, k)
__host__ __device__ inline int queue_width(int q) { return q < 2 ? 4 : q == 3 ? 1 : 7; }

__host__ __device__ inline int64_t stream_snap_size(const int32_t *n) {
    int64_t s = sizeof(StreamSnapHead);
    for (int q = 0; q < 5; ++q) s += sizeof(double) * queue_width(q) * (int64_t)n[q];
    return s;
}

struct StreamSnapRec {                // one record of a save or restore call: its stream slot, its blob's byte offset
    int32_t slot, pad;                // in the call's area
    int64_t at;
};
struct StreamSnapArgs {
    ImuStreamSlot *hdr;
    double *q[5];                     // g, a, s, f, k
    int qcap;
    const StreamSnapRec *recs;
    uint8_t *area;
};

// n doubles from src to dst by the CTA; returns dst + n
__device__ __forceinline__ double *snap_rows(double *dst, const double *src, int n) {
    for (int j = threadIdx.x; j < n; j += kSnapThreads) dst[j] = src[j];
    return dst + n;
}

// One CTA per save record: the slot's device header into the blob's head and each queue's live rows [head, head + n)
// into its section.  The host writes the rest of the head.
__global__ void __launch_bounds__(kSnapThreads) imu_stream_pack_kernel(StreamSnapArgs A) {
    const StreamSnapRec &R = A.recs[blockIdx.x];
    const ImuStreamSlot &S = A.hdr[R.slot];
    uint8_t *blob = A.area + R.at;
    const size_t qb = (size_t)R.slot * A.qcap;
    double *dst = reinterpret_cast<double *>(blob + sizeof(StreamSnapHead));
    dst = snap_rows(dst, A.q[0] + (qb + S.g0) * 4, S.gn * 4);
    dst = snap_rows(dst, A.q[1] + (qb + S.a0) * 4, S.an * 4);
    dst = snap_rows(dst, A.q[2] + (qb + S.s0) * 7, S.sn * 7);
    dst = snap_rows(dst, A.q[3] + (qb + S.f0), S.fn);
    snap_rows(dst, A.q[4] + (qb + S.k0) * 7, S.kn * 7);
    if (threadIdx.x == 0) {
        StreamSnapDev &d = reinterpret_cast<StreamSnapHead *>(blob)->dev;
        for (int j = 0; j < 4; ++j) d.q_ob[j] = S.q_ob[j];
        for (int j = 0; j < 3; ++j) d.p_ob[j] = S.p_ob[j];
        d.state_t = S.state_t;
        for (int j = 0; j < 16; ++j) d.state[j] = S.state[j];
        d.prev_t = S.prev_t;
        for (int j = 0; j < 6; ++j) d.prev_row[j] = S.prev_row[j];
        d.has_state = S.has_state; d.drop_pending = S.drop_pending; d.has_prev = S.has_prev;
        d.prev_nonempty = S.prev_nonempty; d.nfront = S.nfront; d.pad = 0;
    }
}

// One CTA per restore record: each queue's rows to the front of the target slot (heads 0), then its header.
__global__ void __launch_bounds__(kSnapThreads) imu_stream_unpack_kernel(StreamSnapArgs A) {
    const StreamSnapRec &R = A.recs[blockIdx.x];
    const uint8_t *blob = A.area + R.at;
    const StreamSnapHead &H = *reinterpret_cast<const StreamSnapHead *>(blob);
    const double *src = reinterpret_cast<const double *>(blob + sizeof(StreamSnapHead));
    const size_t qb = (size_t)R.slot * A.qcap;
    snap_rows(A.q[0] + qb * 4, src, H.n[0] * 4);
    src += H.n[0] * 4;
    snap_rows(A.q[1] + qb * 4, src, H.n[1] * 4);
    src += H.n[1] * 4;
    snap_rows(A.q[2] + qb * 7, src, H.n[2] * 7);
    src += H.n[2] * 7;
    snap_rows(A.q[3] + qb, src, H.n[3]);
    src += H.n[3];
    snap_rows(A.q[4] + qb * 7, src, H.n[4] * 7);
    if (threadIdx.x == 0) {
        const StreamSnapDev &d = H.dev;
        ImuStreamSlot S{};
        for (int j = 0; j < 4; ++j) S.q_ob[j] = d.q_ob[j];
        for (int j = 0; j < 3; ++j) S.p_ob[j] = d.p_ob[j];
        S.state_t = d.state_t;
        for (int j = 0; j < 16; ++j) S.state[j] = d.state[j];
        S.prev_t = d.prev_t;
        for (int j = 0; j < 6; ++j) S.prev_row[j] = d.prev_row[j];
        S.has_state = d.has_state; S.drop_pending = d.drop_pending; S.has_prev = d.has_prev;
        S.prev_nonempty = d.prev_nonempty; S.nfront = d.nfront;
        S.gn = H.n[0]; S.an = H.n[1]; S.sn = H.n[2]; S.fn = H.n[3]; S.kn = H.n[4];
        A.hdr[R.slot] = S;
    }
}

StreamSnapArgs snap_args(Handle *h, const StreamSnapRec *recs, uint8_t *area) {
    ImuStreams &M = h->imus;
    StreamSnapArgs A;
    A.hdr = reinterpret_cast<ImuStreamSlot *>(M.hdr.d);
    A.q[0] = M.g.d; A.q[1] = M.a.d; A.q[2] = M.s.d; A.q[3] = M.f.d; A.q[4] = M.k.d;
    A.qcap = M.qcap;
    A.recs = recs;
    A.area = area;
    return A;
}

int stream_save_impl(Handle *h, int n, pvio_b200_imu_stream_snapshot *recs) {
    if (n < 0 || (n > 0 && !recs)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_save: bad record list");
    if (n == 0) return 0;
    ImuStreams &M = h->imus;
    std::vector<uint8_t> taken;
    std::vector<int64_t> size(n), at(n, -1);
    int64_t area = 0;
    int packed = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_snapshot &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_imu_stream_save"));
        if ((size_t)r.slot >= M.host.size() || !M.host[r.slot].set)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_save: the slot was never reset");
        const ImuStreamHost &S = M.host[r.slot];
        const int32_t cnt[5] = {(int32_t)S.g, (int32_t)S.a, (int32_t)S.s, (int32_t)S.f, (int32_t)S.k};
        size[i] = stream_snap_size(cnt);
        if (!r.data) continue;
        if (r.capacity < size[i]) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_save: capacity below the record's size");
        at[i] = area;
        area += (int64_t)align256(size[i]);
        ++packed;
    }
    if (packed) {
        // staging: records (uploaded) | blobs (downloaded)
        Stage stage(M.stage);
        const auto rc = stage.add<StreamSnapRec>(Stage::kUp, packed);
        const auto blobs = stage.add<uint8_t>(Stage::kDown, area);
        TRY(stage.place(h));
        StreamSnapRec *hr = stage.host(rc);
        for (int i = 0, j = 0; i < n; ++i)
            if (at[i] >= 0) hr[j++] = StreamSnapRec{recs[i].slot, 0, at[i]};
        cudaStream_t st = h->stream;
        TRY(stage.upload(h));
        imu_stream_pack_kernel<<<packed, kSnapThreads, 0, st>>>(snap_args(h, stage.dev(rc), stage.dev(blobs)));
        ++h->launches;
        CK(h, cudaGetLastError());
        TRY(stage.download(h));
        CK(h, cudaStreamSynchronize(st));
        for (int i = 0; i < n; ++i) {
            if (at[i] < 0) continue;
            const ImuStreamHost &S = M.host[recs[i].slot];
            uint8_t *out = recs[i].data;
            memcpy(out, stage.host(blobs) + at[i], size[i]);
            StreamSnapHead H;
            memcpy(&H, out, sizeof(H));
            H.magic = PVIO_B200_IMU_STREAM_SNAPSHOT_MAGIC;
            H.version = PVIO_B200_IMU_STREAM_SNAPSHOT_VERSION;
            H.size = size[i];
            H.n[0] = (int32_t)S.g; H.n[1] = (int32_t)S.a; H.n[2] = (int32_t)S.s; H.n[3] = (int32_t)S.f; H.n[4] = (int32_t)S.k;
            H.seen_g = S.seen_g; H.seen_a = S.seen_a; H.dropped = S.dropped;
            H.last_g = S.last_g; H.last_a = S.last_a; H.t_drop = S.t_drop;
            memcpy(out, &H, sizeof(H));
        }
    }
    for (int i = 0; i < n; ++i) recs[i].size = size[i];
    return 0;
}

// why a blob cannot be restored, or nullptr
const char *stream_snap_check(const uint8_t *data, int64_t bytes, StreamSnapHead &H) {
    if (!data || bytes < (int64_t)sizeof(StreamSnapHead)) return "a blob shorter than its head";
    memcpy(&H, data, sizeof(H));
    if (H.magic != PVIO_B200_IMU_STREAM_SNAPSHOT_MAGIC || H.version != PVIO_B200_IMU_STREAM_SNAPSHOT_VERSION)
        return "not a stream slot blob of this version";
    for (int q = 0; q < 5; ++q)
        if (H.n[q] < 0 || H.n[q] > PVIO_B200_IMU_STREAM_MAX_QUEUE) return "a queue count out of range";
    const StreamSnapDev &d = H.dev;
    if (d.nfront < 0 || d.nfront > H.n[2]) return "nfront above the unreleased samples";
    if (H.size != bytes || H.size != stream_snap_size(H.n)) return "the declared size is not the blob's";
    const int32_t flags[7] = {H.seen_g, H.seen_a, H.dropped, d.has_state, d.drop_pending, d.has_prev, d.prev_nonempty};
    for (int32_t f : flags)
        if (f != 0 && f != 1) return "a flag outside 0 / 1";
    if (d.pad != 0) return "a padding field not zero";
    if (d.drop_pending && !d.has_state) return "drop_pending without a state";
    if (d.prev_nonempty && !d.has_prev) return "prev_nonempty without a previous frame";
    const double head_v[3] = {H.last_g, H.last_a, H.t_drop};
    if (!finite_all(head_v, 3) || !finite_all(d.q_ob, 4) || !finite_all(d.p_ob, 3) || !finite_all(&d.state_t, 1) ||
        !finite_all(d.state, 16) || !finite_all(&d.prev_t, 1) || !finite_all(d.prev_row, 6))
        return "a head value is not finite";
    if (d.has_state && H.dropped && H.t_drop > d.state_t) return "the state is older than a frame released without one";
    const double *v = reinterpret_cast<const double *>(data + sizeof(StreamSnapHead));
    const bool seen[5] = {H.seen_g != 0, H.seen_a != 0, H.seen_g && H.seen_a, true, H.seen_g && H.seen_a};
    for (int q = 0; q < 5; ++q) {
        const int w = queue_width(q);
        if (!finite_all(v, w * H.n[q])) return "a queue value is not finite";
        if (H.n[q] > 0 && !seen[q]) return "a non-empty queue of a stream never seen";
        for (int r = 1; r < H.n[q] && q != 3; ++r)
            if (v[r * w] < v[(r - 1) * w]) return "a queue's times decrease";
        if (H.n[q] > 0 && q < 2 && v[(H.n[q] - 1) * w] > (q == 0 ? H.last_g : H.last_a))
            return "a queued reading newer than its stream's last";
        v += (size_t)w * H.n[q];
    }
    return nullptr;
}

int stream_restore_impl(Handle *h, int n, const pvio_b200_imu_stream_snapshot *recs) {
    if (n < 0 || (n > 0 && !recs)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_restore: bad record list");
    if (n == 0) return 0;
    ImuStreams &M = h->imus;
    std::vector<uint8_t> taken;
    std::vector<StreamSnapHead> heads(n);
    int top = 0, qcap = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_snapshot &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_imu_stream_restore"));
        if (const char *why = stream_snap_check(r.data, r.capacity, heads[i]))
            return fail(h, PVIO_B200_EINVAL, (std::string("batch_imu_stream_restore: ") + why).c_str());
        top = std::max(top, r.slot + 1);
        for (int q = 0; q < 5; ++q) qcap = std::max(qcap, heads[i].n[q]);
    }
    TRY(ensure_streams(h, top, qcap));

    // staging: records | blobs, uploaded
    size_t area = 0;
    for (int i = 0; i < n; ++i) area += align256(heads[i].size);
    Stage stage(M.stage);
    const auto rc = stage.add<StreamSnapRec>(Stage::kUp, n);
    const auto blobs = stage.add<uint8_t>(Stage::kUp, area);
    TRY(stage.place(h));
    StreamSnapRec *hr = stage.host(rc);
    size_t at = 0;
    for (int i = 0; i < n; ++i) {
        hr[i] = StreamSnapRec{recs[i].slot, 0, (int64_t)at};
        memcpy(stage.host(blobs) + at, recs[i].data, heads[i].size);
        at += align256(heads[i].size);
    }
    cudaStream_t st = h->stream;
    TRY(stage.upload(h));
    imu_stream_unpack_kernel<<<n, kSnapThreads, 0, st>>>(snap_args(h, stage.dev(rc), stage.dev(blobs)));
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(st));
    if ((size_t)top > M.host.size()) M.host.resize(top);
    M.cov_host.resize(M.host.size());
    for (int i = 0; i < n; ++i) {
        const StreamSnapHead &H = heads[i];
        ImuStreamCovHost &C = M.cov_host[recs[i].slot];
        ++C.gen;
        C.state_t = H.dev.state_t;
        ImuStreamHost &S = M.host[recs[i].slot];
        S.set = true;
        S.has_state = H.dev.has_state;
        S.seen_g = H.seen_g; S.last_g = H.last_g;
        S.seen_a = H.seen_a; S.last_a = H.last_a;
        S.dropped = H.dropped; S.t_drop = H.t_drop;
        S.g = H.n[0]; S.a = H.n[1]; S.s = H.n[2]; S.f = H.n[3]; S.k = H.n[4];
    }
    return 0;
}


// ------------------------------------------------------------ covariance (pvio_b200_batch_imu_stream_set_covariance / predict)
// A slot's seed (ImuStreams::cov) is the covariance of its latest state in [dtheta dp dv dbg dba], q perturbed on the
// right, with the noise_cov the prediction propagates with.  Both kernels run one warp per record on 15 x 15 matrices in
// shared memory (row-major).
constexpr int kCovWarps = 4;                          // records per CTA

struct StreamSeedRec {                // one set_covariance record as staged
    int32_t slot, mode;
    double state_t;
    double cov[225];
    double imu[PVIO_B200_IMU_STRIDE];  // FACTOR: the factor of the prediction
    double noise[36];
};

// One warp per record.  DIRECT: the symmetrised cov.  FACTOR: Phi Sigma_src Phi^T + Psi Sigma_d Psi^T
// (imu_factor_propagate), with Sigma_d = U^-1 U^-T from the factor's upper-triangular U = sqrt_inv_cov.
__global__ void __launch_bounds__(32 * kCovWarps) imu_stream_seed_kernel(int n, const StreamSeedRec *recs,
                                                                         const ImuStreamSlot *hdr, double *cov) {
    __shared__ double sm[kCovWarps][4][225];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kCovWarps + w;
    if (i >= n) return;
    const StreamSeedRec &R = recs[i];
    double *A = sm[w][0], *B = sm[w][1], *C = sm[w][2], *D = sm[w][3];
    for (int e = lane; e < 225; e += 32) {
        const int r = e / 15, c = e % 15;
        A[e] = 0.5 * (R.cov[r * 15 + c] + R.cov[c * 15 + r]);
        D[e] = 0.0;
    }
    __syncwarp();
    if (R.mode == PVIO_B200_IMU_STREAM_COV_FACTOR) {
        const double *rec = R.imu, *dq = rec + PVIO_B200_IMU_DQ;
        double qs[4], Rs[9], dR[9];
        {
            double ci[4];
            quat_conj(dq, ci);
            quat_mul(hdr[R.slot].state, ci, qs);
            quat_to_mat(qs, Rs);
            quat_to_mat(dq, dR);
        }
        if (lane < 15) {                                 // column `lane` of U^-1 into C, by back substitution
            const double *U = rec + PVIO_B200_IMU_SQRT_INV_COV;
            const int j = lane;
            for (int r = 14; r > j; --r) C[r * 15 + j] = 0.0;
            C[j * 15 + j] = 1.0 / U[j * 15 + j];
            for (int r = j - 1; r >= 0; --r) {
                double s = 0.0;
                for (int m = r + 1; m <= j; ++m) s += U[r * 15 + m] * C[m * 15 + j];
                C[r * 15 + j] = -s / U[r * 15 + r];
            }
        }
        __syncwarp();
        warp_mm15(C, C, D, true, lane);                  // Sigma_d = U^-1 U^-T
        const ImuFactorJac f{rec[PVIO_B200_IMU_DT], rec + PVIO_B200_IMU_DP, rec + PVIO_B200_IMU_DV,
                             rec + PVIO_B200_IMU_DQ_DBG, rec + PVIO_B200_IMU_DP_DBG, rec + PVIO_B200_IMU_DP_DBA,
                             rec + PVIO_B200_IMU_DV_DBG, rec + PVIO_B200_IMU_DV_DBA};
        imu_factor_propagate(A, B, C, D, f, Rs, dR, lane);
    }
    double *out = cov + (size_t)R.slot * kStreamCovStride;
    for (int e = lane; e < 225; e += 32) {
        const int r = e / 15, c = e % 15;
        out[e] = 0.5 * ((A[e] + D[e]) + (A[c * 15 + r] + D[c * 15 + r]));
    }
    for (int e = lane; e < 36; e += 32) out[225 + e] = R.noise[e];
    if (lane == 0) { out[261] = R.state_t; out[262] = out[263] = 0.0; }
}

struct StreamPredRec {                // one predict record as staged
    int32_t slot, n_times, has_cov, pad;
    int64_t t_at;                     // its first time in the call's times
    int64_t pose_at, state_at, pcov_at, scov_at;   // its first row in each output section; -1: not asked
};
struct StreamPredArgs {
    const ImuStreamSlot *hdr;
    const double *k, *cov;
    int qcap;
    const StreamPredRec *recs;
    const double *times;
    double *poses, *states, *pcov, *scov;         // [*][7], [*][16], [*][36], [*][225]
    int n;
};
constexpr int kStepVals = 96;         // per warp: one step's F and noise blocks, the emit's blocks, the seed's noise_cov

// One warp per record.  Every lane runs the pose chain of imu_stream_kernel's predict (the same operations in the same
// order, so the same bits); lane 0 writes each step's blocks of F and of the noise, and the lanes propagate P:
// F = I + [theta: E^T, -dt Jr at bg; p: -dt^2/2 R hat(a), dt I at v, -dt^2/2 R at ba; v: -dt R hat(a), -dt R at ba],
// P <- F P F^T as two column passes (Y = F P, then F Y^T) that each touch only the theta, p and v rows, then the exact
// symmetrisation plus the noise.  Outputs as the chain passes each requested time.
__global__ void __launch_bounds__(32 * kCovWarps) imu_stream_predict_kernel(StreamPredArgs A) {
    __shared__ double sm[kCovWarps][2][225];
    __shared__ double sv[kCovWarps][kStepVals];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int i = blockIdx.x * kCovWarps + w;
    if (i >= A.n) return;
    const StreamPredRec &R = A.recs[i];
    const ImuStreamSlot &S = A.hdr[R.slot];
    const bool has_state = S.has_state != 0, has_cov = has_state && R.has_cov;
    double *P = sm[w][0], *Y = sm[w][1], *V = sv[w];
    // V: [0] R, [9] R hat(a), [18] E^T, [27] dt Jr, [36] Nw, [45] Na (3 x 3 each), [54] dt, [55] R_ob, [64] R hat(p_ob),
    // [73] noise_cov bg, [82] ba
    double *Rv = V, *Mv = V + 9, *Et = V + 18, *Jv = V + 27, *Nw = V + 36, *Na = V + 45, *Rob = V + 55, *Kp = V + 64;
    const double *seed = A.cov + (size_t)R.slot * kStreamCovStride;
    if (has_cov) {
        for (int e = lane; e < 225; e += 32) P[e] = seed[e];
        if (lane < 18) V[73 + lane] = seed[225 + 18 + lane];
        if (lane == 0) quat_to_mat(S.q_ob, Rob);
    }
    __syncwarp();
    const double *K = A.k + ((size_t)R.slot * A.qcap + S.k0) * 7;
    const int kn = S.kn;
    const double state_t = S.state_t;
    int c = 0;
    if (has_state && S.drop_pending)                    // predict_pose :149-151, skipped: the call changes no slot
        while (c < kn && K[c * 7] <= state_t) ++c;
    double ct = state_t, cq[4], cp[3], cv[3];
    for (int j = 0; j < 4; ++j) cq[j] = S.state[j];
    for (int j = 0; j < 3; ++j) { cp[j] = S.state[4 + j]; cv[j] = S.state[7 + j]; }
    const double *bg = S.state + 10, *ba = S.state + 13;
    const double nan = __longlong_as_double(0x7ff8000000000000LL);
    for (int q = 0; q < R.n_times; ++q) {
        const double t = A.times[R.t_at + q];
        for (; has_state && c < kn && K[c * 7] <= t; ++c) {   // propagate_state, core.cpp:32-39
            const double *r = K + c * 7;
            const double dt = r[0] - ct;
            const double d[3] = {r[4] - ba[0], r[5] - ba[1], r[6] - ba[2]};
            double ra[3];
            bw_qrot(cq, d, ra);
            const double acc[3] = {0.0 + ra[0], 0.0 + ra[1], -kGravityNominal + ra[2]};
            const double hdt = 0.5 * dt * dt;
            if (has_cov && lane == 0) {                  // the step's blocks, at the old rotation
                double H[9], Jr[9], X[9];
                const double u[3] = {(r[1] - bg[0]) * dt, (r[2] - bg[1]) * dt, (r[3] - bg[2]) * dt};
                quat_to_mat(cq, Rv);
                hat(d, H);
                mat3_mul(Rv, H, Mv);
                double e[4], Em[9];
                expmap(u, e);
                quat_to_mat(e, Em);
                for (int a = 0; a < 3; ++a)
                    for (int b = 0; b < 3; ++b) Et[3 * a + b] = Em[3 * b + a];
                right_jacobian(u, Jr);
                for (int j = 0; j < 9; ++j) Jv[j] = dt * Jr[j];
                const double inv_dt = 1.0 / fmax(dt, 1.0e-7);
                mat3_mul(Jv, seed + 225, X);             // dt Jr cov_w (dt Jr)^T / max(dt, 1e-7)
                for (int a = 0; a < 3; ++a)
                    for (int b = 0; b < 3; ++b)
                        Nw[3 * a + b] = (X[3 * a] * Jv[3 * b] + X[3 * a + 1] * Jv[3 * b + 1] + X[3 * a + 2] * Jv[3 * b + 2]) * inv_dt;
                mat3_mul(Rv, seed + 234, X);             // R cov_a R^T / max(dt, 1e-7)
                for (int a = 0; a < 3; ++a)
                    for (int b = 0; b < 3; ++b)
                        Na[3 * a + b] = (X[3 * a] * Rv[3 * b] + X[3 * a + 1] * Rv[3 * b + 1] + X[3 * a + 2] * Rv[3 * b + 2]) * inv_dt;
                V[54] = dt;
            }
            for (int j = 0; j < 3; ++j) {
                cp[j] = cp[j] + dt * cv[j] + hdt * acc[j];
                cv[j] = cv[j] + dt * acc[j];
            }
            const double u[3] = {(r[1] - bg[0]) * dt, (r[2] - bg[1]) * dt, (r[3] - bg[2]) * dt};
            double e[4], qn[4];
            expmap(u, e);
            eigen_qmul(cq, e, qn);
            const double nrm = sqrt(qn[0] * qn[0] + qn[1] * qn[1] + qn[2] * qn[2] + qn[3] * qn[3]);
            for (int j = 0; j < 4; ++j) cq[j] = qn[j] / nrm;
            ct = r[0];
            if (!has_cov) continue;
            __syncwarp();
            for (int pass = 0; pass < 2; ++pass) {       // Y = F P (columns of P), then P = F Y^T (rows of Y)
                const double *src = pass ? Y : P;
                double *dst = pass ? P : Y;
                if (lane < 15) {
                    const int so = pass ? 15 * lane : lane, ss = pass ? 1 : 15;    // the vector's start and stride
                    double x[15];
                    for (int j = 0; j < 15; ++j) x[j] = src[so + ss * j];
                    const double h2 = 0.5 * V[54] * V[54], t1 = V[54];
                    double o[9];
                    for (int a = 0; a < 3; ++a) {
                        double th = Et[3 * a] * x[0] + Et[3 * a + 1] * x[1] + Et[3 * a + 2] * x[2];
                        th = th - (Jv[3 * a] * x[9] + Jv[3 * a + 1] * x[10] + Jv[3 * a + 2] * x[11]);
                        const double mt = Mv[3 * a] * x[0] + Mv[3 * a + 1] * x[1] + Mv[3 * a + 2] * x[2];
                        const double rb = Rv[3 * a] * x[12] + Rv[3 * a + 1] * x[13] + Rv[3 * a + 2] * x[14];
                        o[a] = th;
                        o[3 + a] = x[3 + a] - h2 * mt + t1 * x[6 + a] - h2 * rb;
                        o[6 + a] = x[6 + a] - t1 * mt - t1 * rb;
                    }
                    const int dso = lane, dss = 15;      // written as column `lane`
                    for (int j = 0; j < 9; ++j) dst[dso + dss * j] = o[j];
                    for (int j = 9; j < 15; ++j) dst[dso + dss * j] = x[j];
                }
                __syncwarp();
            }
            for (int e = lane; e < 225; e += 32) {       // symmetrise and add the noise, each pair by one lane
                const int a = e / 15, b = e % 15;
                if (a > b) continue;
                const int ba_ = a / 3, bb = b / 3, k3 = 3 * (a % 3) + b % 3;
                const double dt = V[54];
                double nz = 0.0;
                if (ba_ == 0 && bb == 0) nz = Nw[k3];
                else if (ba_ == 1 && bb == 1) nz = 0.25 * dt * dt * dt * dt * Na[k3];
                else if (ba_ == 1 && bb == 2) nz = 0.5 * dt * dt * dt * Na[k3];
                else if (ba_ == 2 && bb == 2) nz = dt * dt * Na[k3];
                else if (ba_ == 3 && bb == 3) nz = V[73 + k3] * dt;
                else if (ba_ == 4 && bb == 4) nz = V[82 + k3] * dt;
                const double v = 0.5 * (P[a * 15 + b] + P[b * 15 + a]) + nz;
                P[a * 15 + b] = v;
                P[b * 15 + a] = v;
            }
            __syncwarp();
        }
        // outputs at t
        if (lane == 0) {
            double *o = A.poses + (R.pose_at + q) * 7;
            if (!has_state) {
                for (int j = 0; j < 7; ++j) o[j] = 0.0;
            } else {
                double qo[4], rp[3];
                eigen_qmul(cq, S.q_ob, qo);              // :158-159
                bw_qrot(cq, S.p_ob, rp);
                for (int j = 0; j < 4; ++j) o[j] = qo[j];
                for (int j = 0; j < 3; ++j) o[4 + j] = cp[j] + rp[j];
            }
            if (R.state_at >= 0) {
                double *st = A.states + (R.state_at + q) * 16;
                for (int j = 0; j < 4; ++j) st[j] = has_state ? cq[j] : 0.0;
                for (int j = 0; j < 3; ++j) {
                    st[4 + j] = has_state ? cp[j] : 0.0;
                    st[7 + j] = has_state ? cv[j] : 0.0;
                    st[10 + j] = has_state ? bg[j] : 0.0;
                    st[13 + j] = has_state ? ba[j] : 0.0;
                }
            }
            if (has_cov && R.pcov_at >= 0) {             // R hat(p_ob)
                double Rc[9], H[9];
                quat_to_mat(cq, Rc);
                hat(S.p_ob, H);
                mat3_mul(Rc, H, Kp);
            }
        }
        if (R.scov_at >= 0) {
            double *o = A.scov + (R.scov_at + q) * 225;
            for (int e = lane; e < 225; e += 32) o[e] = has_cov ? P[e] : nan;
        }
        if (R.pcov_at >= 0) {
            double *o = A.pcov + (R.pcov_at + q) * 36;
            if (has_cov) {
                __syncwarp();
                // J = [[R_ob^T, 0], [-R hat(p_ob), I]] over [dtheta dp]; Y <- J P[0:6, 0:6] J^T, then exactly symmetric
                for (int e = lane; e < 36; e += 32) {
                    const int a = e / 6, b = e % 6;
                    double ja[6], jb[6];
                    for (int m = 0; m < 3; ++m) {
                        ja[m] = a < 3 ? Rob[3 * m + a] : -Kp[3 * (a - 3) + m];
                        ja[3 + m] = a < 3 ? 0.0 : (a - 3 == m ? 1.0 : 0.0);
                        jb[m] = b < 3 ? Rob[3 * m + b] : -Kp[3 * (b - 3) + m];
                        jb[3 + m] = b < 3 ? 0.0 : (b - 3 == m ? 1.0 : 0.0);
                    }
                    double s = 0.0;
                    for (int m = 0; m < 6; ++m) {
                        double r = 0.0;
                        for (int k2 = 0; k2 < 6; ++k2) r += P[m * 15 + k2] * jb[k2];
                        s += ja[m] * r;
                    }
                    Y[e] = s;
                }
                __syncwarp();
                for (int e = lane; e < 36; e += 32) o[e] = 0.5 * (Y[e] + Y[(e % 6) * 6 + e / 6]);
                __syncwarp();
            } else {
                for (int e = lane; e < 36; e += 32) o[e] = nan;
            }
        }
    }
}

// why record r cannot seed its slot, or nullptr
const char *seed_check(const ImuStreams &M, const pvio_b200_imu_stream_cov_seed &r) {
    if (!M.host[r.slot].has_state) return "the slot has no latest state";
    if (r.state_time != M.cov_host[r.slot].state_t) return "state_time is not the slot's latest-state time";
    if (r.mode != PVIO_B200_IMU_STREAM_COV_DIRECT && r.mode != PVIO_B200_IMU_STREAM_COV_FACTOR) return "unknown mode";
    const bool factor = r.mode == PVIO_B200_IMU_STREAM_COV_FACTOR;
    if (!r.cov || !r.noise_cov || (factor && !r.imu_record)) return "a missing array";
    if (!std::isfinite(r.state_time) || !finite_all(r.cov, 225) || !finite_all(r.noise_cov, 36) ||
        (factor && !finite_all(r.imu_record, PVIO_B200_IMU_BG0)))
        return "a value that is not finite";
    double big = 0.0;
    for (int e = 0; e < 225; ++e) big = std::max(big, std::fabs(r.cov[e]));
    for (int a = 0; a < 15; ++a) {
        if (r.cov[a * 16] < 0) return "a negative diagonal in cov";
        for (int b = a + 1; b < 15; ++b)
            if (std::fabs(r.cov[a * 15 + b] - r.cov[b * 15 + a]) > 1e-12 * big) return "cov is not symmetric";
    }
    if (factor)
        for (int a = 0; a < 15; ++a)
            if (r.imu_record[PVIO_B200_IMU_SQRT_INV_COV + a * 16] == 0.0) return "a zero diagonal in sqrt_inv_cov";
    return nullptr;
}

int stream_set_covariance_impl(Handle *h, int n, const pvio_b200_imu_stream_cov_seed *recs) {
    if (n < 0 || (n > 0 && !recs)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_set_covariance: bad record list");
    if (n == 0) return 0;
    ImuStreams &M = h->imus;
    std::vector<uint8_t> taken;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_cov_seed &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_imu_stream_set_covariance"));
        if ((size_t)r.slot >= M.host.size() || !M.host[r.slot].set)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_set_covariance: the slot was never reset");
        if (const char *why = seed_check(M, r))
            return fail(h, PVIO_B200_EINVAL, (std::string("batch_imu_stream_set_covariance: ") + why).c_str());
    }
    Stage stage(M.stage);
    const auto rc = stage.add<StreamSeedRec>(Stage::kUp, n);
    TRY(stage.place(h));
    StreamSeedRec *hr = stage.host(rc);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_cov_seed &r = recs[i];
        StreamSeedRec &R = hr[i];
        R.slot = r.slot;
        R.mode = r.mode;
        R.state_t = r.state_time;
        memcpy(R.cov, r.cov, sizeof(R.cov));
        if (r.mode == PVIO_B200_IMU_STREAM_COV_FACTOR) memcpy(R.imu, r.imu_record, sizeof(R.imu));
        else memset(R.imu, 0, sizeof(R.imu));
        memcpy(R.noise, r.noise_cov, sizeof(R.noise));
    }
    cudaStream_t st = h->stream;
    TRY(stage.upload(h));
    imu_stream_seed_kernel<<<(n + kCovWarps - 1) / kCovWarps, 32 * kCovWarps, 0, st>>>(
        n, stage.dev(rc), reinterpret_cast<const ImuStreamSlot *>(M.hdr.d), M.cov.d);
    ++h->launches;
    CK(h, cudaGetLastError());
    CK(h, cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) M.cov_host[recs[i].slot].seed_gen = M.cov_host[recs[i].slot].gen;
    return 0;
}

int stream_predict_impl(Handle *h, int n, pvio_b200_imu_stream_predict *recs) {
    if (n < 0 || (n > 0 && !recs)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_predict: bad record list");
    if (n == 0) return 0;
    ImuStreams &M = h->imus;
    std::vector<uint8_t> taken;
    int64_t nt = 0, ns = 0, npc = 0, nsc = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_predict &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_imu_stream_predict"));
        if ((size_t)r.slot >= M.host.size() || !M.host[r.slot].set)
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_predict: the slot was never reset");
        if (r.n_times < 0 || (r.n_times > 0 && (!r.times || !r.poses)))
            return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_predict: bad time count or pointer");
        if (!finite_all(r.times, r.n_times)) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_predict: a time is not finite");
        for (int k = 1; k < r.n_times; ++k)
            if (r.times[k] < r.times[k - 1]) return fail(h, PVIO_B200_EINVAL, "batch_imu_stream_predict: the times decrease");
        nt += r.n_times;
        ns += r.states ? r.n_times : 0;
        npc += r.pose_cov ? r.n_times : 0;
        nsc += r.state_cov ? r.n_times : 0;
    }
    // staging: records | times (uploaded) || poses | states | pose covariances | state covariances (downloaded)
    Stage stage(M.stage);
    const auto rc = stage.add<StreamPredRec>(Stage::kUp, n);
    const auto tm = stage.add<double>(Stage::kUp, nt);
    const auto po = stage.add<double>(Stage::kDown, 7 * nt);
    const auto sto = stage.add<double>(Stage::kDown, 16 * ns);
    const auto pc = stage.add<double>(Stage::kDown, 36 * npc);
    const auto sc = stage.add<double>(Stage::kDown, 225 * nsc);
    TRY(stage.place(h));
    StreamPredRec *hr = stage.host(rc);
    std::vector<int32_t> status(n);
    int64_t at = 0, as = 0, apc = 0, asc = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_imu_stream_predict &r = recs[i];
        const ImuStreamCovHost &C = M.cov_host[r.slot];
        const bool has_state = M.host[r.slot].has_state, has_cov = has_state && C.seed_gen == C.gen;
        status[i] = !has_state ? PVIO_B200_IMU_STREAM_NO_STATE : has_cov ? PVIO_B200_OK : PVIO_B200_IMU_STREAM_NO_COVARIANCE;
        StreamPredRec R{};
        R.slot = r.slot; R.n_times = r.n_times; R.has_cov = has_cov;
        R.t_at = at; R.pose_at = at;
        R.state_at = r.states ? as : -1;
        R.pcov_at = r.pose_cov ? apc : -1;
        R.scov_at = r.state_cov ? asc : -1;
        hr[i] = R;
        if (r.n_times) memcpy(stage.host(tm) + at, r.times, sizeof(double) * r.n_times);
        at += r.n_times;
        as += r.states ? r.n_times : 0;
        apc += r.pose_cov ? r.n_times : 0;
        asc += r.state_cov ? r.n_times : 0;
    }
    StreamPredArgs A;
    A.hdr = reinterpret_cast<const ImuStreamSlot *>(M.hdr.d);
    A.k = M.k.d; A.cov = M.cov.d; A.qcap = M.qcap;
    A.recs = stage.dev(rc); A.times = stage.dev(tm);
    A.poses = stage.dev(po); A.states = stage.dev(sto); A.pcov = stage.dev(pc); A.scov = stage.dev(sc);
    A.n = n;
    cudaStream_t st = h->stream;
    TRY(stage.upload(h));
    imu_stream_predict_kernel<<<(n + kCovWarps - 1) / kCovWarps, 32 * kCovWarps, 0, st>>>(A);
    ++h->launches;
    CK(h, cudaGetLastError());
    TRY(stage.download(h));
    CK(h, cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i) {
        pvio_b200_imu_stream_predict &r = recs[i];
        const StreamPredRec &R = hr[i];
        const size_t k = r.n_times;
        if (k) memcpy(r.poses, stage.host(po) + 7 * R.pose_at, sizeof(double) * 7 * k);
        if (k && r.states) memcpy(r.states, stage.host(sto) + 16 * R.state_at, sizeof(double) * 16 * k);
        if (k && r.pose_cov) memcpy(r.pose_cov, stage.host(pc) + 36 * R.pcov_at, sizeof(double) * 36 * k);
        if (k && r.state_cov) memcpy(r.state_cov, stage.host(sc) + 225 * R.scov_at, sizeof(double) * 225 * k);
        r.status = status[i];
    }
    return 0;
}
}  // namespace

}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_batch_imu_stream_reset(pvio_b200_handle hh, int n, const int32_t *slots, const double *output_q,
                                                const double *output_p) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_reset_impl(h, n, slots, output_q, output_p);
}

extern "C" int pvio_b200_batch_imu_stream(pvio_b200_handle hh, int n, pvio_b200_imu_stream_record *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_impl(h, n, records);
}

extern "C" int pvio_b200_batch_imu_stream_save(pvio_b200_handle hh, int n, pvio_b200_imu_stream_snapshot *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_save_impl(h, n, records);
}

extern "C" int pvio_b200_batch_imu_stream_restore(pvio_b200_handle hh, int n, const pvio_b200_imu_stream_snapshot *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_restore_impl(h, n, records);
}

extern "C" int pvio_b200_batch_imu_stream_set_covariance(pvio_b200_handle hh, int n,
                                                         const pvio_b200_imu_stream_cov_seed *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_set_covariance_impl(h, n, records);
}

extern "C" int pvio_b200_batch_imu_stream_predict(pvio_b200_handle hh, int n, pvio_b200_imu_stream_predict *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return stream_predict_impl(h, n, records);
}
