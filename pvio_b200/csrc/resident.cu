// Resident sliding window (SURVEY 8(f) rank 1): the window persists in the handle between keyframes instead of
// being rebuilt from Map / Frame / Track at every BundleAdjustor::solve (bundle_adjustor.cpp:75-242).  The shim tells
// the handle what CHANGED -- a frame appended (sliding_window_tracker.cpp:113-118), tracks created / extended
// (frame.cpp:108-139), the oldest frame dropped (map.cpp:76-88) -- and the handle keeps
//   * the frame states, IMU factors and tracks (observation lists, anchors, inverse depths) as plain arrays,
//   * the marginalisation prior ON THE DEVICE: pvio_b200_window_drop_victim runs the marginaliser
//     (bundle_adjustor.cpp:348-599) and leaves S, e and the linearisation point in the prior arrays the solve kernels
//     read; S (120 x 120 doubles for N = 9) never crosses PCIe again.
// Track bookkeeping on the host side of the handle follows map.cpp:76-88 / track.cpp:42-49: when the victim leaves, its
// observations are removed, a track anchored in it is re-anchored in its next frame with the inverse depth
// re-expressed from the CURRENT estimate (quirk Q5).  A track takes part in a solve once it has two observations in
// the window.
#include <array>
#include <cmath>
#include <cstring>
#include <vector>

#include "api_internal.h"

namespace pvio {
namespace {

// quaternions (x, y, z, w), Hamilton product, q * v = rotate: the reference's Eigen conventions (estimation/state.h)
void qmul(const double *a, const double *b, double *o) {
    o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
    o[1] = a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0];
    o[2] = a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3];
    o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}
void qrot(const double *q, const double *v, double *o) {
    const double x = q[0], y = q[1], z = q[2], w = q[3];
    const double tx = 2.0 * (y * v[2] - z * v[1]), ty = 2.0 * (z * v[0] - x * v[2]), tz = 2.0 * (x * v[1] - y * v[0]);
    o[0] = v[0] + w * tx + (y * tz - z * ty);
    o[1] = v[1] + w * ty + (z * tx - x * tz);
    o[2] = v[2] + w * tz + (x * ty - y * tx);
}
void cam_pose(const ResidentWindow &r, int f, double *qc, double *pc) {       // body pose -> camera pose
    const double *fs = r.frames[f].data();
    qmul(fs, r.cst.cam_q_cs, qc);
    double t[3];
    qrot(fs, r.cst.cam_p_cs, t);
    for (int i = 0; i < 3; ++i) pc[i] = fs[4 + i] + t[i];
}

// Track::remove_keypoint with the anchor leaving (track.cpp:42-49): rho re-expressed in frame `to` from the current estimate
void reanchor(const ResidentWindow &r, ResTrack &t, int from_pos, int to_pos) {
    double qa[4], pa[3], qn[4], pn[3];
    cam_pose(r, t.frames[from_pos], qa, pa);
    cam_pose(r, t.frames[to_pos], qn, pn);
    const double ray[3] = {t.z[2 * from_pos] / t.rho, t.z[2 * from_pos + 1] / t.rho, 1.0 / t.rho};
    double x[3], d[3], y[3];
    qrot(qa, ray, x);
    for (int i = 0; i < 3; ++i) d[i] = x[i] + pa[i] - pn[i];
    const double qc[4] = {-qn[0], -qn[1], -qn[2], qn[3]};
    qrot(qc, d, y);
    t.rho = 1.0 / y[2];
}

// landmark-major view over the tracks with >= 2 observations, in track-id order
void build_view(ResidentWindow &r, pvio_b200_window &w, pvio_b200_state &s) {
    const int N = (int)r.frames.size();
    r.lm_anchor.clear(); r.lm_obs_begin.assign(1, 0); r.obs_frame.clear(); r.lm_z_ref.clear(); r.obs_z.clear();
    r.lm_in_victim.clear(); r.lm_track.clear(); r.st_rho.clear();
    for (size_t id = 0; id < r.tracks.size(); ++id) {
        const ResTrack &t = r.tracks[id];
        if (!t.alive || t.frames.size() < 2) continue;
        r.lm_track.push_back((int32_t)id);
        r.lm_anchor.push_back(t.frames[0]);
        r.lm_z_ref.push_back(t.z[0]); r.lm_z_ref.push_back(t.z[1]);
        for (size_t k = 1; k < t.frames.size(); ++k) {
            r.obs_frame.push_back(t.frames[k]);
            r.obs_z.push_back(t.z[2 * k]); r.obs_z.push_back(t.z[2 * k + 1]);
        }
        r.lm_obs_begin.push_back((int32_t)r.obs_frame.size());
        r.lm_in_victim.push_back(t.frames[0] == 0 ? 1 : 0);       // anchor = lowest frame: seen by frame 0 <=> anchored there
        r.st_rho.push_back(t.rho);
    }
    r.st_frames.resize((size_t)N * kFrameStride);
    for (int f = 0; f < N; ++f) memcpy(&r.st_frames[(size_t)f * kFrameStride], r.frames[f].data(), sizeof(double) * kFrameStride);
    const int n_imu = r.cst.use_inertial ? (int)r.imu.size() : 0;
    r.imu_i.resize(n_imu); r.imu_j.resize(n_imu); r.imu_data.resize((size_t)n_imu * kImuStride);
    for (int k = 0; k < n_imu; ++k) {
        r.imu_i[k] = k; r.imu_j[k] = k + 1;
        memcpy(&r.imu_data[(size_t)k * kImuStride], r.imu[k].data(), sizeof(double) * kImuStride);
    }
    r.prior_frames.resize(r.n_prior);
    for (int k = 0; k < r.n_prior; ++k) r.prior_frames[k] = k;
    w = r.cst;
    w.n_frames = N; w.n_landmarks = (int)r.lm_anchor.size(); w.n_obs = (int)r.obs_frame.size();
    w.frame_fixed = r.fixed.data();
    w.lm_anchor = r.lm_anchor.data(); w.lm_z_ref = r.lm_z_ref.data(); w.lm_obs_begin = r.lm_obs_begin.data();
    w.lm_in_victim = r.lm_in_victim.data(); w.obs_frame = r.obs_frame.data(); w.obs_z = r.obs_z.data();
    w.n_imu = n_imu; w.imu_frame_i = r.imu_i.data(); w.imu_frame_j = r.imu_j.data(); w.imu_data = r.imu_data.data();
    w.n_prior = r.n_prior; w.prior_frames = r.prior_frames.data();
    if (r.prior_on_device || r.n_prior == 0) { w.prior_S = nullptr; w.prior_e = nullptr; w.prior_state0 = nullptr; }
    else { w.prior_S = r.host_S.data(); w.prior_e = r.host_e.data(); w.prior_state0 = r.host_x0.data(); }
    w.n_planes = 0; w.plane_param = nullptr; w.n_plane_tracks = 0;
    w.pt_plane = nullptr; w.pt_obs_begin = nullptr; w.pt_obs_frame = nullptr; w.pt_obs_z = nullptr;
    s.frames = r.st_frames.data(); s.inv_depth = r.st_rho.data();
}

ResidentWindow *get(Handle *h) {
    if (!h->resident) fail(h, PVIO_B200_EINVAL, "no resident window: call pvio_b200_window_reset first");
    return h->resident.get();
}

}  // namespace
}  // namespace pvio

using namespace pvio;

extern "C" {

int pvio_b200_window_reset(pvio_b200_handle hh, const pvio_b200_window *constants) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !constants) return PVIO_B200_EINVAL;
    h->resident = std::make_unique<ResidentWindow>();
    h->resident->cst = *constants;
    h->prior_resident[0] = 0;
    return 0;
}

int pvio_b200_window_append_frame(pvio_b200_handle hh, const double *state, int fixed, const double *imu_record) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || !state) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    if ((int)r->frames.size() >= h->Ncap) return fail(h, PVIO_B200_EINVAL, "window full: drop the victim first");
    if (r->cst.use_inertial && !r->frames.empty() && !imu_record) return fail(h, PVIO_B200_EINVAL, "an inertial window needs the IMU factor to the previous frame");
    std::array<double, kFrameStride> f;
    memcpy(f.data(), state, sizeof(double) * kFrameStride);
    if (r->cst.use_inertial && !r->frames.empty()) {
        std::array<double, kImuStride> rec;
        memcpy(rec.data(), imu_record, sizeof(double) * kImuStride);
        r->imu.push_back(rec);
    }
    r->frames.push_back(f);
    r->fixed.push_back(fixed ? 1 : 0);
    return 0;
}

int pvio_b200_window_add_tracks(pvio_b200_handle hh, int n, const int32_t *frame, const double *z, const double *inv_depth, int32_t *ids_out) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || n < 0 || (n > 0 && (!frame || !z || !inv_depth))) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    for (int i = 0; i < n; ++i) {
        if (frame[i] < 0 || frame[i] >= (int)r->frames.size()) return fail(h, PVIO_B200_EINVAL, "track starts outside the window");
        ResTrack t;
        t.frames.push_back(frame[i]);
        t.z.push_back(z[2 * i]); t.z.push_back(z[2 * i + 1]);
        t.rho = inv_depth[i];
        if (ids_out) ids_out[i] = (int32_t)r->tracks.size();
        r->tracks.push_back(std::move(t));
    }
    return 0;
}

int pvio_b200_window_add_observations(pvio_b200_handle hh, int n, const int32_t *track, const int32_t *frame, const double *z) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || n < 0 || (n > 0 && (!track || !frame || !z))) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    for (int i = 0; i < n; ++i) {
        if (track[i] < 0 || track[i] >= (int)r->tracks.size() || !r->tracks[track[i]].alive) return fail(h, PVIO_B200_EINVAL, "unknown track");
        ResTrack &t = r->tracks[track[i]];
        if (frame[i] < 0 || frame[i] >= (int)r->frames.size() || frame[i] <= t.frames.back())
            return fail(h, PVIO_B200_EINVAL, "observations of a track arrive in increasing frame order");
        t.frames.push_back(frame[i]);
        t.z.push_back(z[2 * i]); t.z.push_back(z[2 * i + 1]);
    }
    return 0;
}

int pvio_b200_window_remove_track(pvio_b200_handle hh, int32_t track) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    if (track < 0 || track >= (int)r->tracks.size()) return fail(h, PVIO_B200_EINVAL, "unknown track");
    r->tracks[track].alive = false;
    return 0;
}

int pvio_b200_window_set_prior(pvio_b200_handle hh, int n_prior, const double *S, const double *e, const double *state0) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h || n_prior < 0 || (n_prior > 0 && (!S || !e || !state0))) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    if (n_prior > (int)r->frames.size()) return fail(h, PVIO_B200_EINVAL, "prior over more frames than the window holds");
    const size_t d = 15 * (size_t)n_prior;
    r->n_prior = n_prior; r->prior_on_device = false;
    r->host_S.assign(S, S + d * d); r->host_e.assign(e, e + d); r->host_x0.assign(state0, state0 + (size_t)n_prior * kFrameStride);
    return 0;
}

int pvio_b200_window_solve(pvio_b200_handle hh, const pvio_b200_options *opt, pvio_b200_summary *summary) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    pvio_b200_window w;
    pvio_b200_state s;
    build_view(*r, w, s);
    const int rc = pvio_b200_ba_solve(hh, &w, &s, opt, summary, nullptr, nullptr);
    if (rc != 0) return rc;
    for (size_t f = 0; f < r->frames.size(); ++f) memcpy(r->frames[f].data(), &r->st_frames[f * kFrameStride], sizeof(double) * kFrameStride);
    for (size_t i = 0; i < r->lm_track.size(); ++i) r->tracks[r->lm_track[i]].rho = r->st_rho[i];
    return 0;
}

int pvio_b200_window_drop_victim(pvio_b200_handle hh) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    const int N = (int)r->frames.size();
    if (N < 2) return fail(h, PVIO_B200_EINVAL, "nothing to marginalise");
    pvio_b200_window w;
    pvio_b200_state s;
    build_view(*r, w, s);
    const int rc = marginalize_impl(h, &w, &s, 0, true, nullptr, nullptr, nullptr, nullptr);
    if (rc != 0) return rc;
    r->n_prior = N - 1; r->prior_on_device = true;
    r->host_S.clear(); r->host_e.clear(); r->host_x0.clear();
    // map.cpp:76-88: the victim's keypoints leave their tracks
    for (ResTrack &t : r->tracks) {
        if (!t.alive) continue;
        if (!t.frames.empty() && t.frames[0] == 0) {
            if (t.frames.size() >= 2) reanchor(*r, t, 0, 1);
            t.frames.erase(t.frames.begin());
            t.z.erase(t.z.begin(), t.z.begin() + 2);
        }
        if (t.frames.empty()) { t.alive = false; continue; }
        for (int32_t &f : t.frames) --f;
    }
    r->frames.erase(r->frames.begin());
    r->fixed.erase(r->fixed.begin());
    if (!r->imu.empty()) r->imu.erase(r->imu.begin());
    return 0;
}

int pvio_b200_window_get(pvio_b200_handle hh, int32_t *n_frames, double *frames, int n_tracks, const int32_t *tracks,
                         double *inv_depth, int32_t *anchor_frame, int32_t *n_observations) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    ResidentWindow *r = get(h);
    if (!r) return PVIO_B200_EINVAL;
    if (n_frames) *n_frames = (int32_t)r->frames.size();
    if (frames) for (size_t f = 0; f < r->frames.size(); ++f) memcpy(frames + f * kFrameStride, r->frames[f].data(), sizeof(double) * kFrameStride);
    for (int i = 0; i < n_tracks; ++i) {
        if (tracks[i] < 0 || tracks[i] >= (int)r->tracks.size()) return fail(h, PVIO_B200_EINVAL, "unknown track");
        const ResTrack &t = r->tracks[tracks[i]];
        if (inv_depth) inv_depth[i] = t.rho;
        if (anchor_frame) anchor_frame[i] = (t.alive && !t.frames.empty()) ? t.frames[0] : -1;
        if (n_observations) n_observations[i] = t.alive ? (int32_t)t.frames.size() : 0;
    }
    return 0;
}

}  // extern "C"
