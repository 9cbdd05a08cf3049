// Lens distortion removal with OpenCV's arithmetic: replaces the cv::undistort call of EurocDatasetReader::read_image
// (pvio-pc/src/euroc_dataset_reader.cpp:70-74, also OpenCvImage::correct_distortion, opencv_image.cpp:162-175) and the
// remap of ImageUndistorter (pvio-extra/include/pvio/extra/image_undistorter.h:28-95, used by tum_dataset_reader.cpp:71-81).
//
//   undistort_map_host  the map of one lens, on the host in fp64 (once per sequence): OpenCV's CV_16SC2 pair, m1 the
//                       integer source pixel, m2 the 1/32-pixel fraction as the table index (iv & 31) * 32 + (iu & 31)
//   undistort_kernel    cv::remap(INTER_LINEAR, BORDER_CONSTANT 0) of 8-bit frames through such a map, one thread per
//                       pixel, every uploaded frame of a call in one launch (grid z = frame); integer arithmetic only
//
// The map arithmetic is restated in oracle/undistort_oracle.py, which is pinned bit for bit against cv2.  This file's
// host code is compiled with -ffp-contract=off: a fused multiply-add would change map entries.
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>
#include "api_internal.h"

namespace pvio {
namespace {

constexpr int kMaxMapSide = 32767;            // cv::remap's limit (SHRT_MAX): the map holds int16 source pixels

// cvRound / saturate_cast<int>: nearest, ties to even, saturated
inline int cv_round(double v) {
    const double r = std::nearbyint(v);
    return r >= (double)INT_MAX ? INT_MAX : r <= (double)INT_MIN ? INT_MIN : (int)r;
}

inline short sat_short(int v) { return (short)std::min(std::max(v, -32768), 32767); }

// cv::invert / Matx33d::inv with DECOMP_LU of a 3x3 double matrix: OpenCV's closed form for n == 3
void inv3(const double a[3][3], double t[9]) {
    double d = a[0][0] * (a[1][1] * a[2][2] - a[1][2] * a[2][1]) - a[0][1] * (a[1][0] * a[2][2] - a[1][2] * a[2][0]) +
               a[0][2] * (a[1][0] * a[2][1] - a[1][1] * a[2][0]);
    d = 1. / d;
    t[0] = (a[1][1] * a[2][2] - a[1][2] * a[2][1]) * d;
    t[1] = (a[0][2] * a[2][1] - a[0][1] * a[2][2]) * d;
    t[2] = (a[0][1] * a[1][2] - a[0][2] * a[1][1]) * d;
    t[3] = (a[1][2] * a[2][0] - a[1][0] * a[2][2]) * d;
    t[4] = (a[0][0] * a[2][2] - a[0][2] * a[2][0]) * d;
    t[5] = (a[0][2] * a[1][0] - a[0][0] * a[1][2]) * d;
    t[6] = (a[1][0] * a[2][1] - a[1][1] * a[2][0]) * d;
    t[7] = (a[0][1] * a[2][0] - a[0][0] * a[2][1]) * d;
    t[8] = (a[0][0] * a[1][1] - a[0][1] * a[1][0]) * d;
}

// cv::undistort(src, dst, K, D) with K, D as cv::Mat_<float>: the parameters rounded to float32; stripes of
// min(max(1, 4096 / width), height) rows, each built by initUndistortRectifyMap (R = I, new camera matrix Ar = K with
// Ar(1, 2) = cy - y0) and its scalar loop in its order; k3..k6, s1..s4 and tau are zero (matTilt = I, invProj = 1).
// false when a coordinate is not finite
bool radtan_map(int width, int height, const double *p, const double *c, int16_t *m1, uint16_t *m2) {
    const double fx = (float)p[0], fy = (float)p[1], u0 = (float)p[2], v0 = (float)p[3];
    const double k1 = (float)c[0], k2 = (float)c[1], p1 = (float)c[2], p2 = (float)c[3];
    const double k3 = 0, k4 = 0, k5 = 0, k6 = 0, s1 = 0, s2 = 0, s3 = 0, s4 = 0;
    const int stripe = std::min(std::max(1, 4096 / width), height);
    for (int y0 = 0; y0 < height; y0 += stripe) {
        const int rows = std::min(stripe, height - y0);
        const double Ar[3][3] = {{fx, 0, u0}, {0, fy, v0 - y0}, {0, 0, 1}};
        double ir[9];
        inv3(Ar, ir);
        for (int i = 0; i < rows; ++i) {
            double _x = i * ir[1] + ir[2], _y = i * ir[4] + ir[5], _w = i * ir[7] + ir[8];
            const size_t row = (size_t)(y0 + i) * width;
            for (int j = 0; j < width; ++j, _x += ir[0], _y += ir[3], _w += ir[6]) {
                const double w = 1. / _w, x = _x * w, y = _y * w;
                const double x2 = x * x, y2 = y * y;
                const double r2 = x2 + y2, _2xy = 2 * x * y;
                const double kr = (1 + ((k3 * r2 + k2) * r2 + k1) * r2) / (1 + ((k6 * r2 + k5) * r2 + k4) * r2);
                const double xd = x * kr + p1 * _2xy + p2 * (r2 + 2 * x2) + s1 * r2 + s2 * r2 * r2;
                const double yd = y * kr + p1 * (r2 + 2 * y2) + p2 * _2xy + s3 * r2 + s4 * r2 * r2;
                const double u = fx * 1.0 * xd + u0, v = fy * 1.0 * yd + v0;
                if (!std::isfinite(u) || !std::isfinite(v)) return false;
                const int iu = cv_round(u * 32), iv = cv_round(v * 32);
                m1[2 * (row + j)] = (short)(iu >> 5);
                m1[2 * (row + j) + 1] = (short)(iv >> 5);
                m2[row + j] = (uint16_t)((iv & 31) * 32 + (iu & 31));
            }
        }
    }
    return true;
}

// ImageUndistorter: distort_pixel in double for every pixel (K.inverse() as Eigen's 3x3 cofactor inverse, cofactors
// times 1 / det), the float maps, then cv::convertMaps(CV_32FC1 -> CV_16SC2): cvRound(f * 32) in float,
// saturate_cast<short>.  K's zeros make the summation orders of det, both matrix-vector products and hnormalized
// immaterial.  false when a coordinate is not finite
bool equidistant_map(int width, int height, const double *p, const double *c, int16_t *m1, uint16_t *m2) {
    const double fx = p[0], fy = p[1], cx = p[2], cy = p[3];
    const double k1 = c[0], k2 = c[1], k3 = c[2], k4 = c[3];
    const double m[3][3] = {{fx, 0, cx}, {0, fy, cy}, {0, 0, 1}};
    auto cof = [&](int i, int j) {
        const int i1 = (i + 1) % 3, i2 = (i + 2) % 3, j1 = (j + 1) % 3, j2 = (j + 2) % 3;
        return m[i1][j1] * m[i2][j2] - m[i1][j2] * m[i2][j1];
    };
    const double det = cof(0, 0) * m[0][0] + cof(1, 0) * m[1][0] + cof(2, 0) * m[2][0];
    const double invdet = 1.0 / det;
    double ki[3][3];
    for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q) ki[r][q] = cof(q, r) * invdet;
    for (int v = 0; v < height; ++v)
        for (int u = 0; u < width; ++u) {
            const double x = ki[0][0] * u + ki[0][1] * v + ki[0][2] * 1.0;
            const double y = ki[1][0] * u + ki[1][1] * v + ki[1][2] * 1.0;
            const double z = ki[2][0] * u + ki[2][1] * v + ki[2][2] * 1.0;
            double mx = u, my = v;
            const double r = std::sqrt(x * x + y * y);
            if (!(r < 1e-10)) {
                const double theta = std::atan(r);
                const double theta2 = theta * theta, theta4 = theta2 * theta2, theta6 = theta2 * theta4, theta8 = theta4 * theta4;
                const double thetad = theta * (1 + k1 * theta2 + k2 * theta4 + k3 * theta6 + k4 * theta8);
                const double scaling = (r > 1e-8) ? thetad / r : 1.0;
                const double xd = x * scaling, yd = y * scaling;
                const double px = fx * xd + 0.0 * yd + cx * z, py = 0.0 * xd + fy * yd + cy * z, pz = 0.0 * xd + 0.0 * yd + 1.0 * z;
                mx = px / pz; my = py / pz;
            }
            const float fu = (float)mx, fv = (float)my;
            if (!std::isfinite(fu) || !std::isfinite(fv)) return false;
            const int iu = cv_round(std::nearbyint(fu * 32.0f)), iv = cv_round(std::nearbyint(fv * 32.0f));
            const size_t i = (size_t)v * width + u;
            m1[2 * i] = sat_short(iu >> 5);
            m1[2 * i + 1] = sat_short(iv >> 5);
            m2[i] = (uint16_t)((iv & 31) * 32 + (iu & 31));
        }
    return true;
}

// One thread per pixel of frames[blockIdx.z]: the four taps around m1 (0 outside the frame), weighted by the fraction
// of m2 in 1/32 pixel; the sum of the products is exact in int, rounded as cv::remap's 8-bit path rounds it.
__global__ void undistort_kernel(const KltBatchFrame *frames) {
    const KltBatchFrame &f = frames[blockIdx.z];
    const int w = f.w[0], h = f.h[0];
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const size_t i = (size_t)y * w + x;
    const short2 s = f.m1[i];
    const int a = f.m2[i], fx = a & 31, fy = a >> 5;
    const uint8_t *src = f.lens_src;
    auto tap = [&](int xx, int yy) -> int {
        return (unsigned)xx < (unsigned)w && (unsigned)yy < (unsigned)h ? (int)src[(size_t)yy * w + xx] : 0;
    };
    const int sum = tap(s.x, s.y) * ((32 - fx) * (32 - fy)) + tap(s.x + 1, s.y) * (fx * (32 - fy)) +
                    tap(s.x, s.y + 1) * ((32 - fx) * fy) + tap(s.x + 1, s.y + 1) * (fx * fy);
    f.raw[i] = (uint8_t)((sum + 512) >> 10);
}

}  // namespace

int undistort_map_host(int model, int width, int height, const double *p, const double *c, int16_t *m1, uint16_t *m2) {
    if (model != PVIO_B200_LENS_RADTAN && model != PVIO_B200_LENS_EQUIDISTANT) return PVIO_B200_EINVAL;
    if (width < 8 || height < 8 || width > kMaxMapSide || height > kMaxMapSide || !p || !c || !m1 || !m2) return PVIO_B200_EINVAL;
    for (int k = 0; k < 4; ++k)
        if (!std::isfinite(p[k]) || !std::isfinite(c[k])) return PVIO_B200_EINVAL;
    if (!(p[0] > 0) || !(p[1] > 0)) return PVIO_B200_EINVAL;
    const bool ok = model == PVIO_B200_LENS_RADTAN ? radtan_map(width, height, p, c, m1, m2)
                                                   : equidistant_map(width, height, p, c, m1, m2);
    return ok ? 0 : PVIO_B200_EINVAL;
}

const SlotLens *slot_lens(const KltBatchState &B, int slot) {
    return slot >= 0 && (size_t)slot < B.lens.size() && B.lens[slot].model ? &B.lens[slot] : nullptr;
}

void undistort_frames(Handle *h, const KltBatchFrame *frames, int n_frames, int max_w, int max_h) {
    undistort_kernel<<<dim3((max_w + 31) / 32, (max_h + 7) / 8, n_frames), dim3(32, 8), 0, h->stream>>>(frames);
    ++h->launches;
}

// Every record is checked and every map built before a slot changes; then each map is copied into its slot's buffer
// and the slot's cached pyramids are dropped (they were built from frames under the old lens).
int set_lens_impl(Handle *h, int n, const pvio_b200_lens *recs) {
    if (n < 0) return fail(h, PVIO_B200_EINVAL, "batch_set_lens: bad record count");
    if (n == 0) return 0;
    if (!recs) return fail(h, PVIO_B200_EINVAL, "batch_set_lens: bad arguments");
    std::vector<uint8_t> taken;
    std::vector<std::vector<uint8_t>> maps(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_lens &r = recs[i];
        TRY(take_slot(h, taken, r.slot, "batch_set_lens"));
        if (r.model == 0) continue;
        if (r.width < 8 || r.height < 8 || r.width > kMaxMapSide || r.height > kMaxMapSide)
            return fail(h, PVIO_B200_EINVAL, "batch_set_lens: bad frame shape");
        const size_t px = (size_t)r.width * r.height;
        maps[i].resize(6 * px);
        const double p[4] = {r.fx, r.fy, r.cx, r.cy};
        int16_t *m1 = reinterpret_cast<int16_t *>(maps[i].data());
        uint16_t *m2 = reinterpret_cast<uint16_t *>(maps[i].data() + 4 * px);
        if (undistort_map_host(r.model, r.width, r.height, p, r.coeffs, m1, m2))
            return fail(h, PVIO_B200_EINVAL, "batch_set_lens: bad lens (model, parameters, or a map coordinate not finite)");
    }
    KltBatchState &B = h->kltb;
    CK(h, cudaStreamSynchronize(h->stream));          // queued calls may still read a map that is replaced
    if (taken.size() > B.lens.size()) B.lens.resize(taken.size());
    for (int i = 0; i < n; ++i) {
        const pvio_b200_lens &r = recs[i];
        SlotLens &L = B.lens[r.slot];
        L.model = 0;
        if (r.model != 0) {
            TRY(reserve(h, L.map, maps[i].size(), kDevice));
            CK(h, cudaMemcpyAsync(L.map.d, maps[i].data(), maps[i].size(), cudaMemcpyHostToDevice, h->stream));
            L.w = r.width; L.h = r.height; L.model = r.model;
        } else {
            L = SlotLens{};
        }
        if ((size_t)r.slot < B.slots.size()) {
            KltPyramids &s = B.slots[r.slot];
            s.pyr_id[0] = s.pyr_id[1] = 0;
        }
    }
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

// One upload (descriptors and pixels), one launch, one download; no cache is read or changed.
int batch_undistort_impl(Handle *h, int n, const pvio_b200_undistort_request *reqs) {
    if (n < 0 || n > 65535) return fail(h, PVIO_B200_EINVAL, "batch_undistort: bad request count");
    if (n == 0) return 0;
    if (!reqs) return fail(h, PVIO_B200_EINVAL, "batch_undistort: bad arguments");
    KltBatchState &B = h->kltb;
    size_t pix_bytes = 0;
    int max_w = 0, max_h = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_undistort_request &a = reqs[i];
        if (a.slot < 0 || a.slot > kMaxBatchSlot) return fail(h, PVIO_B200_EINVAL, "batch_undistort: slot out of range");
        const SlotLens *L = slot_lens(B, a.slot);
        if (!L) return fail(h, PVIO_B200_EINVAL, "batch_undistort: the slot has no lens");
        if (a.width != L->w || a.height != L->h || a.stride < a.width || !a.src || !a.dst)
            return fail(h, PVIO_B200_EINVAL, "batch_undistort: bad shape, stride or pointer (the shape is the lens's)");
        pix_bytes += align256((size_t)a.width * a.height);
        max_w = std::max(max_w, a.width); max_h = std::max(max_h, a.height);
    }
    // staging: descriptors and raw frames (uploaded) | undistorted frames (downloaded), one 256-byte aligned block per frame
    Stage S(B.ustage);
    const auto frm = S.add<KltBatchFrame>(Stage::kUp, n);
    const auto src = S.add<uint8_t>(Stage::kUp, pix_bytes);
    const auto dst = S.add<uint8_t>(Stage::kDown, pix_bytes);
    TRY(S.place(h));
    size_t pix = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_undistort_request &a = reqs[i];
        const SlotLens &L = *slot_lens(B, a.slot);
        for (int y = 0; y < a.height; ++y)
            memcpy(S.host(src) + pix + (size_t)y * a.width, a.src + (size_t)y * a.stride, a.width);
        KltBatchFrame &F = S.host(frm)[i];
        memset(&F, 0, sizeof(F));
        F.lens_src = S.dev(src) + pix; F.raw = S.dev(dst) + pix; F.m1 = L.m1(); F.m2 = L.m2();
        F.levels = 1; F.w[0] = a.width; F.h[0] = a.height;
        pix += align256((size_t)a.width * a.height);
    }
    cudaStream_t st = h->stream;
    TRY(S.upload(h));
    undistort_frames(h, S.dev(frm), n, max_w, max_h);
    CK(h, cudaGetLastError());
    TRY(S.download(h));
    CK(h, cudaStreamSynchronize(st));
    pix = 0;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_undistort_request &a = reqs[i];
        memcpy(a.dst, S.host(dst) + pix, (size_t)a.width * a.height);
        pix += align256((size_t)a.width * a.height);
    }
    return 0;
}

}  // namespace pvio

using namespace pvio;

extern "C" int pvio_b200_undistort_map(int model, int width, int height, const double *fx_fy_cx_cy, const double *coeffs,
                                       int16_t *m1, uint16_t *m2) {
    return undistort_map_host(model, width, height, fx_fy_cx_cy, coeffs, m1, m2);
}

extern "C" int pvio_b200_batch_set_lens(pvio_b200_handle hh, int n, const pvio_b200_lens *records) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return set_lens_impl(h, n, records);
}

extern "C" int pvio_b200_batch_undistort(pvio_b200_handle hh, int n, const pvio_b200_undistort_request *requests) {
    Handle *h = reinterpret_cast<Handle *>(hh);
    if (!h) return PVIO_B200_EINVAL;
    return batch_undistort_impl(h, n, requests);
}
