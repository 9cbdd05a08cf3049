// Pyramidal Lucas-Kanade on the GPU with OpenCV's arithmetic: replaces the
// cv::calcOpticalFlowPyrLK call of OpenCvImage::track_keypoints
// (pvio-extra/src/pvio/extra/opencv_image.cpp:103; pyramid from preprocess() :145).
//
//   pyrdown_kernel   cv::pyrDown, 5x5 [1 4 6 4 1]/16, BORDER_REFLECT_101, (s + 128) >> 8
//   klt_track_kernel one warp per keypoint, all pyramid levels (coarse to fine) in one launch:
//                    24x24 image patch staged in shared memory, Scharr derivatives (int16, as
//                    calcSharrDeriv) computed from it, 21x21 window with 14-bit fixed-point
//                    bilinear weights, exact int64 warp-shuffle reductions for the 2x2 system,
//                    <= max_iter Newton steps with OpenCV's eps / oscillation stopping rules.
// Compiled with -fmad=false: the float expressions must round like OpenCV's (no contraction),
// because status flags are compared bit-exactly with cv2.
#include <cstring>
#include <vector>
#include "api_internal.h"

namespace pvio {

constexpr int kWin = 21;
constexpr int kWBits = 14;
constexpr int kKltWarps = 4;

// 20-pixel border rejection of OpenCvImage::track_keypoints (opencv_image.cpp:106-108) on the device
__global__ void klt_border_kernel(const float *pts, uint8_t *status, int n, int w, int h, int border) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = pts[2 * i], y = pts[2 * i + 1];
    if (x < (float)border || x >= (float)(w - border) || y < (float)border || y >= (float)(h - border)) status[i] = 0;
}

struct KltLevels {
    const uint8_t *I[kMaxLevels];
    const uint8_t *J[kMaxLevels];
    int w[kMaxLevels], h[kMaxLevels];
    int n;
};

__device__ __forceinline__ int reflect101(int i, int n) {
    i = i < 0 ? -i : i;
    return i >= n ? 2 * (n - 1) - i : i;
}

// ---- CLAHE (cv::createCLAHE(clip, tiles)->apply, opencv_image.cpp:138-143; algorithm: OpenCV imgproc/clahe.cpp,
// restated in oracle/clahe_oracle.py which is pinned bit for bit against cv2).  Image sizes that are multiples
// of the tile grid only.  Kernel 1: one CTA per tile -- histogram in shared memory, clip + redistribute, prefix
// sum, LUT = cvRound(cdf * 255 / area).  Kernel 2: one thread per pixel, bilinear blend of the four neighbouring
// tiles' LUTs in OpenCV's float32 operation order (explicit _rn intrinsics: no FMA contraction).
__global__ void __launch_bounds__(256) clahe_lut_kernel(const uint8_t *src, int w, int tw, int th, int tiles_x,
                                                        int clip, float lut_scale, uint8_t *lut) {
    __shared__ int hist[256];
    __shared__ int wsum[8];
    __shared__ int total_clipped;
    const int t = blockIdx.x, tx = t % tiles_x, ty = t / tiles_x, tid = threadIdx.x;
    hist[tid] = 0;
    __syncthreads();
    const uint8_t *base = src + (size_t)ty * th * w + (size_t)tx * tw;
    for (int i = tid; i < tw * th; i += 256) atomicAdd(&hist[base[(size_t)(i / tw) * w + (i % tw)]], 1);
    __syncthreads();
    int hv = hist[tid];
    int excess = max(hv - clip, 0);
    hv = min(hv, clip);
    int e = excess;
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) e += __shfl_xor_sync(0xffffffffu, e, off);
    if ((tid & 31) == 0) wsum[tid >> 5] = e;
    __syncthreads();
    if (tid == 0) { int s = 0; for (int k = 0; k < 8; ++k) s += wsum[k]; total_clipped = s; }
    __syncthreads();
    const int clipped = total_clipped;
    const int batch = clipped / 256;
    int residual = clipped - batch * 256;
    hv += batch;
    if (residual != 0) {
        const int step = max(256 / residual, 1);
        if (tid % step == 0 && tid / step < residual) hv += 1;       // bins 0, step, 2 step, ... (residual of them)
    }
    // inclusive prefix sum over the 256 bins
    int v = hv;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) { const int n = __shfl_up_sync(0xffffffffu, v, off); if ((tid & 31) >= off) v += n; }
    __syncthreads();
    if ((tid & 31) == 31) wsum[tid >> 5] = v;
    __syncthreads();
    int pre = 0;
    for (int k = 0; k < (tid >> 5); ++k) pre += wsum[k];
    const float f = __fmul_rn((float)(v + pre), lut_scale);
    lut[(size_t)t * 256 + tid] = (uint8_t)min(max(__float2int_rn(f), 0), 255);
}

__global__ void clahe_apply_kernel(const uint8_t *src, int w, int h, int tw, int th, int tiles_x, int tiles_y,
                                   const uint8_t *lut, uint8_t *dst) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= w || y >= h) return;
    const float inv_tw = __fdiv_rn(1.0f, (float)tw), inv_th = __fdiv_rn(1.0f, (float)th);
    const float txf = __fsub_rn(__fmul_rn((float)x, inv_tw), 0.5f), tyf = __fsub_rn(__fmul_rn((float)y, inv_th), 0.5f);
    int tx1 = (int)floorf(txf), ty1 = (int)floorf(tyf);
    const float xa = __fsub_rn(txf, (float)tx1), ya = __fsub_rn(tyf, (float)ty1);
    const float xa1 = __fsub_rn(1.0f, xa), ya1 = __fsub_rn(1.0f, ya);
    const int tx2 = min(tx1 + 1, tiles_x - 1), ty2 = min(ty1 + 1, tiles_y - 1);
    tx1 = max(tx1, 0); ty1 = max(ty1, 0);
    const int v = src[(size_t)y * w + x];
    const float l11 = (float)lut[((size_t)ty1 * tiles_x + tx1) * 256 + v], l12 = (float)lut[((size_t)ty1 * tiles_x + tx2) * 256 + v];
    const float l21 = (float)lut[((size_t)ty2 * tiles_x + tx1) * 256 + v], l22 = (float)lut[((size_t)ty2 * tiles_x + tx2) * 256 + v];
    const float top = __fadd_rn(__fmul_rn(l11, xa1), __fmul_rn(l12, xa));
    const float bot = __fadd_rn(__fmul_rn(l21, xa1), __fmul_rn(l22, xa));
    const float res = __fadd_rn(__fmul_rn(top, ya1), __fmul_rn(bot, ya));
    dst[(size_t)y * w + x] = (uint8_t)min(max(__float2int_rn(res), 0), 255);
}

// device-resident CLAHE of a w x h image (row stride w)
static int clahe_device(Handle *h, const uint8_t *src, uint8_t *dst, uint8_t *lut, int w, int hgt, double clip_limit,
                        int tiles_x, int tiles_y) {
    const int tw = w / tiles_x, th = hgt / tiles_y, area = tw * th;
    const int clip = std::max((int)(clip_limit * area / 256), 1);
    const float lut_scale = 255.0f / (float)area;
    clahe_lut_kernel<<<tiles_x * tiles_y, 256, 0, h->stream>>>(src, w, tw, th, tiles_x, clip, lut_scale, lut);
    dim3 b(32, 8), g((w + 31) / 32, (hgt + 7) / 8);
    clahe_apply_kernel<<<g, b, 0, h->stream>>>(src, w, hgt, tw, th, tiles_x, tiles_y, lut, dst);
    h->launches += 2;
    return 0;
}

__global__ void pyrdown_kernel(const uint8_t *src, int sw, int sh, uint8_t *dst, int dw, int dh) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    if (x >= dw || y >= dh) return;
    const int k[5] = {1, 4, 6, 4, 1};
    int acc = 0;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
        const uint8_t *row = src + (size_t)reflect101(2 * y + dy, sh) * sw;
        int r = 0;
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) r += k[dx + 2] * row[reflect101(2 * x + dx, sw)];
        acc += k[dy + 2] * r;
    }
    dst[(size_t)y * dw + x] = (uint8_t)((acc + 128) >> 8);
}

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

__device__ __forceinline__ void bilinear_weights(float a, float b, int &w00, int &w01, int &w10, int &w11) {
    const float s = (float)(1 << kWBits);
    w00 = __float2int_rn((1.f - a) * (1.f - b) * s);     // cvRound
    w01 = __float2int_rn(a * (1.f - b) * s);
    w10 = __float2int_rn((1.f - a) * b * s);
    w11 = (1 << kWBits) - w00 - w01 - w10;
}

__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

__global__ void __launch_bounds__(32 * kKltWarps)
klt_track_kernel(KltLevels L, const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                 int max_iter, double eps2, float min_eig_thr) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pt = blockIdx.x * kKltWarps + warp;
    __shared__ int Ipatch[kKltWarps][24 * 24];
    __shared__ short Dpatch[kKltWarps][22 * 22 * 2];
    __shared__ short IWin[kKltWarps][kWin * kWin];
    __shared__ short dIWin[kKltWarps][kWin * kWin * 2];
    if (pt >= n_points) return;
    const float px0 = prev_pts[2 * pt], py0 = prev_pts[2 * pt + 1];
    float nx = next_pts[2 * pt], ny = next_pts[2 * pt + 1];      // OPTFLOW_USE_INITIAL_FLOW
    bool st = true;
    float err_out = 0.f;
    const float half = (kWin - 1) * 0.5f;
    int *Ip = Ipatch[warp];
    short *Dp = Dpatch[warp], *Iw = IWin[warp], *dIw = dIWin[warp];

    for (int level = L.n - 1; level >= 0; --level) {
        const uint8_t *I = L.I[level], *J = L.J[level];
        const int cols = L.w[level], rows = L.h[level];
        const float sc = (float)(1. / (1 << level));
        float ppx = px0 * sc, ppy = py0 * sc;
        if (level == L.n - 1) { nx = nx * sc; ny = ny * sc; } else { nx = nx * 2.f; ny = ny * 2.f; }
        ppx -= half; ppy -= half;
        const int ipx = (int)floorf(ppx), ipy = (int)floorf(ppy);
        if (ipx < -kWin || ipx >= cols || ipy < -kWin || ipy >= rows) {
            if (level == 0) { st = false; err_out = 0.f; }
            continue;
        }
        int w00, w01, w10, w11;
        bilinear_weights(ppx - (float)ipx, ppy - (float)ipy, w00, w01, w10, w11);
        // stage the 24x24 neighbourhood (REFLECT_101 outside the image: pyrBorder)
        for (int e = lane; e < 24 * 24; e += 32) {
            const int yy = e / 24, xx = e - yy * 24;
            Ip[e] = I[(size_t)reflect101(ipy - 1 + yy, rows) * cols + reflect101(ipx - 1 + xx, cols)];
        }
        __syncwarp();
        // Scharr derivatives on the 22x22 interior; zero outside the image (derivBorder = CONSTANT)
        for (int e = lane; e < 22 * 22; e += 32) {
            const int yy = e / 22, xx = e - yy * 22;
            const int gx = ipx + xx, gy = ipy + yy;
            int dx = 0, dy = 0;
            if (gx >= 0 && gx < cols && gy >= 0 && gy < rows) {
                const int *c = Ip + (yy + 1) * 24 + (xx + 1);
                // neighbours must reflect about the IMAGE edge; the staged patch did exactly that
                const int a00 = c[-25], a01 = c[-24], a02 = c[-23], a10 = c[-1], a12 = c[1], a20 = c[23], a21 = c[24], a22 = c[25];
                dx = 3 * (a02 - a00) + 10 * (a12 - a10) + 3 * (a22 - a20);
                dy = 3 * (a20 - a00) + 10 * (a21 - a01) + 3 * (a22 - a02);
            }
            Dp[2 * e] = (short)dx; Dp[2 * e + 1] = (short)dy;
        }
        __syncwarp();
        long long sA11 = 0, sA12 = 0, sA22 = 0;
        for (int e = lane; e < kWin * kWin; e += 32) {
            const int yy = e / kWin, xx = e - yy * kWin;
            const int *c = Ip + (yy + 1) * 24 + (xx + 1);
            const int ival = descale(c[0] * w00 + c[1] * w01 + c[24] * w10 + c[25] * w11, kWBits - 5);
            const short *d = Dp + 2 * (yy * 22 + xx);
            const int ixv = descale(d[0] * w00 + d[2] * w01 + d[44] * w10 + d[46] * w11, kWBits);
            const int iyv = descale(d[1] * w00 + d[3] * w01 + d[45] * w10 + d[47] * w11, kWBits);
            Iw[e] = (short)ival; dIw[2 * e] = (short)ixv; dIw[2 * e + 1] = (short)iyv;
            sA11 += (long long)ixv * ixv; sA12 += (long long)ixv * iyv; sA22 += (long long)iyv * iyv;
        }
        sA11 = warp_sum(sA11); sA12 = warp_sum(sA12); sA22 = warp_sum(sA22);
        __syncwarp();
        const float FLT_SCALE = 1.f / (1 << 20);
        const float A11 = (float)sA11 * FLT_SCALE, A12 = (float)sA12 * FLT_SCALE, A22 = (float)sA22 * FLT_SCALE;
        float D = A11 * A22 - A12 * A12;
        const float min_eig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * kWin * kWin);
        if (min_eig < min_eig_thr || D < 1.1920929e-07f) {
            if (level == 0) st = false;
            continue;
        }
        D = 1.f / D;
        nx -= half; ny -= half;
        float pdx = 0.f, pdy = 0.f;
        float outx = nx + half, outy = ny + half;
        for (int j = 0; j < max_iter; ++j) {
            const int inx = (int)floorf(nx), iny = (int)floorf(ny);
            if (inx < -kWin || inx >= cols || iny < -kWin || iny >= rows) {
                if (level == 0) st = false;
                break;
            }
            bilinear_weights(nx - (float)inx, ny - (float)iny, w00, w01, w10, w11);
            long long sb1 = 0, sb2 = 0;
            for (int e = lane; e < kWin * kWin; e += 32) {
                const int yy = e / kWin, xx = e - yy * kWin;
                const int y0 = reflect101(iny + yy, rows), y1 = reflect101(iny + yy + 1, rows);
                const int x0 = reflect101(inx + xx, cols), x1 = reflect101(inx + xx + 1, cols);
                const int v = J[(size_t)y0 * cols + x0] * w00 + J[(size_t)y0 * cols + x1] * w01 +
                              J[(size_t)y1 * cols + x0] * w10 + J[(size_t)y1 * cols + x1] * w11;
                const int diff = descale(v, kWBits - 5) - Iw[e];
                sb1 += (long long)diff * dIw[2 * e]; sb2 += (long long)diff * dIw[2 * e + 1];
            }
            sb1 = warp_sum(sb1); sb2 = warp_sum(sb2);
            const float b1 = (float)sb1 * FLT_SCALE, b2 = (float)sb2 * FLT_SCALE;
            const float dx = (A12 * b2 - A22 * b1) * D, dy = (A12 * b1 - A11 * b2) * D;
            nx += dx; ny += dy;
            outx = nx + half; outy = ny + half;
            if ((double)dx * dx + (double)dy * dy <= eps2) break;
            if (j > 0 && fabs((double)(dx + pdx)) < 0.01 && fabs((double)(dy + pdy)) < 0.01) {
                outx -= dx * 0.5f; outy -= dy * 0.5f;
                break;
            }
            pdx = dx; pdy = dy;
        }
        nx = outx; ny = outy;
        if (st && level == 0) {
            const float qx = nx - half, qy = ny - half;
            const int inx = (int)floorf(qx), iny = (int)floorf(qy);
            if (inx < -kWin || inx >= cols || iny < -kWin || iny >= rows) {
                st = false;
            } else {
                bilinear_weights(qx - (float)inx, qy - (float)iny, w00, w01, w10, w11);
                long long se = 0;
                for (int e = lane; e < kWin * kWin; e += 32) {
                    const int yy = e / kWin, xx = e - yy * kWin;
                    const int y0 = reflect101(iny + yy, rows), y1 = reflect101(iny + yy + 1, rows);
                    const int x0 = reflect101(inx + xx, cols), x1 = reflect101(inx + xx + 1, cols);
                    const int v = J[(size_t)y0 * cols + x0] * w00 + J[(size_t)y0 * cols + x1] * w01 +
                                  J[(size_t)y1 * cols + x0] * w10 + J[(size_t)y1 * cols + x1] * w11;
                    const int diff = descale(v, kWBits - 5) - Iw[e];
                    se += diff < 0 ? -diff : diff;
                }
                se = warp_sum(se);
                err_out = (float)se * 1.f / (float)(32 * kWin * kWin);
            }
        }
    }
    if (lane == 0) {
        next_pts[2 * pt] = nx; next_pts[2 * pt + 1] = ny;
        status[pt] = st ? 1 : 0;
        if (err) err[pt] = st ? err_out : 0.f;
    }
}

static int klt_prepare(Handle *h, int w, int hgt, int max_level, int n_points) {
    KltState &k = h->klt;
    if (k.w != w || k.h != hgt || k.levels != max_level + 1 || k.cap_pts < n_points) {   // (drops the image cache)
        k = KltState{};
        k.w = w; k.h = hgt; k.levels = max_level + 1; k.cap_pts = std::max(n_points, 1024);
        size_t off = 0;
        int lw = w, lh = hgt;
        for (int l = 0; l <= max_level; ++l) {
            k.lw[l] = lw; k.lh[l] = lh; k.off[l] = off;
            off += ((size_t)lw * lh + 255) & ~(size_t)255;
            lw = (lw + 1) / 2; lh = (lh + 1) / 2;
        }
        k.off[max_level + 1] = off;
    }
    for (auto &p : k.pyr) TRY(reserve(h, p, k.off[k.levels], kDevice));
    TRY(reserve(h, k.pts, 5 * (size_t)k.cap_pts, kBoth));
    TRY(reserve(h, k.status, k.cap_pts, kBoth));
    TRY(reserve(h, k.img, (size_t)2 * w * hgt, kPinned));
    return 0;
}

int klt_track_impl(Handle *h, const uint8_t *prev, const uint8_t *next, int width, int height, int stride,
                   const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                   int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                   uint8_t *prev_eq, uint8_t *next_eq, uint64_t prev_id, uint64_t next_id, int border) {
    if (width < 2 || height < 2 || stride < width || n_points < 0 || max_level < 0 || max_level >= kMaxLevels || border < 0)
        return fail(h, PVIO_B200_EINVAL, "klt: bad arguments");
    const bool do_clahe = clahe_clip > 0.0;
    if (do_clahe && (tiles_x < 1 || tiles_y < 1 || width % tiles_x || height % tiles_y))
        return fail(h, PVIO_B200_EINVAL, "clahe: the image size must be a multiple of the tile grid");
    if (n_points == 0) return 0;
    // cv::buildOpticalFlowPyramid halves first and drops the NEW level if it is not larger than the window
    int levels = 1, lw = width, lh = height;
    while (levels <= max_level) {
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
        if (lw <= kWin || lh <= kWin) break;
        ++levels;
    }
    if (levels - 1 < max_level) max_level = levels - 1;
    TRY(klt_prepare(h, width, height, max_level, n_points));
    KltState &k = h->klt;
    const size_t img_bytes = (size_t)width * height, cap = k.cap_pts;
    float *h_pts = k.pts.h, *d_prev = k.pts.d, *d_next = k.pts.d + 2 * cap, *d_err = k.pts.d + 4 * cap;
    // which pyramid slot holds which frame: cached frames (same id, same preprocessing) are neither uploaded nor rebuilt
    int sp = -1, sn = -1;
    for (int i = 0; i < 2; ++i) {
        if (prev_id && k.pyr_id[i] == prev_id && k.pyr_clahe[i] == clahe_clip) sp = i;
        if (next_id && k.pyr_id[i] == next_id && k.pyr_clahe[i] == clahe_clip && i != sp) sn = i;
    }
    const bool have_prev = sp >= 0, have_next = sn >= 0;
    if (!have_prev) sp = have_next ? 1 - sn : 0;
    if (!have_next) sn = 1 - sp;
    if ((!have_prev && !prev) || (!have_next && !next)) return fail(h, PVIO_B200_EINVAL, "klt: image not cached and no pixels given");
    const uint8_t *src[2] = {prev, next};
    const int slot[2] = {sp, sn};
    const bool have[2] = {have_prev, have_next};
    for (int i = 0; i < 2; ++i) {
        if (have[i]) continue;
        for (int y = 0; y < height; ++y) memcpy(k.img.h + i * img_bytes + (size_t)y * width, src[i] + (size_t)y * stride, width);
    }
    memcpy(h_pts, prev_pts, sizeof(float) * 2 * n_points);
    memcpy(h_pts + 2 * cap, next_pts, sizeof(float) * 2 * n_points);
    if (do_clahe) {
        // raw frames -> device, CLAHE on the device into level 0 of the pyramids (opencv_image.cpp:138-143)
        for (auto &r : k.raw) TRY(reserve(h, r, img_bytes, kDevice));
        TRY(reserve(h, k.lut, (size_t)tiles_x * tiles_y * 256, kDevice));
    }
    for (int i = 0; i < 2; ++i) {
        if (have[i]) continue;
        uint8_t *P = k.pyr[slot[i]].d;
        if (do_clahe) {
            CK(h, cudaMemcpyAsync(k.raw[i].d, k.img.h + i * img_bytes, img_bytes, cudaMemcpyHostToDevice, h->stream));
            clahe_device(h, k.raw[i].d, P, k.lut.d, width, height, clahe_clip, tiles_x, tiles_y);
        } else {
            CK(h, cudaMemcpyAsync(P, k.img.h + i * img_bytes, img_bytes, cudaMemcpyHostToDevice, h->stream));
        }
        for (int l = 1; l <= max_level; ++l) {
            dim3 b(32, 8), g((k.lw[l] + 31) / 32, (k.lh[l] + 7) / 8);
            pyrdown_kernel<<<g, b, 0, h->stream>>>(P + k.off[l - 1], k.lw[l - 1], k.lh[l - 1], P + k.off[l], k.lw[l], k.lh[l]);
            ++h->launches;
        }
    }
    k.pyr_id[sp] = prev_id; k.pyr_clahe[sp] = clahe_clip;
    k.pyr_id[sn] = next_id; k.pyr_clahe[sn] = clahe_clip;
    CK(h, cudaMemcpyAsync(d_prev, h_pts, sizeof(float) * 2 * n_points, cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(d_next, h_pts + 2 * cap, sizeof(float) * 2 * n_points, cudaMemcpyHostToDevice, h->stream));
    KltLevels L;
    L.n = max_level + 1;
    for (int l = 0; l <= max_level; ++l) {
        L.I[l] = k.pyr[sp].d + k.off[l]; L.J[l] = k.pyr[sn].d + k.off[l];
        L.w[l] = k.lw[l]; L.h[l] = k.lh[l];
    }
    const int mi = std::min(std::max(max_iter, 0), 100);
    const double e = std::min(std::max(eps, 0.0), 10.0);
    klt_track_kernel<<<(n_points + kKltWarps - 1) / kKltWarps, 32 * kKltWarps, 0, h->stream>>>(
        L, d_prev, d_next, k.status.d, d_err, n_points, mi, e * e, 1e-4f);
    ++h->launches;
    if (border > 0) {
        klt_border_kernel<<<(n_points + 127) / 128, 128, 0, h->stream>>>(d_next, k.status.d, n_points, width, height, border);
        ++h->launches;
    }
    CK(h, cudaMemcpyAsync(h_pts + 2 * cap, d_next, sizeof(float) * 2 * n_points, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(h_pts + 4 * cap, d_err, sizeof(float) * n_points, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaMemcpyAsync(k.status.h, k.status.d, n_points, cudaMemcpyDeviceToHost, h->stream));
    if (do_clahe && (prev_eq || next_eq)) {
        CK(h, cudaMemcpyAsync(k.img.h, k.pyr[sp].d, img_bytes, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaMemcpyAsync(k.img.h + img_bytes, k.pyr[sn].d, img_bytes, cudaMemcpyDeviceToHost, h->stream));
    }
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaGetLastError());
    memcpy(next_pts, h_pts + 2 * cap, sizeof(float) * 2 * n_points);
    if (err) memcpy(err, h_pts + 4 * cap, sizeof(float) * n_points);
    memcpy(status, k.status.h, n_points);
    if (do_clahe && prev_eq) memcpy(prev_eq, k.img.h, img_bytes);
    if (do_clahe && next_eq) memcpy(next_eq, k.img.h + img_bytes, img_bytes);
    return 0;
}

// Level 0 (the equalised image) of a frame in the pyramid cache, or nullptr: the detector reads the frame the tracker
// has just uploaded (frame.cpp:108-130 detects on the image it tracked into)
const uint8_t *klt_cached_level0(Handle *h, uint64_t frame_id, int width, int height, double clahe_clip) {
    const KltState &k = h->klt;
    if (!frame_id || k.w != width || k.h != height) return nullptr;
    for (int i = 0; i < 2; ++i) if (k.pyr_id[i] == frame_id && k.pyr_clahe[i] == clahe_clip) return k.pyr[i].d;
    return nullptr;
}
// CLAHE of a device image into a device image (the detector's own upload path)
int klt_clahe_device(Handle *h, const uint8_t *d_src, uint8_t *d_dst, uint8_t *d_lut, int width, int height, double clip, int tiles_x, int tiles_y) {
    clahe_device(h, d_src, d_dst, d_lut, width, height, clip, tiles_x, tiles_y);
    return 0;
}

// stand-alone CLAHE of one host image (dst row stride = width)
int clahe_impl(Handle *h, const uint8_t *src, int width, int height, int stride, double clip, int tiles_x, int tiles_y, uint8_t *dst) {
    if (width < 1 || height < 1 || stride < width || clip <= 0.0 || tiles_x < 1 || tiles_y < 1 || width % tiles_x || height % tiles_y)
        return fail(h, PVIO_B200_EINVAL, "clahe: bad arguments (the image size must be a multiple of the tile grid)");
    const size_t bytes = (size_t)width * height;
    DevBuf<uint8_t> buf;
    TRY(alloc(h, buf, 2 * bytes + (size_t)tiles_x * tiles_y * 256, kDevice));
    uint8_t *d = buf.d;
    CK(h, cudaMemcpy2DAsync(d, width, src, stride, width, height, cudaMemcpyHostToDevice, h->stream));
    clahe_device(h, d, d + bytes, d + 2 * bytes, width, height, clip, tiles_x, tiles_y);
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(dst, d + bytes, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // namespace pvio
