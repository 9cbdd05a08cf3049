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
#include <algorithm>
#include <cstring>
#include <functional>
#include <vector>
#include "api_internal.h"
#include "klt_border.cuh"

namespace pvio {

constexpr int kWin = 21;
constexpr int kWBits = 14;
constexpr int kKltWarps = 4;

struct KltLevels {
    const uint8_t *I[kMaxLevels];
    const uint8_t *J[kMaxLevels];
    int w[kMaxLevels], h[kMaxLevels];
    int n;
};

// ---- CLAHE (cv::createCLAHE(clip, tiles)->apply, opencv_image.cpp:138-143; algorithm: OpenCV imgproc/clahe.cpp,
// restated in oracle/clahe_oracle.py which is pinned bit for bit against cv2).  Image sizes that are multiples
// of the tile grid only.  Kernel 1: one CTA per tile -- histogram in shared memory, clip + redistribute, prefix
// sum, LUT = cvRound(cdf * 255 / area).  Kernel 2: one thread per pixel, bilinear blend of the four neighbouring
// tiles' LUTs in OpenCV's float32 operation order (explicit _rn intrinsics: no FMA contraction).
// The frame is frames[blockIdx.y] (lut kernel) / frames[blockIdx.z] (apply kernel).
__global__ void __launch_bounds__(256) clahe_lut_kernel(int tiles_x, const KltBatchFrame *frames) {
    __shared__ int hist[256];
    __shared__ int wsum[8];
    __shared__ int total_clipped;
    const KltBatchFrame &fr = frames[blockIdx.y];
    const uint8_t *src = fr.raw;
    uint8_t *lut = fr.lut;
    const int w = fr.w[0], tw = fr.tw, th = fr.th, clip = fr.clip;
    const float lut_scale = fr.lut_scale;
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

__global__ void clahe_apply_kernel(int tiles_x, int tiles_y, const KltBatchFrame *frames) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const KltBatchFrame &f = frames[blockIdx.z];
    const uint8_t *src = f.raw, *lut = f.lut;
    uint8_t *dst = f.pyr;
    const int w = f.w[0], h = f.h[0], tw = f.tw, th = f.th;
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

// cv::CLAHE's per-tile constants of a w x h image
void klt_clahe_params(int w, int hgt, double clip_limit, int tiles_x, int tiles_y, int &tw, int &th, int &clip,
                      float &lut_scale) {
    tw = w / tiles_x; th = hgt / tiles_y;
    const int area = tw * th;
    clip = std::max((int)(clip_limit * area / 256), 1);
    lut_scale = 255.0f / (float)area;
}

// CLAHE of n_frames frames (in device memory), each into level 0 of its f.pyr
void klt_batch_clahe(Handle *h, const KltBatchFrame *frames, int n_frames, int tiles_x, int tiles_y, int max_w, int max_h) {
    clahe_lut_kernel<<<dim3((unsigned)(tiles_x * tiles_y), n_frames), 256, 0, h->stream>>>(tiles_x, frames);
    clahe_apply_kernel<<<dim3((max_w + 31) / 32, (max_h + 7) / 8, n_frames), dim3(32, 8), 0, h->stream>>>(tiles_x, tiles_y, frames);
    h->launches += 2;
}

// Level `level` of frame frames[blockIdx.z] (frames with fewer levels exit).
// The taps 2x - 2 .. 2x + 2 of a dw = (sw + 1) / 2 wide level reach -2 and at most 2 dw <= sw + 1: one fold brings them
// inside whenever sw >= 3 (reflect101_once), and klt_levels only builds a level from one of at least 43 px.
__global__ void pyrdown_kernel(const KltBatchFrame *frames, int level) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
    const KltBatchFrame &f = frames[blockIdx.z];
    if (level >= f.levels) return;
    const uint8_t *src = f.pyr + f.off[level - 1];
    uint8_t *dst = f.pyr + f.off[level];
    const int sw = f.w[level - 1], sh = f.h[level - 1], dw = f.w[level], dh = f.h[level];
    if (x >= dw || y >= dh) return;
    const int k[5] = {1, 4, 6, 4, 1};
    int acc = 0;
#pragma unroll
    for (int dy = -2; dy <= 2; ++dy) {
        const uint8_t *row = src + (size_t)reflect101_once(2 * y + dy, sh) * sw;
        int r = 0;
#pragma unroll
        for (int dx = -2; dx <= 2; ++dx) r += k[dx + 2] * row[reflect101_once(2 * x + dx, sw)];
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

// Point pt belongs to pair pair_of[pt], whose pyramids are pairs[pair_of[pt]] (in device memory); with border > 0 the
// 20-pixel border rejection of OpenCvImage::track_keypoints (opencv_image.cpp:106-108) on that pair's frame size follows.
__global__ void __launch_bounds__(32 * kKltWarps)
klt_track_kernel(const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points, int max_iter, double eps2,
                 float min_eig_thr, const KltLevels *pairs, const int *pair_of, int border) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int pt = blockIdx.x * kKltWarps + warp;
    __shared__ int Ipatch[kKltWarps][24 * 24];
    __shared__ short Dpatch[kKltWarps][22 * 22 * 2];
    __shared__ short IWin[kKltWarps][kWin * kWin];
    __shared__ short dIWin[kKltWarps][kWin * kWin * 2];
    if (pt >= n_points) return;
    const KltLevels &Lv = pairs[pair_of[pt]];
    const float px0 = prev_pts[2 * pt], py0 = prev_pts[2 * pt + 1];
    float nx = next_pts[2 * pt], ny = next_pts[2 * pt + 1];      // OPTFLOW_USE_INITIAL_FLOW
    bool st = true;
    float err_out = 0.f;
    const float half = (kWin - 1) * 0.5f;
    int *Ip = Ipatch[warp];
    short *Dp = Dpatch[warp], *Iw = IWin[warp], *dIw = dIWin[warp];

    for (int level = Lv.n - 1; level >= 0; --level) {
        const uint8_t *I = Lv.I[level], *J = Lv.J[level];
        const int cols = Lv.w[level], rows = Lv.h[level];
        const float sc = (float)(1. / (1 << level));
        float ppx = px0 * sc, ppy = py0 * sc;
        if (level == Lv.n - 1) { nx = nx * sc; ny = ny * sc; } else { nx = nx * 2.f; ny = ny * 2.f; }
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
        bool keep = st;
        if (border > 0) {
            const int w = Lv.w[0], h = Lv.h[0];
            if (nx < (float)border || nx >= (float)(w - border) || ny < (float)border || ny >= (float)(h - border)) keep = false;
        }
        status[pt] = keep ? 1 : 0;
        if (err) err[pt] = st ? err_out : 0.f;
    }
}

// cv::buildOpticalFlowPyramid halves first and drops the NEW level if it is not larger than the window: the number of
// levels (level 0 included) a width x height frame gets for maxLevel max_level
int klt_levels(int width, int height, int max_level) {
    int levels = 1, lw = width, lh = height;
    while (levels <= max_level) {
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
        if (lw <= kWin || lh <= kWin) break;
        ++levels;
    }
    return levels;
}

// the level sizes and offsets of an empty cache for w x hgt frames with `levels` levels
void klt_layout(KltPyramids &k, int w, int hgt, int levels) {
    k.w = w; k.h = hgt; k.levels = levels;
    size_t off = 0;
    int lw = w, lh = hgt;
    for (int l = 0; l < levels; ++l) {
        k.lw[l] = lw; k.lh[l] = lh; k.off[l] = off;
        off += ((size_t)lw * lh + 255) & ~(size_t)255;
        lw = (lw + 1) / 2; lh = (lh + 1) / 2;
    }
    k.off[levels] = off;
}

// which pyramid of the cache takes which frame (pyr[slot[0]] prev, pyr[slot[1]] next): cached frames (same id, same
// preprocessing) are neither uploaded nor rebuilt (have[i])
static void klt_lookup(const KltPyramids &k, uint64_t prev_id, uint64_t next_id, double clahe_clip, int slot[2], bool have[2]) {
    int sp = -1, sn = -1;
    for (int i = 0; i < 2; ++i) {
        if (prev_id && k.pyr_id[i] == prev_id && k.pyr_clahe[i] == clahe_clip) sp = i;
        if (next_id && k.pyr_id[i] == next_id && k.pyr_clahe[i] == clahe_clip && i != sp) sn = i;
    }
    have[0] = sp >= 0; have[1] = sn >= 0;
    if (!have[0]) sp = have[1] ? 1 - sn : 0;
    if (!have[1]) sn = 1 - sp;
    slot[0] = sp; slot[1] = sn;
}

// The pyramids of n_frames new frames (frames: host copies of the descriptors at d_frames): CLAHE into level 0, or
// without CLAHE a device copy of the raw pixels into level 0 unless they were uploaded there; then one pyrDown launch per
// level over every frame (grid z)
static int klt_build_pyramids(Handle *h, const KltBatchFrame *frames, const KltBatchFrame *d_frames, int n_frames, bool clahe,
                              int tiles_x, int tiles_y) {
    int levels = 1, lw[kMaxLevels] = {}, lh[kMaxLevels] = {};
    for (int j = 0; j < n_frames; ++j) {
        const KltBatchFrame &f = frames[j];
        levels = std::max(levels, f.levels);
        for (int l = 0; l < f.levels; ++l) { lw[l] = std::max(lw[l], f.w[l]); lh[l] = std::max(lh[l], f.h[l]); }
        if (!clahe && f.raw != f.pyr)
            CK(h, cudaMemcpyAsync(f.pyr, f.raw, (size_t)f.w[0] * f.h[0], cudaMemcpyDeviceToDevice, h->stream));
    }
    if (clahe) klt_batch_clahe(h, d_frames, n_frames, tiles_x, tiles_y, lw[0], lh[0]);
    for (int l = 1; l < levels; ++l) {
        pyrdown_kernel<<<dim3((lw[l] + 31) / 32, (lh[l] + 7) / 8, n_frames), dim3(32, 8), 0, h->stream>>>(d_frames, l);
        ++h->launches;
    }
    return 0;
}

// LK + border over n_pts points of the pairs `pairs` (every array in device memory)
static void klt_lk(Handle *h, const KltLevels *pairs, const int *pair_of, const float *prev_pts, float *next_pts, uint8_t *status,
                   float *err, size_t n_pts, int max_iter, double eps, int border) {
    const int mi = std::min(std::max(max_iter, 0), 100);
    const double e = std::min(std::max(eps, 0.0), 10.0);
    klt_track_kernel<<<(unsigned)((n_pts + kKltWarps - 1) / kKltWarps), 32 * kKltWarps, 0, h->stream>>>(
        prev_pts, next_pts, status, err, (int)n_pts, mi, e * e, 1e-4f, pairs, pair_of, border);
    ++h->launches;
}

// the descriptor of the pair s.pyr[slot[0]] (prev), s.pyr[slot[1]] (next) as klt_track_kernel reads it
static KltLevels klt_pair(const KltPyramids &s, const int slot[2]) {
    KltLevels L{};
    L.n = s.levels;
    for (int l = 0; l < s.levels; ++l) {
        L.I[l] = s.pyr[slot[0]].d + s.off[l]; L.J[l] = s.pyr[slot[1]].d + s.off[l];
        L.w[l] = s.lw[l]; L.h[l] = s.lh[l];
    }
    return L;
}

// the descriptor of a new frame whose pyramid is s.pyr[i]: its pixels at raw, its CLAHE tables at lut (clip > 0)
static KltBatchFrame klt_frame(const KltPyramids &s, int i, uint8_t *raw, uint8_t *lut, double clip, int tiles_x, int tiles_y) {
    KltBatchFrame F{};
    F.raw = raw; F.lut = lut; F.pyr = s.pyr[i].d; F.levels = s.levels;
    for (int l = 0; l < s.levels; ++l) { F.w[l] = s.lw[l]; F.h[l] = s.lh[l]; F.off[l] = s.off[l]; }
    if (clip > 0.0) klt_clahe_params(s.w, s.h, clip, tiles_x, tiles_y, F.tw, F.th, F.clip, F.lut_scale);
    return F;
}

static int klt_prepare(Handle *h, int w, int hgt, int max_level, int n_points) {
    KltState &k = h->klt;
    if (k.w != w || k.h != hgt || k.levels != max_level + 1 || k.cap_pts < n_points) {   // (drops the image cache)
        k = KltState{};
        klt_layout(k, w, hgt, max_level + 1);
        k.cap_pts = std::max(n_points, 1024);
    }
    for (auto &p : k.pyr) TRY(reserve(h, p, k.off[k.levels], kDevice));
    TRY(reserve(h, k.img, (size_t)2 * w * hgt, kPinned));
    return 0;
}

// The single call: one pair of the cache h->klt.  Its pair descriptor, the descriptors of the frames it uploads, a zero
// pair index per point and the points go to the device in one copy; each new frame's pixels are copied into level 0 of
// its pyramid (raw[i] with CLAHE).  The pyramids are built one frame at a time, so the launches of a call tell how many
// it built; one D2H copy brings positions, errors and status back.
int klt_track_impl(Handle *h, const uint8_t *prev, const uint8_t *next, int width, int height, int stride,
                   const float *prev_pts, float *next_pts, uint8_t *status, float *err, int n_points,
                   int max_level, int max_iter, double eps, double clahe_clip, int tiles_x, int tiles_y,
                   uint8_t *prev_eq, uint8_t *next_eq, uint64_t prev_id, uint64_t next_id, int border) {
    if (width < kKltMinFrame || height < kKltMinFrame || stride < width || n_points < 0 || max_level < 0 || max_level >= kMaxLevels || border < 0)
        return fail(h, PVIO_B200_EINVAL, "klt: bad arguments");
    const bool do_clahe = clahe_clip > 0.0;
    if (do_clahe && (tiles_x < 1 || tiles_y < 1 || width % tiles_x || height % tiles_y))
        return fail(h, PVIO_B200_EINVAL, "clahe: the image size must be a multiple of the tile grid");
    if (n_points == 0) return 0;
    max_level = klt_levels(width, height, max_level) - 1;
    TRY(klt_prepare(h, width, height, max_level, n_points));
    KltState &k = h->klt;
    const size_t img_bytes = (size_t)width * height, n = n_points;
    int slot[2];
    bool have[2];
    klt_lookup(k, prev_id, next_id, clahe_clip, slot, have);
    const int sp = slot[0], sn = slot[1];
    if ((!have[0] && !prev) || (!have[1] && !next)) return fail(h, PVIO_B200_EINVAL, "klt: image not cached and no pixels given");
    if (do_clahe) {
        for (auto &r : k.raw) TRY(reserve(h, r, img_bytes, kDevice));
        TRY(reserve(h, k.lut, (size_t)tiles_x * tiles_y * 256, kDevice));
    }

    // staging: pair descriptor, frame descriptors, pair indices, points (uploaded) | initial guesses in, positions out |
    // errors, status (downloaded)
    Stage S(k.stage);
    const auto lv = S.add<KltLevels>(Stage::kUp, 1);
    const auto fr = S.add<KltBatchFrame>(Stage::kUp, 2);
    const auto pof = S.add<int>(Stage::kUp, n);
    const auto pp = S.add(Stage::kUp, 2 * n, prev_pts);
    const auto np = S.add(Stage::kInOut, 2 * n, next_pts);
    const auto er = S.add<float>(Stage::kDown, n);
    const auto stat = S.add<uint8_t>(Stage::kDown, n);
    TRY(S.place(h));
    *S.host(lv) = klt_pair(k, slot);
    memset(S.host(pof), 0, sizeof(int) * n);
    KltBatchFrame *frm = S.host(fr);
    const uint8_t *src[2] = {prev, next};
    int nf = 0;
    for (int i = 0; i < 2; ++i) {
        if (have[i]) continue;
        uint8_t *img = k.img.h + i * img_bytes;
        for (int y = 0; y < height; ++y) memcpy(img + (size_t)y * width, src[i] + (size_t)y * stride, width);
        uint8_t *dst = do_clahe ? k.raw[i].d : k.pyr[slot[i]].d;     // without CLAHE: straight into level 0
        frm[nf++] = klt_frame(k, slot[i], dst, k.lut.d, clahe_clip, tiles_x, tiles_y);
        CK(h, cudaMemcpyAsync(dst, img, img_bytes, cudaMemcpyHostToDevice, h->stream));
    }
    TRY(S.upload(h));
    for (int j = 0; j < nf; ++j) TRY(klt_build_pyramids(h, frm + j, S.dev(fr) + j, 1, do_clahe, tiles_x, tiles_y));
    k.pyr_id[sp] = prev_id; k.pyr_clahe[sp] = clahe_clip;
    k.pyr_id[sn] = next_id; k.pyr_clahe[sn] = clahe_clip;
    klt_lk(h, S.dev(lv), S.dev(pof), S.dev(pp), S.dev(np), S.dev(stat), S.dev(er), n, max_iter, eps, border);
    TRY(S.download(h));
    if (do_clahe && (prev_eq || next_eq)) {
        CK(h, cudaMemcpyAsync(k.img.h, k.pyr[sp].d, img_bytes, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaMemcpyAsync(k.img.h + img_bytes, k.pyr[sn].d, img_bytes, cudaMemcpyDeviceToHost, h->stream));
    }
    CK(h, cudaStreamSynchronize(h->stream));
    CK(h, cudaGetLastError());
    memcpy(next_pts, S.host(np), sizeof(float) * 2 * n);
    if (err) memcpy(err, S.host(er), sizeof(float) * n);
    memcpy(status, S.host(stat), n);
    if (do_clahe && prev_eq) memcpy(prev_eq, k.img.h, img_bytes);
    if (do_clahe && next_eq) memcpy(next_eq, k.img.h + img_bytes, img_bytes);
    return 0;
}

// ---- the batched tracker (pvio_b200_batch_track_keypoints) --------------------------------------------------------
// n frame pairs of n sequences, each with its own pyramid cache (h->kltb.slots[pair.slot]).  Every pair is checked before
// anything changes.  Then: one H2D copy of the packed staging; CLAHE (2 launches) and pyrDown (one launch per level)
// over every new frame; LK + border over every point of every pair (1); per pair, the survivors compacted and OpenCV's
// sample schedule drawn on the device (1); every RANSAC iteration of every pair (1); one D2H copy of the results and a
// synchronise; the host replays each pair as fm_ransac_impl does; one launch writes every winner's mask, one D2H copy,
// a synchronise.  Without CLAHE each new frame is copied into level 0 of its pyramid (a device copy per frame).
// A new frame of a slot with a lens (pvio_b200_batch_set_lens) is uploaded raw and remapped first (1 launch over every
// such frame, undistort.cu): into a scratch frame that CLAHE reads, or without CLAHE straight into level 0 of its
// pyramid in place of its device copy.  These frames come first in the descriptor array, so the remap's grid covers
// them alone.
namespace {
constexpr int kMaxBatchPairs = 32767;         // grid y / z limits: one block row per pair, per new frame
constexpr int kFmIters = 1000;                // findFundamentalMat's maxIters, as pvio_b200_track_keypoints passes it
}  // namespace

int batch_track_impl(Handle *h, int n, const pvio_b200_klt_pair *pairs, int max_level, int max_iter, double eps,
                     double clahe_clip, int tiles_x, int tiles_y, int border, double ransac_threshold,
                     double ransac_confidence) {
    if (n < 0 || n > kMaxBatchPairs) return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad pair count");
    if (n == 0) return 0;
    if (!pairs) return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad arguments");
    std::vector<KltBatchItem> items(n);
    for (int i = 0; i < n; ++i) {
        const pvio_b200_klt_pair &a = pairs[i];
        if (!a.prev_id) return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad shape, stride or frame id");
        if (a.n_points > 0 && !a.status) return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad points");
        items[i] = KltBatchItem{a.slot, a.width, a.height, a.stride, a.n_points, a.prev_id, a.next_id, a.prev, a.next,
                                a.prev_pts, a.next_pts};
    }
    const KltBatchOptions o{max_level, max_iter, eps, clahe_clip, tiles_x, tiles_y, border, ransac_threshold, ransac_confidence};
    KltBatchResults r;
    TRY(klt_batch_track(h, n, items.data(), o, nullptr, r));
    bool any_job = false;
    for (int i = 0; i < n; ++i) {
        const pvio_b200_klt_pair &a = pairs[i];
        const int np = a.n_points;
        if (np > 0) {
            memcpy(a.next_pts, r.next + 2 * r.first[i], sizeof(float) * 2 * np);
            memcpy(a.status, r.status + r.first[i], np);
            if (a.err) memcpy(a.err, r.err + r.first[i], sizeof(float) * np);
            if (r.clear[i]) memset(a.status, 0, np);     // getSubset gave up at once, or no model won: the mask is all zero
        }
        any_job |= r.mask[i] != nullptr;
    }
    if (any_job) {
        CK(h, cudaMemcpyAsync(r.mw, r.d_mw, sizeof(unsigned) * r.words, cudaMemcpyDeviceToHost, h->stream));
        CK(h, cudaStreamSynchronize(h->stream));
        for (int i = 0; i < n; ++i) {
            const pvio_b200_klt_pair &a = pairs[i];
            if (!r.mask[i]) continue;
            const unsigned *m = r.mw + (r.mask[i] - r.d_mw);
            for (int j = 0, k = 0; j < a.n_points; ++j) {
                if (!a.status[j]) continue;
                if (!((m[k >> 5] >> (k & 31)) & 1u)) a.status[j] = 0;
                ++k;
            }
        }
    }
    for (int i = 0; i < n; ++i)
        if (pairs[i].info) memcpy(pairs[i].info, &r.info[4 * (size_t)i], sizeof(int32_t) * 4);
    return 0;
}

int klt_batch_track(Handle *h, int n, const KltBatchItem *pairs, const KltBatchOptions &opt, const KltDevicePoints *dev,
                    KltBatchResults &res) {
    const int max_level = opt.max_level, max_iter = opt.max_iter, tiles_x = opt.tiles_x, tiles_y = opt.tiles_y;
    const int border = opt.border;
    const double eps = opt.eps, clahe_clip = opt.clahe_clip;
    res.first.assign(n, 0);
    res.mask.assign(n, nullptr);
    res.clear.assign(n, 0);
    res.info.assign(4 * (size_t)n, 0);
    if (max_level < 0 || max_level >= kMaxLevels || border < 0 || !(clahe_clip >= 0.0))
        return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad arguments");
    const bool do_clahe = clahe_clip > 0.0;
    if (do_clahe && (tiles_x < 1 || tiles_y < 1)) return fail(h, PVIO_B200_EINVAL, "clahe: bad tile grid");
    KltBatchState &B = h->kltb;
    struct Plan {
        int levels, slot[2];                  // level count; which pyramid of the slot takes prev / next
        bool have[2], rebuild;                // prev / next cached; the slot's buffers are rebuilt (its cache dropped)
    };
    std::vector<Plan> plan(n);
    std::vector<uint8_t> taken;
    const KltPyramids empty;
    size_t n_pts = 0;
    for (int i = 0; i < n; ++i) {
        const KltBatchItem &a = pairs[i];
        TRY(take_slot(h, taken, a.slot, "batch_track_keypoints"));
        if (a.width < kKltMinFrame || a.height < kKltMinFrame || a.stride < a.width || !a.next_id)
            return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad shape, stride or frame id");
        if (do_clahe && (a.width % tiles_x || a.height % tiles_y))
            return fail(h, PVIO_B200_EINVAL, "clahe: the image size must be a multiple of the tile grid");
        const SlotLens *L = slot_lens(B, a.slot);
        if (L && (L->w != a.width || L->h != a.height))
            return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: the frame shape differs from the slot's lens");
        if (a.n_points < 0 || (a.n_points > 0 && !dev && (!a.prev_pts || !a.next_pts)) || (a.n_points > 0 && !a.prev_id))
            return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: bad points");
        Plan &pl = plan[i];
        pl.levels = klt_levels(a.width, a.height, max_level);
        const KltPyramids *c = (size_t)a.slot < B.slots.size() ? &B.slots[a.slot] : nullptr;
        pl.rebuild = !c || c->w != a.width || c->h != a.height || c->levels != pl.levels;
        klt_lookup(pl.rebuild ? empty : *c, a.prev_id, a.next_id, clahe_clip, pl.slot, pl.have);
        if (!a.prev_id) pl.have[0] = true;    // no previous frame: the next frame is only cached
        if ((!pl.have[0] && !a.prev) || (!pl.have[1] && !a.next))
            return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: image not cached in its slot and no pixels given");
        n_pts += a.n_points;
    }
    if (n_pts > ((size_t)1 << 28)) return fail(h, PVIO_B200_EINVAL, "batch_track_keypoints: too many points");

    // the slots: grown on demand, rebuilt on a shape change; per pair its RANSAC budget (iterations reserved)
    double thr = opt.ransac_threshold, conf = opt.ransac_confidence;
    int fm_iters = kFmIters;
    fm_options(thr, conf, fm_iters);
    const int lmeds_iters = fm_lmeds_iters(conf, fm_iters);
    if (taken.size() > B.slots.size()) B.slots.resize(taken.size());
    std::vector<int> budget(n);
    size_t n_frames = 0, pix_bytes = 0, budget_sum = 0, words_sum = 0, mask_words = 0, n_lens = 0, und_bytes = 0;
    int max_budget = 0, max_words = 0, lens_w = 0, lens_h = 0;
    for (int i = 0; i < n; ++i) {
        const KltBatchItem &a = pairs[i];
        const Plan &pl = plan[i];
        KltPyramids &s = B.slots[a.slot];
        if (pl.rebuild) {
            s = KltPyramids{};
            klt_layout(s, a.width, a.height, pl.levels);
        }
        for (auto &p : s.pyr) TRY(reserve(h, p, s.off[s.levels], kDevice));
        for (int side = 0; side < 2; ++side) {
            if (pl.have[side]) continue;
            ++n_frames;
            pix_bytes += align256((size_t)a.width * a.height);
            if (slot_lens(B, a.slot)) {
                ++n_lens;
                if (do_clahe) und_bytes += align256((size_t)a.width * a.height);
                lens_w = std::max(lens_w, a.width); lens_h = std::max(lens_h, a.height);
            }
        }
        const int np = a.n_points, nw = (np + 31) / 32;
        budget[i] = np < 8 ? 0 : np < 15 ? lmeds_iters : std::max(fm_iters, lmeds_iters);
        budget_sum += budget[i];
        words_sum += nw;
        mask_words += (size_t)3 * budget[i] * nw;
        max_budget = std::max(max_budget, budget[i]);
        max_words = std::max(max_words, nw);
    }

    // staging: pair descriptors, RANSAC problems, frame descriptors, pair indices, pixels, LK inputs (uploaded) | initial
    // guesses in, positions out | errors, status, survivors, counts (downloaded) and the winners' mask words (downloaded
    // by the caller) | mask jobs (read in place).  Points written on the device leave LK's inputs and outputs in scratch.
    // Scratch: CLAHE tables | survivors p, q | schedules | models | per-iteration masks | undistorted frames (CLAHE's
    // input)
    const size_t tiles = do_clahe ? (size_t)tiles_x * tiles_y : 0;
    Stage S(B.stage, &B.scratch);
    const auto sLv = S.add<KltLevels>(Stage::kUp, n);
    const auto sFmp = S.add<FmBatchProblem>(Stage::kUp, n);
    const auto sFrm = S.add<KltBatchFrame>(Stage::kUp, n_frames);
    const auto sPof = S.add<int>(Stage::kUp, n_pts);
    const auto sPix = S.add<uint8_t>(Stage::kUp, pix_bytes);
    const auto sPrev = S.add<float>(dev ? Stage::kScratch : Stage::kUp, 2 * n_pts);
    const auto sNext = S.add<float>(dev ? Stage::kScratch : Stage::kInOut, 2 * n_pts);
    const auto sErr = S.add<float>(dev ? Stage::kScratch : Stage::kDown, n_pts);
    const auto sSt = S.add<uint8_t>(dev ? Stage::kScratch : Stage::kDown, n_pts);
    const auto sSurv = S.add<int>(Stage::kDown, 2 * n);
    const auto sCnt = S.add<int>(Stage::kDown, 4 * budget_sum);
    const auto sMw = S.add<unsigned>(Stage::kDown, words_sum);
    const auto sJob = S.add<FmMaskJob>(Stage::kMapped, n);
    const auto sLut = S.add<uint8_t>(Stage::kScratch, tiles * 256 * n_frames);
    const auto sPq = S.add<float2>(Stage::kScratch, 2 * n_pts);
    const auto sSched = S.add<int>(Stage::kScratch, 7 * budget_sum);
    const auto sF = S.add<double>(Stage::kScratch, 27 * budget_sum);
    const auto sMasks = S.add<unsigned>(Stage::kScratch, mask_words);
    const auto sUnd = S.add<uint8_t>(Stage::kScratch, und_bytes);
    TRY(S.place(h));
    KltLevels *lv = S.host(sLv);
    FmBatchProblem *fmp = S.host(sFmp);
    KltBatchFrame *frm = S.host(sFrm);
    int *pof = S.host(sPof);
    float *h_prev = S.host(sPrev), *h_next = S.host(sNext);
    size_t p = 0, f_lens = 0, f_plain = n_lens, pix = 0, und = 0, bsum = 0, msum = 0;
    for (int i = 0; i < n; ++i) {
        const KltBatchItem &a = pairs[i];
        const Plan &pl = plan[i];
        KltPyramids &s = B.slots[a.slot];
        const SlotLens *L = slot_lens(B, a.slot);
        lv[i] = klt_pair(s, pl.slot);
        const uint8_t *src[2] = {a.prev, a.next};
        for (int side = 0; side < 2; ++side) {
            if (pl.have[side]) continue;
            uint8_t *dst = S.host(sPix) + pix;
            for (int y = 0; y < a.height; ++y) memcpy(dst + (size_t)y * a.width, src[side] + (size_t)y * a.stride, a.width);
            const size_t f = L ? f_lens++ : f_plain++;
            uint8_t *raw = S.dev(sPix) + pix;
            if (L) raw = do_clahe ? S.dev(sUnd) + und : s.pyr[pl.slot[side]].d;    // remapped: CLAHE's input, or level 0
            frm[f] = klt_frame(s, pl.slot[side], raw, S.dev(sLut) + f * tiles * 256, clahe_clip, tiles_x, tiles_y);
            if (L) {
                frm[f].lens_src = S.dev(sPix) + pix; frm[f].m1 = L->m1(); frm[f].m2 = L->m2();
                if (do_clahe) und += align256((size_t)a.width * a.height);
            }
            pix += align256((size_t)a.width * a.height);
        }
        if (a.prev_id) { s.pyr_id[pl.slot[0]] = a.prev_id; s.pyr_clahe[pl.slot[0]] = clahe_clip; }
        s.pyr_id[pl.slot[1]] = a.next_id; s.pyr_clahe[pl.slot[1]] = clahe_clip;
        const int np = a.n_points;
        res.first[i] = p;
        if (np > 0) {
            if (!dev) {
                memcpy(h_prev + 2 * p, a.prev_pts, sizeof(float) * 2 * np);
                memcpy(h_next + 2 * p, a.next_pts, sizeof(float) * 2 * np);
            }
            std::fill(pof + p, pof + p + np, i);
        }
        FmBatchProblem &P = fmp[i];
        P.prev_pts = S.dev(sPrev) + 2 * p;
        P.next_pts = S.dev(sNext) + 2 * p;
        P.status = S.dev(sSt) + p;
        P.p = S.dev(sPq) + p;
        P.q = S.dev(sPq) + n_pts + p;
        P.sched = S.dev(sSched) + 7 * bsum;
        P.counts = S.dev(sCnt) + 4 * bsum;
        P.F = S.dev(sF) + 27 * bsum;
        P.masks = S.dev(sMasks) + msum;
        P.surv = S.dev(sSurv) + 2 * i;
        P.n_pts = np;
        P.budget = budget[i];
        p += np;
        bsum += budget[i];
        msum += (size_t)3 * budget[i] * ((np + 31) / 32);
    }

    cudaStream_t st = h->stream;
    TRY(S.upload(h));
    if (dev && n_pts > 0) TRY(dev->write_points(h, S.dev(sPrev), S.dev(sNext), S.dev(sPof)));
    if (n_lens > 0) undistort_frames(h, S.dev(sFrm), (int)n_lens, lens_w, lens_h);
    if (n_frames > 0) TRY(klt_build_pyramids(h, frm, S.dev(sFrm), (int)n_frames, do_clahe, tiles_x, tiles_y));
    if (n_pts > 0)
        klt_lk(h, S.dev(sLv), S.dev(sPof), S.dev(sPrev), S.dev(sNext), S.dev(sSt), S.dev(sErr), n_pts, max_iter, eps, border);
    const FmBatchProblem *d_fmp = S.dev(sFmp);
    if (max_budget > 0) {
        fm_batch_schedule(h, d_fmp, n, fm_iters, lmeds_iters);
        fm_batch_hypotheses(h, d_fmp, n, max_budget, (float)(thr * thr));
    }
    CK(h, cudaGetLastError());
    // with the points on the device, only what the replay reads comes back
    TRY(dev ? S.download(h, sSurv, sCnt) : S.download(h, sNext, sCnt));
    CK(h, cudaStreamSynchronize(st));

    // each pair's replay (opencv_image.cpp:112-129: findFundamentalMat over >= 8 survivors)
    const int *r_surv = S.host(sSurv), *r_cnt = S.host(sCnt);
    FmMaskJob *jobs = S.host(sJob);
    res.next = dev ? S.dev(sNext) : S.host(sNext);
    res.err = dev ? S.dev(sErr) : S.host(sErr);
    res.status = dev ? S.dev(sSt) : S.host(sSt);
    res.mw = S.host(sMw);
    res.d_mw = S.dev(sMw);
    res.words = words_sum;
    bool any_job = false;
    bsum = 0;
    size_t wsum = 0;
    for (int i = 0; i < n; ++i) {
        const int np = pairs[i].n_points;
        int32_t *inf = &res.info[4 * (size_t)i];
        inf[0] = 0; inf[1] = -1; inf[2] = -1; inf[3] = 0;
        FmMaskJob &J = jobs[i];
        memset(&J, 0, sizeof(J));
        const int s = budget[i] ? r_surv[2 * i] : 0, have = budget[i] ? r_surv[2 * i + 1] : 0;
        if (s >= 8) {
            float thr_lmeds = 0.f;
            if (have > 0) thr_lmeds = fm_replay(r_cnt + 4 * bsum, s, have, fm_iters, conf, inf);
            const int bi = inf[1], bk = inf[2];
            if (have > 0 && bi >= 0) {
                const FmBatchProblem &P = fmp[i];
                J.p = P.p; J.q = P.q; J.n = s;
                J.out = S.dev(sMw) + wsum;
                if (s >= 15) J.src = P.masks + (size_t)(3 * bi + bk) * ((s + 31) / 32);
                else { J.F = P.F + (size_t)(3 * bi + bk) * 9; J.thr2 = thr_lmeds; }
                res.mask[i] = J.out;
                any_job = true;
            } else {
                res.clear[i] = 1;             // getSubset gave up at once, or no model won: the mask is all zero
            }
        }
        bsum += budget[i];
        wsum += (np + 31) / 32;
    }
    if (any_job) {
        FmMaskJob *d_jobs = nullptr;          // read in place from the pinned staging (mapped: unified addressing)
        CK(h, cudaHostGetDevicePointer(reinterpret_cast<void **>(&d_jobs), jobs, 0));
        fm_batch_masks(h, d_jobs, n, max_words);
        CK(h, cudaGetLastError());
    }
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

// stand-alone CLAHE of one host image (dst row stride = width)
int clahe_impl(Handle *h, const uint8_t *src, int width, int height, int stride, double clip, int tiles_x, int tiles_y, uint8_t *dst) {
    if (width < 1 || height < 1 || stride < width || clip <= 0.0 || tiles_x < 1 || tiles_y < 1 || width % tiles_x || height % tiles_y)
        return fail(h, PVIO_B200_EINVAL, "clahe: bad arguments (the image size must be a multiple of the tile grid)");
    const size_t bytes = (size_t)width * height, o_frm = align256(2 * bytes + (size_t)tiles_x * tiles_y * 256);
    DevBuf<uint8_t> buf;
    TRY(alloc(h, buf, o_frm + sizeof(KltBatchFrame), kDevice));
    uint8_t *d = buf.d;
    KltBatchFrame F{};                        // the image as one frame of one level
    F.raw = d; F.pyr = d + bytes; F.lut = d + 2 * bytes;
    F.levels = 1; F.w[0] = width; F.h[0] = height;
    klt_clahe_params(width, height, clip, tiles_x, tiles_y, F.tw, F.th, F.clip, F.lut_scale);
    CK(h, cudaMemcpy2DAsync(d, width, src, stride, width, height, cudaMemcpyHostToDevice, h->stream));
    CK(h, cudaMemcpyAsync(d + o_frm, &F, sizeof(F), cudaMemcpyHostToDevice, h->stream));
    klt_batch_clahe(h, reinterpret_cast<const KltBatchFrame *>(d + o_frm), 1, tiles_x, tiles_y, width, height);
    CK(h, cudaGetLastError());
    CK(h, cudaMemcpyAsync(dst, d + bytes, bytes, cudaMemcpyDeviceToHost, h->stream));
    CK(h, cudaStreamSynchronize(h->stream));
    return 0;
}

}  // namespace pvio
