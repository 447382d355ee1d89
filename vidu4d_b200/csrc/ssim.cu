// ssim.cu -- fused SSIM loss (gs/utils/loss_utils.py:33-68) and its gradient with respect to img1 (include/surfel_ssim.h).
//
// The reference evaluates SSIM with five depthwise 11x11 conv2d calls and about a dozen elementwise kernels, and keeps
// about 15 full-size intermediates for autograd.  Here:
//   ssim_fwd     one CTA per 32x32 output tile of one (image, channel) plane.  x and y of the tile plus a 5-pixel halo
//                (zero outside the image, as conv2d(padding=5)) are staged in shared memory; the 11-tap window runs
//                horizontally over x, y, x^2, y^2, xy into shared memory, then vertically in registers (four output
//                rows per thread).  Writes one partial sum of the SSIM map per CTA (never the map itself) and, when a
//                gradient is wanted, the three per-pixel maps A, B, Cm of surfel_ssim.h.
//   ssim_reduce  one CTA: a warp per image sums that image's partials in a fixed order (float64), then the block sums
//                the images' totals in a fixed order -- bit-identical run to run, no float atomics.
//   ssim_bwd     one CTA per 32x32 tile of one image, looping over its channels: the three maps (zero outside the
//                image) go through the same separable window, and each pixel's dL/dx is formed by its own thread.  With
//                the background composite the channel sum into dL/dalpha is therefore also one thread's, and the
//                per-CTA dL/dbkgd partials go through ssim_bkgd_reduce in a fixed order.
// Planes are indexed along gridDim.x (tile-major inside a plane), so N*C may exceed 65 535.
#include <cmath>

#include "common.cuh"
#include "../../include/surfel_ssim.h"

namespace {

constexpr int SS_T = 32;                 // output tile edge
constexpr int SS_R = 5;                  // window radius (11 taps)
constexpr int SS_S = SS_T + 2 * SS_R;    // staged tile edge, 42
constexpr int SS_THREADS = 256;          // 32 columns x 8 row groups of 4 output rows
constexpr int SS_ROWS = SS_T / (SS_THREADS / SS_T);   // 4
constexpr int SS_REDUCE_THREADS = 1024;
constexpr float SS_C1 = 0.01f * 0.01f, SS_C2 = 0.03f * 0.03f;

struct SsimWin {
    float w[2 * SS_R + 1];
};

// gs/utils/loss_utils.py:24-26 (gaussian(11, 1.5)): float32 of exp(double), divided by their float32 sum.  torch's
// vectorised sum of these 11 values is their exact sum rounded once to float32 (a sequential float32 sum is 1 ulp lower),
// so the sum is taken in double and rounded once.
SsimWin ssim_window() {
    SsimWin g;
    double s = 0.0;
    for (int i = 0; i < 2 * SS_R + 1; i++) {
        g.w[i] = (float)std::exp(-(double)((i - SS_R) * (i - SS_R)) / (2.0 * 1.5 * 1.5));
        s += (double)g.w[i];
    }
    const float sf = (float)s;
    for (int i = 0; i < 2 * SS_R + 1; i++) g.w[i] /= sf;
    return g;
}

struct SsimShape {
    int N, C, H, W, tiles_x, tiles;
    long long alpha_stride;
};

// the image value seen by the loss: img1, or img1 + (1 - alpha) * bkgd[ch] with the background composite
__device__ __forceinline__ float image_x(const float* img1, const float* alpha, const float* bkgd, int ch, size_t p) {
    float x = img1[p];
    if (alpha) x += (1.f - alpha[p]) * __ldg(bkgd + ch);
    return x;
}

// sum of `v` over the CTA (fixed shuffle tree, then the warps in order); valid in thread 0
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                     // `red` may still be read from the previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float t = 0.f;
    if (threadIdx.x == 0)
        for (int w = 0; w < SS_THREADS / 32; w++) t += red[w];
    return t;
}

__global__ void __launch_bounds__(SS_THREADS)
ssim_fwd_kernel(const SsimShape s, const SsimWin win, const float* __restrict__ img1, const float* __restrict__ img2,
                const float* __restrict__ alpha, const float* __restrict__ bkgd, float* __restrict__ partials,
                float* __restrict__ maps) {
    __shared__ float xs[SS_S][SS_S], ys[SS_S][SS_S];
    __shared__ float hs[5][SS_S][SS_T];
    __shared__ float red[SS_THREADS / 32];
    const size_t plane = blockIdx.x / (unsigned)s.tiles;
    const int tile = (int)(blockIdx.x - plane * (unsigned)s.tiles);
    const int n = (int)(plane / (unsigned)s.C), ch = (int)(plane - (size_t)n * s.C);
    const int x0 = (tile % s.tiles_x) * SS_T - SS_R, y0 = (tile / s.tiles_x) * SS_T - SS_R;
    const size_t HW = (size_t)s.H * s.W, base = plane * HW;
    const float* al = alpha ? alpha + (size_t)n * s.alpha_stride : nullptr;
    for (int i = threadIdx.x; i < SS_S * SS_S; i += SS_THREADS) {
        const int r = i / SS_S, c = i - r * SS_S, gy = y0 + r, gx = x0 + c;
        float xv = 0.f, yv = 0.f;
        if (gy >= 0 && gy < s.H && gx >= 0 && gx < s.W) {
            const size_t p = (size_t)gy * s.W + gx;
            xv = image_x(img1 + base, al, bkgd, ch, p);
            yv = img2[base + p];
        }
        xs[r][c] = xv;
        ys[r][c] = yv;
    }
    __syncthreads();
    const int c = threadIdx.x & 31, rg = threadIdx.x >> 5;
    for (int r = rg; r < SS_S; r += SS_THREADS / 32) {
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#pragma unroll
        for (int k = 0; k < 2 * SS_R + 1; k++) {
            const float xv = xs[r][c + k], yv = ys[r][c + k], w = win.w[k];
            a0 = fmaf(w, xv, a0);
            a1 = fmaf(w, yv, a1);
            a2 = fmaf(w, xv * xv, a2);
            a3 = fmaf(w, yv * yv, a3);
            a4 = fmaf(w, xv * yv, a4);
        }
        hs[0][r][c] = a0; hs[1][r][c] = a1; hs[2][r][c] = a2; hs[3][r][c] = a3; hs[4][r][c] = a4;
    }
    __syncthreads();
    float v[5][SS_ROWS];
#pragma unroll
    for (int q = 0; q < 5; q++)
#pragma unroll
        for (int j = 0; j < SS_ROWS; j++) v[q][j] = 0.f;
    const int r0 = rg * SS_ROWS;
#pragma unroll
    for (int k = 0; k < SS_ROWS + 2 * SS_R; k++) {
#pragma unroll
        for (int q = 0; q < 5; q++) {
            const float hv = hs[q][r0 + k][c];
#pragma unroll
            for (int j = 0; j < SS_ROWS; j++)
                if (k - j >= 0 && k - j <= 2 * SS_R) v[q][j] = fmaf(win.w[k - j], hv, v[q][j]);
        }
    }
    float part = 0.f;
    const int gx = x0 + SS_R + c;
#pragma unroll
    for (int j = 0; j < SS_ROWS; j++) {
        const int gy = y0 + SS_R + r0 + j;
        if (gx >= s.W || gy >= s.H) continue;
        const float mu1 = v[0][j], mu2 = v[1][j];
        const float mu1_sq = mu1 * mu1, mu2_sq = mu2 * mu2, mu12 = mu1 * mu2;
        const float s11 = v[2][j] - mu1_sq, s22 = v[3][j] - mu2_sq, s12 = v[4][j] - mu12;
        const float n1 = 2.f * mu12 + SS_C1, n2 = 2.f * s12 + SS_C2;
        const float d1 = mu1_sq + mu2_sq + SS_C1, d2 = s11 + s22 + SS_C2;
        const float den = d1 * d2 + 1e-10f;
        const float m = (n1 * n2) / den;
        part += m;
        if (maps) {
            const float inv = 1.f / den;
            const float dmu1 = (2.f * mu2 * n2 - m * 2.f * mu1 * d2) * inv;
            const float ds11 = -m * d1 * inv;
            const float ds12 = 2.f * n1 * inv;
            const size_t p = base + (size_t)gy * s.W + gx, NP = (size_t)s.N * s.C * HW;
            maps[p] = dmu1 - 2.f * mu1 * ds11 - mu2 * ds12;
            maps[NP + p] = ds11;
            maps[2 * NP + p] = ds12;
        }
    }
    const float t = block_sum(part, red);
    if (threadIdx.x == 0) partials[blockIdx.x] = t;
}

// warp-wide float64 sum of row[0, len) in a fixed order; valid in every lane
__device__ __forceinline__ double warp_row_sum(const float* __restrict__ row, int len) {
    const int lane = threadIdx.x & 31;
    double a = 0.0;
    for (int i = lane; i < len; i += 32) a += (double)row[i];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    return a;
}

__global__ void __launch_bounds__(SS_REDUCE_THREADS)
ssim_reduce_kernel(int N, int row_len, double inv_img, double inv_all, const float* __restrict__ partials,
                   float* __restrict__ ssim_img, float* __restrict__ ssim_mean) {
    __shared__ double red[SS_REDUCE_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    double tot = 0.0;
    for (int n = warp; n < N; n += SS_REDUCE_THREADS / 32) {
        const double a = warp_row_sum(partials + (size_t)n * row_len, row_len);
        if (lane == 0) ssim_img[n] = (float)(a * inv_img);
        tot += a;
    }
    if (lane == 0) red[warp] = tot;
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int w = 0; w < SS_REDUCE_THREADS / 32; w++) t += red[w];
        ssim_mean[0] = (float)(t * inv_all);
    }
}

__global__ void __launch_bounds__(SS_THREADS)
ssim_bwd_kernel(const SsimShape s, const SsimWin win, const float* __restrict__ img1, const float* __restrict__ img2,
                const float* __restrict__ alpha, const float* __restrict__ bkgd, const float* __restrict__ maps,
                const float* __restrict__ dL_dssim, int per_image, float inv_count, float* __restrict__ dL_dimg1,
                int accumulate, float* __restrict__ dL_dalpha, float* __restrict__ bk_partials) {
    __shared__ float ms[3][SS_S][SS_S];
    __shared__ float hs[3][SS_S][SS_T];
    __shared__ float red[SS_THREADS / 32];
    const int n = (int)(blockIdx.x / (unsigned)s.tiles);
    const int tile = (int)(blockIdx.x - (unsigned)n * (unsigned)s.tiles);
    const int x0 = (tile % s.tiles_x) * SS_T - SS_R, y0 = (tile / s.tiles_x) * SS_T - SS_R;
    const size_t HW = (size_t)s.H * s.W, NP = (size_t)s.N * s.C * HW;
    const float* al = alpha ? alpha + (size_t)n * s.alpha_stride : nullptr;
    const float g = __ldg(dL_dssim + (per_image ? n : 0)) * inv_count;
    const int c = threadIdx.x & 31, rg = threadIdx.x >> 5, r0 = rg * SS_ROWS;
    const int gx = x0 + SS_R + c;
    float da[SS_ROWS];
#pragma unroll
    for (int j = 0; j < SS_ROWS; j++) da[j] = 0.f;
    for (int ch = 0; ch < s.C; ch++) {
        const size_t base = ((size_t)n * s.C + ch) * HW;
        __syncthreads();                 // the previous channel's reads of ms / hs are done
        for (int i = threadIdx.x; i < SS_S * SS_S; i += SS_THREADS) {
            const int r = i / SS_S, cc = i - r * SS_S, yy = y0 + r, xx = x0 + cc;
            float a = 0.f, b = 0.f, m = 0.f;
            if (yy >= 0 && yy < s.H && xx >= 0 && xx < s.W) {
                const size_t p = base + (size_t)yy * s.W + xx;
                a = maps[p]; b = maps[NP + p]; m = maps[2 * NP + p];
            }
            ms[0][r][cc] = a; ms[1][r][cc] = b; ms[2][r][cc] = m;
        }
        __syncthreads();
        for (int r = rg; r < SS_S; r += SS_THREADS / 32) {
            float a0 = 0.f, a1 = 0.f, a2 = 0.f;
#pragma unroll
            for (int k = 0; k < 2 * SS_R + 1; k++) {
                const float w = win.w[k];
                a0 = fmaf(w, ms[0][r][c + k], a0);
                a1 = fmaf(w, ms[1][r][c + k], a1);
                a2 = fmaf(w, ms[2][r][c + k], a2);
            }
            hs[0][r][c] = a0; hs[1][r][c] = a1; hs[2][r][c] = a2;
        }
        __syncthreads();
        float v[3][SS_ROWS];
#pragma unroll
        for (int q = 0; q < 3; q++)
#pragma unroll
            for (int j = 0; j < SS_ROWS; j++) v[q][j] = 0.f;
#pragma unroll
        for (int k = 0; k < SS_ROWS + 2 * SS_R; k++) {
#pragma unroll
            for (int q = 0; q < 3; q++) {
                const float hv = hs[q][r0 + k][c];
#pragma unroll
                for (int j = 0; j < SS_ROWS; j++)
                    if (k - j >= 0 && k - j <= 2 * SS_R) v[q][j] = fmaf(win.w[k - j], hv, v[q][j]);
            }
        }
        float bk_part = 0.f;
#pragma unroll
        for (int j = 0; j < SS_ROWS; j++) {
            const int gy = y0 + SS_R + r0 + j;
            if (gx >= s.W || gy >= s.H) continue;
            const size_t p = (size_t)gy * s.W + gx;
            const float x = image_x(img1 + base, al, bkgd, ch, p), y = img2[base + p];
            const float gxv = g * (v[0][j] + 2.f * x * v[1][j] + y * v[2][j]);
            float* d = dL_dimg1 + base + p;
            *d = accumulate ? *d + gxv : gxv;
            if (al) {
                da[j] = fmaf(gxv, __ldg(bkgd + ch), da[j]);
                bk_part += gxv * (1.f - al[p]);
            }
        }
        if (al) {
            const float t = block_sum(bk_part, red);
            if (threadIdx.x == 0) bk_partials[((size_t)n * 3 + ch) * s.tiles + tile] = t;
        }
    }
    if (al) {
        float* dal = dL_dalpha + (size_t)n * s.alpha_stride;
#pragma unroll
        for (int j = 0; j < SS_ROWS; j++) {
            const int gy = y0 + SS_R + r0 + j;
            if (gx < s.W && gy < s.H) dal[(size_t)gy * s.W + gx] -= da[j];
        }
    }
}

// dL_dbkgd[n][ch] += the sum of image n's per-CTA partials of channel ch, in a fixed order
__global__ void __launch_bounds__(SS_REDUCE_THREADS)
ssim_bkgd_reduce_kernel(int rows, int len, const float* __restrict__ bk_partials, float* __restrict__ dL_dbkgd) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = warp; r < rows; r += SS_REDUCE_THREADS / 32) {
        const double a = warp_row_sum(bk_partials + (size_t)r * len, len);
        if (lane == 0) dL_dbkgd[r] += (float)a;
    }
}

struct SsimLayout {
    size_t partials, bk_partials, total;
};

SsimLayout ssim_layout(const SsimShape& s) {
    SsimLayout L;
    size_t o = 0;
    L.partials = o;    o = sr_align_up(o + (size_t)s.N * s.C * s.tiles * sizeof(float));
    L.bk_partials = o; o = sr_align_up(o + (size_t)s.N * 3 * s.tiles * sizeof(float));
    L.total = o;
    return L;
}

// validates the shape (and the grid size it implies); fills `s`
int ssim_shape(const char* who, int32_t N, int32_t C, int32_t H, int32_t W, SsimShape& s) {
    if (N < 1 || C < 1 || H < 1 || W < 1)
        return sr_fail(SR_EINVAL, "%s: N, C, H and W must be >= 1, got %d, %d, %d, %d", who, N, C, H, W);
    s.N = N; s.C = C; s.H = H; s.W = W;
    s.tiles_x = (W + SS_T - 1) / SS_T;
    const long long tiles = (long long)s.tiles_x * ((H + SS_T - 1) / SS_T);
    if (tiles * N * C > 0x7fffffffLL) return sr_fail(SR_EINVAL, "%s: N*C*H*W is too large for one launch", who);
    s.tiles = (int)tiles;
    s.alpha_stride = 0;
    return 0;
}

int ssim_composite(const char* who, const SsimShape& s, const float* alpha, int64_t alpha_stride, const float* bkgd) {
    if (!alpha) return 0;
    if (!bkgd) return sr_fail(SR_EINVAL, "%s: alpha needs bkgd", who);
    if (s.C != 3) return sr_fail(SR_EINVAL, "%s: the background composite needs C = 3, got %d", who, s.C);
    if (alpha_stride < (int64_t)s.H * s.W)
        return sr_fail(SR_EINVAL, "%s: alpha_stride %lld is below H*W = %lld", who, (long long)alpha_stride,
                       (long long)s.H * s.W);
    return 0;
}

}  // namespace

extern "C" {

SR_API int64_t sr_ssim_scratch_bytes(int32_t N, int32_t C, int32_t H, int32_t W) {
    if (N < 1 || C < 1 || H < 1 || W < 1) return -1;
    SsimShape s{N, C, H, W, (W + SS_T - 1) / SS_T, 0, 0};
    s.tiles = s.tiles_x * ((H + SS_T - 1) / SS_T);
    return (int64_t)ssim_layout(s).total;
}

SR_API int sr_ssim_forward(int32_t N, int32_t C, int32_t H, int32_t W, const float* img1, const float* img2,
                           const float* alpha, int64_t alpha_stride, const float* bkgd, float* ssim_img, float* ssim_mean,
                           float* maps, void* scratch, int64_t scratch_bytes, void* stream_) {
    SsimShape s;
    if (int rc = ssim_shape("sr_ssim_forward", N, C, H, W, s)) return rc;
    if (int rc = ssim_composite("sr_ssim_forward", s, alpha, alpha_stride, bkgd)) return rc;
    if (!img1 || !img2 || !ssim_img || !ssim_mean || !scratch)
        return sr_fail(SR_EINVAL, "sr_ssim_forward: img1, img2, ssim_img, ssim_mean and scratch must not be NULL");
    const SsimLayout L = ssim_layout(s);
    if (scratch_bytes < (int64_t)L.total)
        return sr_fail(SR_EINVAL, "sr_ssim_forward: scratch holds fewer bytes than sr_ssim_scratch_bytes(%d, %d, %d, %d)", N, C,
                       H, W);
    s.alpha_stride = alpha ? alpha_stride : 0;
    static const SsimWin win = ssim_window();
    cudaStream_t st = (cudaStream_t)stream_;
    float* partials = (float*)((char*)scratch + L.partials);
    const double pix = (double)H * W;
    {
        ProfileScope ps("ssim_fwd", st);
        ssim_fwd_kernel<<<(unsigned)((size_t)s.tiles * N * C), SS_THREADS, 0, st>>>(s, win, img1, img2, alpha, bkgd, partials, maps);
    }
    {
        ProfileScope ps("ssim_reduce", st);
        ssim_reduce_kernel<<<1, SS_REDUCE_THREADS, 0, st>>>(N, C * s.tiles, 1.0 / (C * pix), 1.0 / ((double)N * C * pix), partials,
                                                          ssim_img, ssim_mean);
    }
    return sr_launched(2, "sr_ssim_forward");
}

SR_API int sr_ssim_backward(int32_t N, int32_t C, int32_t H, int32_t W, const float* img1, const float* img2,
                            const float* alpha, int64_t alpha_stride, const float* bkgd, const float* maps,
                            const float* dL_dssim, int32_t per_image, float* dL_dimg1, int32_t accumulate, float* dL_dalpha,
                            float* dL_dbkgd, void* scratch, int64_t scratch_bytes, void* stream_) {
    SsimShape s;
    if (int rc = ssim_shape("sr_ssim_backward", N, C, H, W, s)) return rc;
    if (int rc = ssim_composite("sr_ssim_backward", s, alpha, alpha_stride, bkgd)) return rc;
    if (per_image != 0 && per_image != 1) return sr_fail(SR_EINVAL, "sr_ssim_backward: per_image must be 0 or 1, got %d", per_image);
    if (accumulate != 0 && accumulate != 1)
        return sr_fail(SR_EINVAL, "sr_ssim_backward: accumulate must be 0 or 1, got %d", accumulate);
    if (!img1 || !img2 || !maps || !dL_dssim || !dL_dimg1 || !scratch)
        return sr_fail(SR_EINVAL, "sr_ssim_backward: img1, img2, maps, dL_dssim, dL_dimg1 and scratch must not be NULL");
    if (alpha && (!dL_dalpha || !dL_dbkgd))
        return sr_fail(SR_EINVAL, "sr_ssim_backward: the background composite needs dL_dalpha and dL_dbkgd");
    const SsimLayout L = ssim_layout(s);
    if (scratch_bytes < (int64_t)L.total)
        return sr_fail(SR_EINVAL, "sr_ssim_backward: scratch holds fewer bytes than sr_ssim_scratch_bytes(%d, %d, %d, %d)", N, C,
                       H, W);
    s.alpha_stride = alpha ? alpha_stride : 0;
    static const SsimWin win = ssim_window();
    cudaStream_t st = (cudaStream_t)stream_;
    float* bk = (float*)((char*)scratch + L.bk_partials);
    const float inv_count = (float)(1.0 / ((per_image ? 1.0 : (double)N) * C * H * W));
    {
        ProfileScope ps("ssim_bwd", st);
        ssim_bwd_kernel<<<(unsigned)((size_t)s.tiles * N), SS_THREADS, 0, st>>>(s, win, img1, img2, alpha, bkgd, maps, dL_dssim,
                                                                             per_image, inv_count, dL_dimg1, accumulate,
                                                                             dL_dalpha, bk);
    }
    if (!alpha) return sr_launched(1, "sr_ssim_backward");
    {
        ProfileScope ps("ssim_bkgd_reduce", st);
        ssim_bkgd_reduce_kernel<<<1, SS_REDUCE_THREADS, 0, st>>>(N * 3, s.tiles, bk, dL_dbkgd);
    }
    return sr_launched(2, "sr_ssim_backward");
}

}  // extern "C"
