// mask_loss.cu -- Stage 3's silhouette loss as the reference weighs it (include/surfel_mask_loss.h, DESIGN.md 3.5e).
//
// The balance weights need batch-wide sums before any v can be formed, and the positive mean needs a batch-wide count
// after every v is known, so the term takes three launches on the 32x8 pixel tiles of loss_grad_kernel (loss.cu):
//   mask_stats       the five sums of get_mask_balance_wt; the last CTA to finish turns the per-CTA float64 partials,
//                    summed in a fixed order, into pos_wt, neg_wt and the branch flag.
//   mask_loss        v and the unscaled dv/dacc per pixel, and per CTA the sum of v > 0, the sum of all v and the count
//                    of v > 0; the last CTA forms each frame's sums, the batch count C and the gradient scale.
//   mask_loss_scale  dL/dalpha += scale * dv/dacc (where v > 0 when C > 0, everywhere otherwise).
// "Last CTA" is an integer atomic ticket after a __threadfence; the tickets are zeroed by a memset at the start of the
// call.  No float atomics: results are bit-identical from run to run.
#include "common.cuh"
#include "../../include/surfel_mask_loss.h"

namespace {

constexpr int ML_THREADS = 256;          // 32 x 8 pixels
constexpr int ML_STATS = 5;              // float64 partials per CTA: sum vd, sum m [vd > 0], sum (1 - m) [vd > 0], sum m, sum (1 - m)

struct MaskShape {
    int M, W, H, tiles_x, tiles;         // tiles per frame
    long long alpha_stride;
};

// the state the passes hand each other, at the start of the scratch
struct MaskState {
    unsigned int ticket[2];              // CTAs done in mask_stats / mask_loss (zeroed by the launcher)
    float scale;                         // w / C, or w / (M H W) when C = 0
    int all;                             // 1 when C = 0: every pixel receives gradient
};

struct MaskLayout {
    size_t partials, dv, on, total;
};

MaskLayout mask_layout(const MaskShape& s) {
    MaskLayout L;
    const size_t px = (size_t)s.M * s.W * s.H;
    size_t o = sr_align_up(sizeof(MaskState));
    L.partials = o; o = sr_align_up(o + (size_t)s.M * s.tiles * ML_STATS * sizeof(double));
    L.dv = o;       o = sr_align_up(o + px * sizeof(float));
    L.on = o;       o = sr_align_up(o + px);
    L.total = o;
    return L;
}

// sum of `v` over the CTA in a fixed order (shuffle tree, then the warps in order); valid in thread 0
__device__ __forceinline__ double block_sum(double v, double* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();                     // `red` may still be read from the previous call
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < ML_THREADS / 32; w++) t += red[w];
    return t;
}

// after thread 0 has written this CTA's partials: true in every thread of the CTA that finishes last
__device__ __forceinline__ bool last_cta(unsigned int* ticket, unsigned int n_ctas) {
    __shared__ bool last;
    if (threadIdx.x == 0) {
        __threadfence();
        last = atomicAdd(ticket, 1u) == n_ctas - 1;
    }
    __syncthreads();
    if (last) __threadfence();
    return last;
}

__device__ __forceinline__ int cta_index() {
    return ((int)blockIdx.z * (int)gridDim.y + (int)blockIdx.y) * (int)gridDim.x + (int)blockIdx.x;
}

__global__ void __launch_bounds__(ML_THREADS)
mask_stats_kernel(const MaskShape s, const float* __restrict__ mask, const float* __restrict__ vis2d,
                  const float* __restrict__ is_detected, MaskState* __restrict__ st, double* __restrict__ partials,
                  float* __restrict__ balance) {
    __shared__ double red[ML_THREADS / 32];
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    double t[ML_STATS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    if (x < s.W && y < s.H) {
        const size_t p = (size_t)f * s.W * s.H + (size_t)y * s.W + x;
        const float m = mask[p], n = __fsub_rn(1.f, m);
        const float vd = __fmul_rn(vis2d ? vis2d[p] : 1.f, is_detected ? __ldg(is_detected + f) : 1.f);
        t[0] = vd;
        if (vd > 0.f) { t[1] = m; t[2] = n; }
        t[3] = m;
        t[4] = n;
    }
    const int cta = cta_index();
#pragma unroll
    for (int k = 0; k < ML_STATS; k++) {
        const double b = block_sum(t[k], red);
        if (threadIdx.x == 0) partials[(size_t)cta * ML_STATS + k] = b;
    }
    const unsigned int n_ctas = gridDim.x * gridDim.y * gridDim.z;
    if (!last_cta(&st->ticket[0], n_ctas)) return;
    double a[ML_STATS] = {0.0, 0.0, 0.0, 0.0, 0.0};
    for (unsigned int i = threadIdx.x; i < n_ctas; i += ML_THREADS)
#pragma unroll
        for (int k = 0; k < ML_STATS; k++) a[k] += __ldcg(partials + (size_t)i * ML_STATS + k);
#pragma unroll
    for (int k = 0; k < ML_STATS; k++) a[k] = block_sum(a[k], red);
    if (threadIdx.x == 0) {
        // the reference's fp32 sums (exact for binary masks), then its fp32 divisions: inf or NaN where torch gives them
        const float s_vd = (float)a[0], s_pos = (float)a[1], s_neg = (float)a[2];
        balance[0] = __fdiv_rn(s_vd, s_pos);
        balance[1] = __fdiv_rn(s_vd, s_neg);
        balance[2] = ((float)a[3] > 0.f && (float)a[4] > 0.f) ? 1.f : 0.f;
    }
}

__global__ void __launch_bounds__(ML_THREADS)
mask_loss_kernel(const MaskShape s, const float* __restrict__ alpha, const float* __restrict__ mask,
                 const float* __restrict__ vis2d, const float* __restrict__ is_detected, const float* __restrict__ weight,
                 const float* __restrict__ balance, MaskState* __restrict__ st, double* __restrict__ partials,
                 float* __restrict__ dv, uint8_t* __restrict__ on, float* __restrict__ terms, int32_t* __restrict__ counts) {
    __shared__ double red[ML_THREADS / 32];
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    double vpos = 0.0, vall = 0.0, cnt = 0.0;
    if (x < s.W && y < s.H) {
        const size_t q = (size_t)y * s.W + x, p = (size_t)f * s.W * s.H + q;
        const float m = mask[p], vis = vis2d ? vis2d[p] : 1.f, det = is_detected ? __ldg(is_detected + f) : 1.f;
        // bw = 0.5 * pos_wt * mask + 0.5 * neg_wt * (1 - mask), evaluated left to right as torch does
        const float bw = __ldg(balance + 2) != 0.f
                             ? __fadd_rn(__fmul_rn(__fmul_rn(0.5f, __ldg(balance)), m),
                                         __fmul_rn(__fmul_rn(0.5f, __ldg(balance + 1)), __fsub_rn(1.f, m)))
                             : 1.f;
        const float d = __fsub_rn(alpha[(size_t)f * s.alpha_stride + q], m);
        const float v = __fmul_rn(__fmul_rn(__fmul_rn(__fmul_rn(d, d), bw), vis), det);
        // dv/dacc in the order autograd applies the factors: is_detected, vis2d, bw, then pow's 2 (acc - mask)
        dv[p] = __fmul_rn(__fmul_rn(__fmul_rn(det, vis), bw), __fmul_rn(2.f, d));
        const bool pos = v > 0.f;        // false for NaN: v[v > 0] drops it
        on[p] = pos;
        vpos = pos ? v : 0.0;
        vall = v;
        cnt = pos;
    }
    const int cta = cta_index();
    const double b0 = block_sum(vpos, red), b1 = block_sum(vall, red), b2 = block_sum(cnt, red);
    if (threadIdx.x == 0) {
        double* pt = partials + (size_t)cta * ML_STATS;
        pt[0] = b0; pt[1] = b1; pt[2] = b2;
    }
    const unsigned int n_ctas = gridDim.x * gridDim.y * gridDim.z;
    if (!last_cta(&st->ticket[1], n_ctas)) return;
    // each frame's three sums, a warp per frame, in a fixed order; the frames' totals in order in thread 0
    __shared__ unsigned long long c_all;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) c_all = 0ull;
    __syncthreads();
    for (int m0 = 0; m0 < s.M; m0 += ML_THREADS / 32) {
        const int m = m0 + warp;
        double a0 = 0.0, a1 = 0.0, a2 = 0.0;
        if (m < s.M)
            for (int i = lane; i < s.tiles; i += 32) {
                const double* pt = partials + ((size_t)m * s.tiles + i) * ML_STATS;
                a0 += __ldcg(pt); a1 += __ldcg(pt + 1); a2 += __ldcg(pt + 2);
            }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            a0 += __shfl_xor_sync(0xffffffffu, a0, o);
            a1 += __shfl_xor_sync(0xffffffffu, a1, o);
            a2 += __shfl_xor_sync(0xffffffffu, a2, o);
        }
        if (m < s.M && lane == 0) {
            // the frame's sums stay in the first slots of its first tile until the scale is known
            double* pt = partials + (size_t)m * s.tiles * ML_STATS;
            pt[3] = a0; pt[4] = a1;
            counts[m] = (int32_t)a2;
            atomicAdd(&c_all, (unsigned long long)a2);     // an integer sum: order-free
        }
    }
    __syncthreads();
    const unsigned long long C = c_all;
    const float w = __ldg(weight);
    // torch's mean backward: w / count in fp32
    const float scale = C > 0 ? __fdiv_rn(w, (float)C) : __fdiv_rn(w, (float)((double)s.M * s.W * s.H));
    const double inv = C > 0 ? (double)w / (double)C : (double)w / ((double)s.M * s.W * s.H);
    for (int m = threadIdx.x; m < s.M; m += ML_THREADS) {
        const double* pt = partials + (size_t)m * s.tiles * ML_STATS;
        terms[m] = (float)((C > 0 ? pt[3] : pt[4]) * inv);
    }
    if (threadIdx.x == 0) {
        st->scale = scale;
        st->all = C == 0;
    }
}

__global__ void __launch_bounds__(ML_THREADS)
mask_loss_scale_kernel(const MaskShape s, const MaskState* __restrict__ st, const float* __restrict__ dv,
                       const uint8_t* __restrict__ on, float* __restrict__ dL_dalpha) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (x >= s.W || y >= s.H) return;
    const size_t q = (size_t)y * s.W + x, p = (size_t)f * s.W * s.H + q;
    // with C > 0, a pixel with v <= 0 (or NaN) gets nothing at all: the index backward of v[v > 0] leaves it out
    if (!st->all && !on[p]) return;
    float* g = dL_dalpha + (size_t)f * s.alpha_stride + q;
    *g = __fadd_rn(*g, __fmul_rn(st->scale, dv[p]));
}

int mask_shape(const char* who, int32_t M, int32_t W, int32_t H, MaskShape& s) {
    if (M < 1 || W < 1 || H < 1) return sr_fail(SR_EINVAL, "%s: M, W and H must be >= 1, got %d, %d, %d", who, M, W, H);
    if (M > 65535) return sr_fail(SR_EINVAL, "%s: M must be <= 65535, got %d", who, M);
    if ((H + 7) / 8 > 65535) return sr_fail(SR_EINVAL, "%s: H must be <= 524280, got %d", who, H);
    s.M = M; s.W = W; s.H = H;
    s.tiles_x = (W + 31) / 32;
    const long long tiles = (long long)s.tiles_x * ((H + 7) / 8);
    if (tiles * M > 0x7fffffffLL) return sr_fail(SR_EINVAL, "%s: M*H*W is too large for one launch", who);
    s.tiles = (int)tiles;
    s.alpha_stride = 0;
    return 0;
}

}  // namespace

extern "C" {

SR_API int64_t sr_mask_loss_scratch_bytes(int32_t M, int32_t W, int32_t H) {
    if (M < 1 || W < 1 || H < 1 || M > 65535 || (H + 7) / 8 > 65535) return -1;
    MaskShape s{M, W, H, (W + 31) / 32, 0, 0};
    const long long tiles = (long long)s.tiles_x * ((H + 7) / 8);
    if (tiles * M > 0x7fffffffLL) return -1;
    s.tiles = (int)tiles;
    return (int64_t)mask_layout(s).total;
}

SR_API int sr_mask_loss_batch(int32_t M, int32_t W, int32_t H, const float* alpha, int64_t alpha_stride,
                              const float* mask_gt, const float* vis2d, const float* is_detected, const float* weight,
                              float* terms, int32_t* counts, float* balance, float* dL_dalpha, void* scratch,
                              int64_t scratch_bytes, void* stream_) {
    static const char* who = "sr_mask_loss_batch";
    MaskShape s;
    if (int rc = mask_shape(who, M, W, H, s)) return rc;
    if (alpha_stride < (int64_t)W * H)
        return sr_fail(SR_EINVAL, "%s: alpha_stride %lld is below H*W = %lld", who, (long long)alpha_stride, (long long)W * H);
    if (!alpha || !mask_gt || !weight || !dL_dalpha)
        return sr_fail(SR_EINVAL, "%s: alpha, mask_gt, weight and dL_dalpha must not be NULL", who);
    if (!terms || !counts || !balance)
        return sr_fail(SR_EINVAL, "%s: the outputs terms, counts and balance must not be NULL", who);
    if (!scratch) return sr_fail(SR_EINVAL, "%s: scratch must not be NULL", who);
    if ((uintptr_t)scratch % 256)
        return sr_fail(SR_EINVAL, "%s: scratch must be 256-byte aligned", who);
    const MaskLayout L = mask_layout(s);
    if (scratch_bytes < (int64_t)L.total)
        return sr_fail(SR_EINVAL, "%s: scratch holds %lld bytes, fewer than sr_mask_loss_scratch_bytes(%d, %d, %d) = %lld", who,
                       (long long)scratch_bytes, M, W, H, (long long)L.total);
    s.alpha_stride = alpha_stride;
    cudaStream_t st = (cudaStream_t)stream_;
    char* sc = (char*)scratch;
    MaskState* state = (MaskState*)sc;
    double* partials = (double*)(sc + L.partials);
    float* dv = (float*)(sc + L.dv);
    uint8_t* on = (uint8_t*)(sc + L.on);
    const dim3 grid((unsigned)s.tiles_x, (unsigned)((H + 7) / 8), (unsigned)M);
    CK(cudaMemsetAsync(state, 0, sizeof(MaskState), st), "sr_mask_loss_batch: memset(tickets)");
    {
        ProfileScope ps("mask_stats", st);
        mask_stats_kernel<<<grid, ML_THREADS, 0, st>>>(s, mask_gt, vis2d, is_detected, state, partials, balance);
    }
    {
        ProfileScope ps("mask_loss", st);
        mask_loss_kernel<<<grid, ML_THREADS, 0, st>>>(s, alpha, mask_gt, vis2d, is_detected, weight, balance, state, partials,
                                                     dv, on, terms, counts);
    }
    {
        ProfileScope ps("mask_loss_scale", st);
        mask_loss_scale_kernel<<<grid, ML_THREADS, 0, st>>>(s, state, dv, on, dL_dalpha);
    }
    return sr_launched(3, who);
}

}  // extern "C"
