// skin_mlp.cu -- the delta-skinning MLP (lab4d/nnutils/skinning.py:104-119) and its gradient (include/surfel_skin_mlp.h).
//
// The reference materialises xyz_bone (M,P,B,3), expands the 160 conditioning channels to every point, concatenates an
// (M,P,3B+160) input and keeps it and both (M,P,64) activations for autograd.  Here the first layer arrives folded into
// one (64,4) table per frame (vidu4d_b200/warp.py delta_skin_tables), so the per-point work is a 3 -> 64 -> 64 -> B MLP:
//   skin_mlp_fwd     a CTA owns tiles of 128 points of one frame.  The weights sit in shared memory, transposed and
//                    permuted so that a thread's output units are one vector load; the activations of a tile sit in
//                    shared memory as [unit][point].  Every layer is a register-tiled GEMM: a thread owns 8 points x 4
//                    units (units tx, tx+16, tx+32, tx+48) and issues 3 shared-memory vector loads per 32 FMAs.
//   skin_mlp_bwd     recomputes the tile's h1, h2, y, then walks back: g_y, g_h2 (written over h2), g_h1 (written over
//                    h1), g_x.  The weight gradients are GEMMs with the points as the inner dimension; each thread keeps
//                    its 4 x 4 (g_W2), NJ x 4 (g_W3) and single (g_F, biases) sums in registers over all the CTA's tiles
//                    and writes them once, to this CTA's slot of the scratch.
//   skin_mlp_reduce  one thread per weight-gradient element sums the CTAs' slots in CTA order (float64, rounded once).
// No float atomics: results are bit-identical from run to run.  The grid is persistent (at most SKM_MAX_CTAS CTAs), so
// the scratch stays a few MB whatever N is.  NJ = ceil(B / 16) of 1..4 is a template parameter: the last layer costs
// 16 NJ units, not 64.
#include "common.cuh"
#include "../../include/surfel_skin_mlp.h"

namespace {

constexpr int SKM_W = 64;                 // hidden width
constexpr int SKM_T = 128;                // points per tile
constexpr int SKM_LD = SKM_T + 4;         // row stride of an activation tile: rows 16 B aligned, 4 banks apart
constexpr int SKM_THREADS = 256;          // 16 unit groups (tx) x 16 point groups (ty) of 8 points
constexpr int SKM_PTS = 8;
constexpr int SKM_MAX_CTAS = 264;         // of the backward: 2 x the 132 SMs of an H100, one CTA resident per SM
constexpr int SKM_FWD_CTAS = 1056;        // of the forward (two CTAs resident per SM)
constexpr int SKM_SHARED_ELEMS = SKM_W * SKM_W + SKM_W;   // g_W2, g_b2; g_W3, g_b3 add B * 65

struct SkmShape {
    int M, N, B, Mt, nj, tiles, cpf;      // cpf: CTAs per frame of the backward
    long long f_stride;                   // floats between consecutive frames' F (0 when shared)
};

__host__ __device__ inline int skm_part_floats(int B) { return B * (SKM_W + 1) + SKM_SHARED_ELEMS + SKM_W * 4; }

template <int NJ>
__device__ __forceinline__ void load_units(const float* p, float (&w)[NJ]) {
    if constexpr (NJ == 4) {
        const float4 v = *reinterpret_cast<const float4*>(p);
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
    } else if constexpr (NJ == 2) {
        const float2 v = *reinterpret_cast<const float2*>(p);
        w[0] = v.x; w[1] = v.y;
    } else {
#pragma unroll
        for (int j = 0; j < NJ; j++) w[j] = p[j];
    }
}

// acc[jj][i] += sum_{k < K} wt[k][tx * NJ + jj] * act[k][p0 + i], k ascending
template <int NJ, int K>
__device__ __forceinline__ void tile_gemm(const float* __restrict__ wt, const float* __restrict__ act, int tx, int p0,
                                          float (&acc)[NJ][SKM_PTS]) {
#pragma unroll 4
    for (int k = 0; k < K; k++) {
        float w[NJ];
        load_units<NJ>(wt + k * 16 * NJ + tx * NJ, w);
        const float4 a0 = *reinterpret_cast<const float4*>(act + k * SKM_LD + p0);
        const float4 a1 = *reinterpret_cast<const float4*>(act + k * SKM_LD + p0 + 4);
        const float a[SKM_PTS] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
        for (int jj = 0; jj < NJ; jj++)
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = fmaf(w[jj], a[i], acc[jj][i]);
    }
}

// row tx + 16 jj of an activation tile, columns p0 .. p0 + 7
__device__ __forceinline__ void store_row(float* tile, int row, int p0, const float (&v)[SKM_PTS]) {
    *reinterpret_cast<float4*>(tile + row * SKM_LD + p0) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(tile + row * SKM_LD + p0 + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

// shared-memory layout, in floats; the backward's extra arrays follow the forward's
template <int NJ>
struct SkmSmem {
    static constexpr int F = 0, b2 = F + SKM_W * 4, b3 = b2 + SKM_W, w2t = b3 + SKM_W, w3t = w2t + SKM_W * SKM_W,
                         xs = w3t + SKM_W * 16 * NJ, h1 = xs + 3 * SKM_T, h2 = h1 + SKM_W * SKM_LD,
                         fwd_total = h2 + SKM_W * SKM_LD;
    static constexpr int w2p = fwd_total, w3p = w2p + SKM_W * SKM_W, gy = w3p + 16 * NJ * SKM_W,
                         bwd_total = gy + 16 * NJ * SKM_LD;
};

// F of the frame, the biases and the transposed, permuted weights: w2t[k][tx*4+jj] = W2[tx+16jj][k],
// w3t[k][tx*NJ+jj] = W3[tx+16jj][k] (0 for a unit >= B)
template <int NJ>
__device__ __forceinline__ void load_weights(float* sm, int B, const float* __restrict__ F, const float* __restrict__ W2,
                                             const float* __restrict__ b2, const float* __restrict__ W3,
                                             const float* __restrict__ b3) {
    using S = SkmSmem<NJ>;
    for (int i = threadIdx.x; i < SKM_W * 4; i += SKM_THREADS) sm[S::F + i] = F[i];
    for (int i = threadIdx.x; i < SKM_W; i += SKM_THREADS) {
        sm[S::b2 + i] = b2[i];
        sm[S::b3 + i] = i < B ? b3[i] : 0.f;
    }
    for (int i = threadIdx.x; i < SKM_W * SKM_W; i += SKM_THREADS) {
        const int j = i >> 6, k = i & 63;
        sm[S::w2t + k * SKM_W + (j & 15) * 4 + (j >> 4)] = W2[i];
    }
    for (int i = threadIdx.x; i < 16 * NJ * SKM_W; i += SKM_THREADS) {
        const int j = i >> 6, k = i & 63;
        sm[S::w3t + k * 16 * NJ + (j & 15) * NJ + (j >> 4)] = j < B ? W3[i] : 0.f;
    }
}

// stages the tile's points as xs[c][p] (0 beyond the frame), then h1 and h2 of the tile; returns y in acc3
template <int NJ>
__device__ __forceinline__ void tile_forward(float* sm, const float* __restrict__ pts, int n0, int cnt, int tx, int p0,
                                             float (&acc3)[NJ][SKM_PTS]) {
    using S = SkmSmem<NJ>;
    for (int i = threadIdx.x; i < 3 * SKM_T; i += SKM_THREADS) {
        const int p = i / 3, c = i - 3 * p;
        sm[S::xs + c * SKM_T + p] = p < cnt ? pts[(size_t)n0 * 3 + i] : 0.f;
    }
    __syncthreads();
    float acc[4][SKM_PTS];
    {
        float x[3][SKM_PTS];
#pragma unroll
        for (int c = 0; c < 3; c++)
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) x[c][i] = sm[S::xs + c * SKM_T + p0 + i];
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
            const float4 f = *reinterpret_cast<const float4*>(sm + S::F + (tx + 16 * jj) * 4);
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++)
                acc[jj][i] = fmaxf(fmaf(f.z, x[2][i], fmaf(f.y, x[1][i], fmaf(f.x, x[0][i], f.w))), 0.f);
            store_row(sm + S::h1, tx + 16 * jj, p0, acc[jj]);
        }
    }
    __syncthreads();
#pragma unroll
    for (int jj = 0; jj < 4; jj++)
#pragma unroll
        for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = sm[S::b2 + tx + 16 * jj];
    tile_gemm<4, SKM_W>(sm + S::w2t, sm + S::h1, tx, p0, acc);
#pragma unroll
    for (int jj = 0; jj < 4; jj++) {
#pragma unroll
        for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = fmaxf(acc[jj][i], 0.f);
        store_row(sm + S::h2, tx + 16 * jj, p0, acc[jj]);
    }
    __syncthreads();
#pragma unroll
    for (int jj = 0; jj < NJ; jj++)
#pragma unroll
        for (int i = 0; i < SKM_PTS; i++) acc3[jj][i] = sm[S::b3 + tx + 16 * jj];
    tile_gemm<NJ, SKM_W>(sm + S::w3t, sm + S::h2, tx, p0, acc3);
}

template <int NJ>
__global__ void __launch_bounds__(SKM_THREADS, 2)
skin_mlp_fwd_kernel(const SkmShape s, const float* __restrict__ points, const float* __restrict__ F,
                    const float* __restrict__ W2, const float* __restrict__ b2, const float* __restrict__ W3,
                    const float* __restrict__ b3, float* __restrict__ delta) {
    extern __shared__ float4 skm_smem[];
    float* sm = reinterpret_cast<float*>(skm_smem);
    const int m = blockIdx.y, tx = threadIdx.x & 15, p0 = (threadIdx.x >> 4) * SKM_PTS;
    load_weights<NJ>(sm, s.B, F + m * s.f_stride, W2, b2, W3, b3);
    const float* pts = points + (size_t)m * s.N * 3;
    float* out = delta + (size_t)m * s.N * s.B;
    for (int tile = blockIdx.x; tile < s.tiles; tile += gridDim.x) {
        const int n0 = tile * SKM_T, cnt = min(SKM_T, s.N - n0);
        float y[NJ][SKM_PTS];
        tile_forward<NJ>(sm, pts, n0, cnt, tx, p0, y);   // its first barrier also orders load_weights before any use
#pragma unroll
        for (int i = 0; i < SKM_PTS; i++) {
            if (p0 + i >= cnt) break;
            float* row = out + (size_t)(n0 + p0 + i) * s.B;
#pragma unroll
            for (int jj = 0; jj < NJ; jj++)
                if (tx + 16 * jj < s.B) row[tx + 16 * jj] = 0.1f * fmaxf(y[jj][i], 0.f);
        }
    }
}

// acc[ii][kk] += sum_p ga[(a + 16 ii)][p] * hb[(c + 16 kk)][p], p ascending over the tile
template <int NI>
__device__ __forceinline__ void outer_acc(const float* __restrict__ ga, const float* __restrict__ hb, int a, int c,
                                          float (&acc)[NI][4]) {
#pragma unroll 2
    for (int p = 0; p < SKM_T; p += 4) {
        float4 g[NI], h[4];
#pragma unroll
        for (int ii = 0; ii < NI; ii++) g[ii] = *reinterpret_cast<const float4*>(ga + (a + 16 * ii) * SKM_LD + p);
#pragma unroll
        for (int kk = 0; kk < 4; kk++) h[kk] = *reinterpret_cast<const float4*>(hb + (c + 16 * kk) * SKM_LD + p);
#pragma unroll
        for (int ii = 0; ii < NI; ii++)
#pragma unroll
            for (int kk = 0; kk < 4; kk++) {
                float v = acc[ii][kk];
                v = fmaf(g[ii].x, h[kk].x, v);
                v = fmaf(g[ii].y, h[kk].y, v);
                v = fmaf(g[ii].z, h[kk].z, v);
                v = fmaf(g[ii].w, h[kk].w, v);
                acc[ii][kk] = v;
            }
    }
}

// sum of one row of an activation tile, p ascending
__device__ __forceinline__ float row_sum(const float* __restrict__ row, float v) {
#pragma unroll 4
    for (int p = 0; p < SKM_T; p += 4) {
        const float4 g = *reinterpret_cast<const float4*>(row + p);
        v += g.x; v += g.y; v += g.z; v += g.w;
    }
    return v;
}

template <int NJ>
__global__ void __launch_bounds__(SKM_THREADS, 1)
skin_mlp_bwd_kernel(const SkmShape s, const float* __restrict__ points, const float* __restrict__ F,
                    const float* __restrict__ W2, const float* __restrict__ b2, const float* __restrict__ W3,
                    const float* __restrict__ b3, const float* __restrict__ g_delta, float* __restrict__ g_points,
                    float* __restrict__ partials) {
    using S = SkmSmem<NJ>;
    extern __shared__ float4 skm_smem[];
    float* sm = reinterpret_cast<float*>(skm_smem);
    const int m = blockIdx.y, tid = threadIdx.x, tx = tid & 15, ty = tid >> 4, p0 = ty * SKM_PTS;
    load_weights<NJ>(sm, s.B, F + m * s.f_stride, W2, b2, W3, b3);
    // the same weights with the input unit permuted: w2p[j][tx*4+kk] = W2[j][tx+16kk], w3p[b][tx*4+kk] = W3[b][tx+16kk]
    for (int i = tid; i < SKM_W * SKM_W; i += SKM_THREADS) {
        const int j = i >> 6, k = i & 63;
        sm[S::w2p + j * SKM_W + (k & 15) * 4 + (k >> 4)] = W2[i];
    }
    for (int i = tid; i < 16 * NJ * SKM_W; i += SKM_THREADS) {
        const int j = i >> 6, k = i & 63;
        sm[S::w3p + j * SKM_W + (k & 15) * 4 + (k >> 4)] = j < s.B ? W3[i] : 0.f;
    }
    const float* pts = points + (size_t)m * s.N * 3;
    const float* gd = g_delta + (size_t)m * s.N * s.B;
    float* gp = g_points + (size_t)m * s.N * 3;
    float aW3[NJ][4], aW2[4][4], ab3 = 0.f, ab2 = 0.f, aF = 0.f;
#pragma unroll
    for (int ii = 0; ii < 4; ii++)
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            aW2[ii][kk] = 0.f;
            if (ii < NJ) aW3[ii][kk] = 0.f;
        }
    float* h1 = sm + S::h1;
    float* h2 = sm + S::h2;
    float* gy = sm + S::gy;
    for (int tile = blockIdx.x; tile < s.tiles; tile += gridDim.x) {
        const int n0 = tile * SKM_T, cnt = min(SKM_T, s.N - n0);
        {
            float y[NJ][SKM_PTS];
            tile_forward<NJ>(sm, pts, n0, cnt, tx, p0, y);
            // g_y = 0.1 g_delta [y > 0]; 0 for a unit >= B or a point beyond the frame, which then adds 0 everywhere
#pragma unroll
            for (int jj = 0; jj < NJ; jj++) {
                const int b = tx + 16 * jj;
#pragma unroll
                for (int i = 0; i < SKM_PTS; i++) {
                    const bool live = b < s.B && p0 + i < cnt && y[jj][i] > 0.f;
                    y[jj][i] = live ? 0.1f * gd[(size_t)(n0 + p0 + i) * s.B + b] : 0.f;
                }
                store_row(gy, b, p0, y[jj]);
            }
        }
        __syncthreads();
        outer_acc<NJ>(gy, h2, ty, tx, aW3);
        if (tid < 16 * NJ) ab3 = row_sum(gy + tid * SKM_LD, ab3);
        float acc[4][SKM_PTS];
#pragma unroll
        for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = 0.f;
        tile_gemm<4, 16 * NJ>(sm + S::w3p, gy, tx, p0, acc);
        __syncthreads();                                  // every read of h2 is done: g_h2 takes its place
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
            float* row = h2 + (tx + 16 * jj) * SKM_LD + p0;
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = row[i] > 0.f ? acc[jj][i] : 0.f;
            store_row(h2, tx + 16 * jj, p0, acc[jj]);
        }
        __syncthreads();
        outer_acc<4>(h2, h1, ty, tx, aW2);
        if (tid < SKM_W) ab2 = row_sum(h2 + tid * SKM_LD, ab2);
#pragma unroll
        for (int jj = 0; jj < 4; jj++)
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = 0.f;
        tile_gemm<4, SKM_W>(sm + S::w2p, h2, tx, p0, acc);
        __syncthreads();                                  // every read of h1 is done: g_h1 takes its place
#pragma unroll
        for (int jj = 0; jj < 4; jj++) {
            float* row = h1 + (tx + 16 * jj) * SKM_LD + p0;
#pragma unroll
            for (int i = 0; i < SKM_PTS; i++) acc[jj][i] = row[i] > 0.f ? acc[jj][i] : 0.f;
            store_row(h1, tx + 16 * jj, p0, acc[jj]);
        }
        __syncthreads();
        {   // g_F[j][c] += sum_p g_h1[j][p] [x; 1][c]
            const int j = tid >> 2, c = tid & 3;
            const float* row = h1 + j * SKM_LD;
            if (c < 3) {
                const float* x = sm + S::xs + c * SKM_T;
#pragma unroll 4
                for (int p = 0; p < SKM_T; p += 4) {
                    const float4 g = *reinterpret_cast<const float4*>(row + p), v = *reinterpret_cast<const float4*>(x + p);
                    aF = fmaf(g.x, v.x, aF); aF = fmaf(g.y, v.y, aF); aF = fmaf(g.z, v.z, aF); aF = fmaf(g.w, v.w, aF);
                }
            } else {
                aF = row_sum(row, aF);
            }
        }
        if (tid < cnt) {                                  // g_x = F[:, 0:3]^T g_h1, one point per thread
            float gx = 0.f, gy_ = 0.f, gz = 0.f;
#pragma unroll 8
            for (int j = 0; j < SKM_W; j++) {
                const float4 f = *reinterpret_cast<const float4*>(sm + S::F + j * 4);
                const float g = h1[j * SKM_LD + tid];
                gx = fmaf(f.x, g, gx); gy_ = fmaf(f.y, g, gy_); gz = fmaf(f.z, g, gz);
            }
            float* o = gp + (size_t)(n0 + tid) * 3;
            o[0] = gx; o[1] = gy_; o[2] = gz;
        }
        __syncthreads();                                  // xs, h1 and gy are rewritten by the next tile
    }
    // this CTA's slot: g_W3 [B][64], g_b3 [B], g_W2 [64][64], g_b2 [64], g_F [64][4]
    float* part = partials + (size_t)(m * gridDim.x + blockIdx.x) * skm_part_floats(s.B);
#pragma unroll
    for (int ii = 0; ii < NJ; ii++)
        if (ty + 16 * ii < s.B)
#pragma unroll
            for (int kk = 0; kk < 4; kk++) part[(ty + 16 * ii) * SKM_W + tx + 16 * kk] = aW3[ii][kk];
    part += s.B * SKM_W;
    if (tid < s.B) part[tid] = ab3;
    part += s.B;
#pragma unroll
    for (int ii = 0; ii < 4; ii++)
#pragma unroll
        for (int kk = 0; kk < 4; kk++) part[(ty + 16 * ii) * SKM_W + tx + 16 * kk] = aW2[ii][kk];
    part += SKM_W * SKM_W;
    if (tid < SKM_W) part[tid] = ab2;
    part += SKM_W;
    part[tid] = aF;
}

// element e of [g_W3 | g_b3 | g_W2 | g_b2] sums every CTA's slot, element e of g_F[m] the slots of frame m's CTAs
__global__ void __launch_bounds__(SKM_THREADS)
skin_mlp_reduce_kernel(const SkmShape s, const float* __restrict__ partials, float* __restrict__ g_F, float* __restrict__ g_W2,
                       float* __restrict__ g_b2, float* __restrict__ g_W3, float* __restrict__ g_b3) {
    const int shared = s.B * (SKM_W + 1) + SKM_SHARED_ELEMS, part = skm_part_floats(s.B);
    const int e = blockIdx.x * SKM_THREADS + threadIdx.x;
    if (e >= shared + s.M * SKM_W * 4) return;
    int first = 0, n = s.M * s.cpf, idx = e;
    if (e >= shared) {
        const int fm = (e - shared) / (SKM_W * 4);
        first = fm * s.cpf; n = s.cpf; idx = shared + (e - shared) % (SKM_W * 4);
    }
    double a = 0.0;
    for (int c = 0; c < n; c++) a += (double)partials[(size_t)(first + c) * part + idx];
    const float v = (float)a;
    if (e >= shared) g_F[e - shared] = v;
    else if (e < s.B * SKM_W) g_W3[e] = v;
    else if (e < s.B * (SKM_W + 1)) g_b3[e - s.B * SKM_W] = v;
    else if (e < s.B * (SKM_W + 1) + SKM_W * SKM_W) g_W2[e - s.B * (SKM_W + 1)] = v;
    else g_b2[e - s.B * (SKM_W + 1) - SKM_W * SKM_W] = v;
}

// validates the shape; fills `s`.  One table for every frame makes the frames one frame of M * N points.
int skm_shape(const char* who, int32_t M, int32_t N, int32_t B, int32_t Mt, int32_t width, int32_t depth, SkmShape& s) {
    if (width != SKM_W || depth != 2)
        return sr_fail(SR_EINVAL, "%s: only width = %d hidden units and depth = 2 hidden layers are implemented, got %d and %d",
                       who, SKM_W, width, depth);
    if (B < 1 || B > 64) return sr_fail(SR_EINVAL, "%s: B must be in [1, 64], got %d", who, B);
    if (M < 1 || M > 65535 || N < 1) return sr_fail(SR_EINVAL, "%s: M must be in [1, 65535] and N >= 1, got %d and %d", who, M, N);
    if ((long long)M * N > 0x7fffffffLL) return sr_fail(SR_EINVAL, "%s: M * N = %lld is too large for one call", who, (long long)M * N);
    if (Mt != 1 && Mt != M) return sr_fail(SR_EINVAL, "%s: Mt must be 1 or M = %d, got %d", who, M, Mt);
    s.M = Mt == 1 ? 1 : M;
    s.N = Mt == 1 ? M * N : N;
    s.B = B; s.Mt = Mt;
    s.nj = (B + 15) / 16;
    s.tiles = (s.N + SKM_T - 1) / SKM_T;
    const int per_frame = SKM_MAX_CTAS / s.M > 1 ? SKM_MAX_CTAS / s.M : 1;
    s.cpf = s.tiles < per_frame ? s.tiles : per_frame;
    s.f_stride = s.M > 1 ? SKM_W * 4 : 0;
    return 0;
}

template <int NJ>
int skm_forward(const SkmShape& s, const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                const float* b3, float* delta, cudaStream_t st) {
    const size_t smem = (size_t)SkmSmem<NJ>::fwd_total * sizeof(float);
    CK(sr_opt_in_smem(skin_mlp_fwd_kernel<NJ>, smem), "sr_delta_skin_forward");
    const int per_frame = SKM_FWD_CTAS / s.M > 1 ? SKM_FWD_CTAS / s.M : 1;
    const dim3 grid((unsigned)(s.tiles < per_frame ? s.tiles : per_frame), (unsigned)s.M);
    ProfileScope ps("skin_mlp_fwd", st);
    skin_mlp_fwd_kernel<NJ><<<grid, SKM_THREADS, smem, st>>>(s, points, F, W2, b2, W3, b3, delta);
    return 0;
}

template <int NJ>
int skm_backward(const SkmShape& s, const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                 const float* b3, const float* g_delta, float* g_points, float* partials, cudaStream_t st) {
    const size_t smem = (size_t)SkmSmem<NJ>::bwd_total * sizeof(float);
    CK(sr_opt_in_smem(skin_mlp_bwd_kernel<NJ>, smem), "sr_delta_skin_backward");
    ProfileScope ps("skin_mlp_bwd", st);
    skin_mlp_bwd_kernel<NJ><<<dim3((unsigned)s.cpf, (unsigned)s.M), SKM_THREADS, smem, st>>>(s, points, F, W2, b2, W3, b3, g_delta,
                                                                                           g_points, partials);
    return 0;
}

int64_t skm_scratch_bytes(const SkmShape& s) { return (int64_t)s.M * s.cpf * skm_part_floats(s.B) * (int64_t)sizeof(float); }

}  // namespace

extern "C" {

SR_API int64_t sr_delta_skin_scratch_bytes(int32_t M, int32_t N, int32_t B) {
    if (B < 1 || B > 64 || M < 1 || M > 65535 || N < 1 || (long long)M * N > 0x7fffffffLL) return -1;
    SkmShape shared, per_frame;
    skm_shape("sr_delta_skin_scratch_bytes", M, N, B, 1, SKM_W, 2, shared);
    skm_shape("sr_delta_skin_scratch_bytes", M, N, B, M, SKM_W, 2, per_frame);
    const int64_t a = skm_scratch_bytes(shared), b = skm_scratch_bytes(per_frame);
    return a > b ? a : b;
}

SR_API int sr_delta_skin_forward(int32_t M, int32_t N, int32_t B, int32_t Mt, int32_t width, int32_t depth,
                                 const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                                 const float* b3, float* delta, void* stream_) {
    SkmShape s;
    if (int rc = skm_shape("sr_delta_skin_forward", M, N, B, Mt, width, depth, s)) return rc;
    if (!points || !F || !W2 || !b2 || !W3 || !b3 || !delta)
        return sr_fail(SR_EINVAL, "sr_delta_skin_forward: points, F, W2, b2, W3, b3 and delta must not be NULL");
    cudaStream_t st = (cudaStream_t)stream_;
    int rc = 0;
    switch (s.nj) {
        case 1: rc = skm_forward<1>(s, points, F, W2, b2, W3, b3, delta, st); break;
        case 2: rc = skm_forward<2>(s, points, F, W2, b2, W3, b3, delta, st); break;
        case 3: rc = skm_forward<3>(s, points, F, W2, b2, W3, b3, delta, st); break;
        default: rc = skm_forward<4>(s, points, F, W2, b2, W3, b3, delta, st); break;
    }
    if (rc) return rc;
    return sr_launched(1, "sr_delta_skin_forward");
}

SR_API int sr_delta_skin_backward(int32_t M, int32_t N, int32_t B, int32_t Mt, int32_t width, int32_t depth,
                                  const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                                  const float* b3, const float* g_delta, float* g_points, float* g_F, float* g_W2,
                                  float* g_b2, float* g_W3, float* g_b3, void* scratch, int64_t scratch_bytes,
                                  void* stream_) {
    SkmShape s;
    if (int rc = skm_shape("sr_delta_skin_backward", M, N, B, Mt, width, depth, s)) return rc;
    if (!points || !F || !W2 || !b2 || !W3 || !b3 || !g_delta || !g_points || !g_F || !g_W2 || !g_b2 || !g_W3 || !g_b3 || !scratch)
        return sr_fail(SR_EINVAL, "sr_delta_skin_backward: no input, gradient output or scratch pointer may be NULL");
    if (scratch_bytes < skm_scratch_bytes(s))
        return sr_fail(SR_EINVAL, "sr_delta_skin_backward: scratch holds fewer bytes than sr_delta_skin_scratch_bytes(%d, %d, %d)",
                       M, N, B);
    cudaStream_t st = (cudaStream_t)stream_;
    float* partials = (float*)scratch;
    int rc = 0;
    switch (s.nj) {
        case 1: rc = skm_backward<1>(s, points, F, W2, b2, W3, b3, g_delta, g_points, partials, st); break;
        case 2: rc = skm_backward<2>(s, points, F, W2, b2, W3, b3, g_delta, g_points, partials, st); break;
        case 3: rc = skm_backward<3>(s, points, F, W2, b2, W3, b3, g_delta, g_points, partials, st); break;
        default: rc = skm_backward<4>(s, points, F, W2, b2, W3, b3, g_delta, g_points, partials, st); break;
    }
    if (rc) return rc;
    {
        ProfileScope ps("skin_mlp_reduce", st);
        const int elems = s.B * (SKM_W + 1) + SKM_SHARED_ELEMS + s.M * SKM_W * 4;
        skin_mlp_reduce_kernel<<<(elems + SKM_THREADS - 1) / SKM_THREADS, SKM_THREADS, 0, st>>>(s, partials, g_F, g_W2, g_b2, g_W3,
                                                                                              g_b3);
    }
    return sr_launched(2, "sr_delta_skin_backward");
}

}  // extern "C"
