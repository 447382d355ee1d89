// preprocess.cu -- per-surfel forward stage: cull, tangent-plane homography T, projected AABB,
// tile rectangle, SH -> RGB; then the tile-count scan and (tile|depth) key emission.
//
// Replaces (behaviour, not code) of the reference:
//   preprocessCUDA            RAST/cuda_rasterizer/forward.cu:166-260
//   computeTransMat           RAST/cuda_rasterizer/forward.cu:75-128
//   computeAABB               RAST/cuda_rasterizer/forward.cu:133-163
//   computeColorFromSH        RAST/cuda_rasterizer/forward.cu:20-71
//   in_frustum / getRect      RAST/cuda_rasterizer/auxiliary.h:160-185, 64-74
//   InclusiveSum              RAST/cuda_rasterizer/rasterizer_impl.cu:278
//   duplicateWithKeys         RAST/cuda_rasterizer/rasterizer_impl.cu:70-111
//   checkFrustum              RAST/cuda_rasterizer/rasterizer_impl.cu:54-66
//
// Bit-exact binning: every float operation that feeds the radius / tile rectangle / depth key is
// written with explicit-rounding intrinsics (__fmaf_rn/__fmul_rn/__fadd_rn) in exactly the
// contraction pattern of the reference's sm_100a SASS (DESIGN.md "FMA map"), so tile assignment and
// sort keys are identical to the reference build, not merely close.
#include "common.cuh"
#include "surfel_geom.cuh"

namespace {

__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float ff(float a, float b, float c) { return __fmaf_rn(a, b, c); }

__constant__ float kSH_C0 = 0.28209479177387814f;
__constant__ float kSH_C1 = 0.4886025119029199f;
__constant__ float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                -1.0925484305920792f, 0.5462742152960396f};
__constant__ float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                -0.5900435899266435f};

// the view transform and the rotation matrix: one copy in surfel_geom.cuh, shared with the tracking kernel
using sgeo::View;
using sgeo::load_view;
using sgeo::view_z;
using sgeo::w_mul;
using sgeo::rot_matrix;

// auxiliary.h:64-74: one copy in common.cuh, shared with the deterministic backward's emission index
__device__ __forceinline__ void get_rect(float px, float py, int max_radius, int gx, int gy, uint2& rmin, uint2& rmax) {
    sr_tile_rect(px, py, max_radius, gx, gy, rmin, rmax);
}

// forward.cu:20-71.  No binning decision depends on the colour, so this is not written with explicit-rounding
// intrinsics; it mirrors the reference's expression tree and lets nvcc contract it -- which reproduces the reference
// build's bits ONLY while the compiler sees the function in isolation: inlined into the batched kernel, 9 more
// multiply-adds were fused and 0.1 % of the pixels moved by one ulp (r2b).  Hence __noinline__: the call costs nothing
// next to the 48 coefficient loads, and the colour planes stay bit-identical to the reference (tests assert it).
__device__ __noinline__ float3 sh_to_rgb(int deg, int M, float3 pos, const float* __restrict__ campos,
                                            const float* sh, uint32_t& clamped) {
    float dx = pos.x - __ldg(campos), dy = pos.y - __ldg(campos + 1), dz = pos.z - __ldg(campos + 2);
    float len = sqrtf(dx * dx + dy * dy + dz * dz);
    float x = dx / len, y = dy / len, z = dz / len;
    float r[3];
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        float v = kSH_C0 * sh[ch];
        if (deg > 0) {
            v = v - kSH_C1 * y * sh[3 + ch] + kSH_C1 * z * sh[6 + ch] - kSH_C1 * x * sh[9 + ch];
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                v = v + kSH_C2[0] * xy * sh[12 + ch] + kSH_C2[1] * yz * sh[15 + ch] +
                    kSH_C2[2] * (2.0f * zz - xx - yy) * sh[18 + ch] + kSH_C2[3] * xz * sh[21 + ch] +
                    kSH_C2[4] * (xx - yy) * sh[24 + ch];
                if (deg > 2) {
                    v = v + kSH_C3[0] * y * (3.0f * xx - yy) * sh[27 + ch] + kSH_C3[1] * xy * z * sh[30 + ch] +
                        kSH_C3[2] * y * (4.0f * zz - xx - yy) * sh[33 + ch] +
                        kSH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36 + ch] +
                        kSH_C3[4] * x * (4.0f * zz - xx - yy) * sh[39 + ch] +
                        kSH_C3[5] * z * (xx - yy) * sh[42 + ch] + kSH_C3[6] * x * (xx - 3.0f * yy) * sh[45 + ch];
                }
            }
        }
        v += 0.5f;
        if (v < 0.f) clamped |= 1u << ch;
        r[ch] = fmaxf(v, 0.0f);
    }
    return make_float3(r[0], r[1], r[2]);
}

// Conservative pixel bounding box of everything this surfel can contribute to (alpha >= 1/255),
// used only to SKIP pair evaluations inside the composite kernels (never to change a result).
// A pixel contributes iff min(rho3d, rho2d) <= rho_cut = 2 ln(255 * opacity).
//   rho2d <= rho_cut : disc of radius sqrt(rho_cut/2) about the box centre `xy`
//   rho3d <= rho_cut : image of the tangent-plane disc u^2+v^2 <= rho_cut; its exact pixel bbox is
//                      the same closed form as computeAABB with f = (c2, c2, -1)
// evaluated in double with a generous pad for fp32 evaluation noise in the composite.
__device__ __forceinline__ void cull_bbox(const float* T, float cx, float cy, float opac, int W, int H,
                                          uint32_t& bx, uint32_t& by) {
    const uint32_t EMPTY = 1u;                    // x0 = 1 > x1 = 0
    bx = EMPTY; by = EMPTY;
    if (opac < 1.0f / 255.0f) return;             // alpha <= opacity < 1/255 for every pixel (NaN falls through: no cull)
    double c2 = 2.0 * log(255.0 * (double)opac);
    c2 = c2 * 1.004 + 1e-3;
    double x0, x1, y0, y1;
    const double Twx = T[6], Twy = T[7], Twz = T[8];
    const double Dc = c2 * (Twx * Twx + Twy * Twy) - Twz * Twz;
    if (Dc < 0.0) {
        const double inv = 1.0 / Dc;
        const double f0 = c2 * inv, f2 = -inv;
        const double pcx = f0 * ((double)T[0] * Twx + (double)T[1] * Twy) + f2 * ((double)T[2] * Twz);
        const double pcy = f0 * ((double)T[3] * Twx + (double)T[4] * Twy) + f2 * ((double)T[5] * Twz);
        const double qx = f0 * ((double)T[0] * T[0] + (double)T[1] * T[1]) + f2 * ((double)T[2] * T[2]);
        const double qy = f0 * ((double)T[3] * T[3] + (double)T[4] * T[4]) + f2 * ((double)T[5] * T[5]);
        double ex = sqrt(fmax(0.0, pcx * pcx - qx)), ey = sqrt(fmax(0.0, pcy * pcy - qy));
        ex = ex * 1.004 + 0.1; ey = ey * 1.004 + 0.1;
        x0 = pcx - ex; x1 = pcx + ex; y0 = pcy - ey; y1 = pcy + ey;
    } else {                                      // level set is not a bounded ellipse: do not cull
        x0 = y0 = -1e30; x1 = y1 = 1e30;
    }
    const double r2 = sqrt(0.5 * c2) + 0.1;
    x0 = fmin(x0, (double)cx - r2); x1 = fmax(x1, (double)cx + r2);
    y0 = fmin(y0, (double)cy - r2); y1 = fmax(y1, (double)cy + r2);
    // pixel i has its centre at i + 0.5
    const double fx0 = fmax(0.0, ceil(x0 - 0.5)), fx1 = fmin((double)(W - 1), floor(x1 - 0.5));
    const double fy0 = fmax(0.0, ceil(y0 - 0.5)), fy1 = fmin((double)(H - 1), floor(y1 - 0.5));
    if (!(fx0 <= fx1) || !(fy0 <= fy1)) return;
    bx = (uint32_t)fx0 | ((uint32_t)fx1 << 16);
    by = (uint32_t)fy0 | ((uint32_t)fy1 << 16);
}

// The block's SH coefficients (rows x 3M floats, contiguous) are staged in shared memory with coalesced 128-bit loads;
// each thread then reads its own padded row (stride 3M+1: conflict-free) instead of 48 scalar loads at a 192-byte lane
// stride.
__device__ __forceinline__ void stage_sh(float* shbuf, const float* __restrict__ gsrc, int rows, int M3) {
    const int stride = M3 + 1, total = rows * M3;
    if ((M3 & 3) == 0) {
        const float4* g4 = reinterpret_cast<const float4*>(gsrc);
        for (int i = threadIdx.x; i < total / 4; i += 256) {
            const float4 v = __ldg(g4 + i);
            const int e = i * 4, r = e / M3, col = e - r * M3;
            float* d = shbuf + r * stride + col;
            d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
    } else {
        for (int i = threadIdx.x; i < total; i += 256) { const int r = i / M3; shbuf[r * stride + (i - r * M3)] = __ldg(gsrc + i); }
    }
}

// One thread owns one surfel for every frame of the batch (grid = ceil(P/256) blocks).  An input whose frame stride is 0
// is shared by all frames and is read once per launch: at the headline the SH table alone is larger than L2, so a
// per-frame block grid re-read it from HBM for every frame.  Per-frame inputs are read inside the frame loop.  Each
// frame runs the same operations in the same order as a single-frame launch, so its outputs are bit-identical to one.
__global__ void __launch_bounds__(256)
preprocess_fwd_kernel(const CamParams c0, const FrameStrides fs, const float* __restrict__ means3D, const float* __restrict__ shs,
                      const float* __restrict__ colors_precomp, const float* __restrict__ opacities,
                      const float2* __restrict__ scales, const float4* __restrict__ rotations,
                      int* __restrict__ radii, float4* __restrict__ srec, float* __restrict__ depths,
                      uint32_t* __restrict__ tiles_touched, uint8_t* __restrict__ clamped_out,
                      uint32_t* __restrict__ block_sums, uint32_t* __restrict__ status, int prefiltered) {
    extern __shared__ float shbuf[];
    __shared__ uint32_t wsum[2][8];                 // per-warp tile counts, double-buffered over frames
    const int idx = blockIdx.x * 256 + threadIdx.x;
    const bool live = idx < c0.P;
    const int M3 = 3 * c0.M, stride = M3 + 1;
    const int rows = min(256, c0.P - (int)blockIdx.x * 256);
    const bool use_sh = colors_precomp == nullptr;
    if (use_sh && fs.shs == 0) {
        stage_sh(shbuf, shs + (size_t)blockIdx.x * 256 * M3, rows, M3);
        __syncthreads();
    }
    float px = 0.f, py = 0.f, pz = 0.f, R[9], opac = 0.f;
    float2 sc = make_float2(0.f, 0.f);
    if (live) {
        if (fs.means3D == 0) { px = __ldg(means3D + 3 * (size_t)idx); py = __ldg(means3D + 3 * (size_t)idx + 1); pz = __ldg(means3D + 3 * (size_t)idx + 2); }
        if (fs.rots == 0) rot_matrix(__ldg(rotations + idx), R);
        if (fs.scales == 0) sc = __ldg(scales + idx);
        if (fs.opac == 0) opac = __ldg(opacities + idx);
    }
    for (int f = 0; f < fs.frames; f++) {
        const CamParams c = cam_of_frame(c0, fs, f);
        if (use_sh && fs.shs != 0) {
            // the previous frame's __syncthreads below already ordered every read of shbuf before this overwrite
            stage_sh(shbuf, fr(shs, fs.shs, f) + (size_t)blockIdx.x * 256 * M3, rows, M3);
            __syncthreads();
        }
        uint32_t touched = 0;
        if (live) {
            int radius_i = 0;
            if (fs.means3D != 0) {
                const float* m = fr(means3D, fs.means3D, f) + 3 * (size_t)idx;
                px = __ldg(m); py = __ldg(m + 1); pz = __ldg(m + 2);
            }
            const View V = load_view(c.vm);
            const float depth = view_z(V, px, py, pz);
            if (depth > 0.2f) {
                // ---- computeTransMat ----
                if (fs.rots != 0) rot_matrix(__ldg(fr(rotations, fs.rots, f) + idx), R);
                if (fs.scales != 0) sc = __ldg(fr(scales, fs.scales, f) + idx);
                const float3 pv0 = w_mul(V, make_float3(px, py, pz));
                const float3 pv = make_float3(fa(pv0.x, V.m[12]), fa(pv0.y, V.m[13]), fa(pv0.z, V.m[14]));
                const float3 M0 = w_mul(V, make_float3(fm(R[0], sc.x), fm(R[1], sc.x), fm(R[2], sc.x)));
                const float3 M1 = w_mul(V, make_float3(fm(R[3], sc.y), fm(R[4], sc.y), fm(R[5], sc.y)));
                float3 tn = w_mul(V, make_float3(R[6], R[7], R[8]));
                const float cosv = ff(-pv.z, tn.z, ff(pv.y, -tn.y, -fm(pv.x, tn.x)));
                if (cosv != 0.0f) {
                    const float mult = cosv > 0.f ? 1.f : -1.f;
                    tn.x = fm(tn.x, mult); tn.y = fm(tn.y, mult); tn.z = fm(tn.z, mult);
                    float T[9];
                    T[0] = ff(M0.z, c.cx, fm(c.focal_x, M0.x));
                    T[1] = ff(M1.z, c.cx, fm(c.focal_x, M1.x));
                    T[2] = ff(pv.z, c.cx, fm(c.focal_x, pv.x));
                    T[3] = ff(M0.z, c.cy, fm(c.focal_y, M0.y));
                    T[4] = ff(M1.z, c.cy, fm(c.focal_y, M1.y));
                    T[5] = ff(pv.z, c.cy, fm(c.focal_y, pv.y));
                    T[6] = M0.z; T[7] = M1.z; T[8] = pv.z;
                    // ---- computeAABB ----
                    const float d = ff(-T[8], T[8], ff(T[6], T[6], fm(T[7], T[7])));
                    if (d != 0.0f) {
                        const float r = __fdiv_rn(1.0f, d);
                        const float cxp = ff(fm(T[2], T[8]), -r, ff(fm(T[1], T[7]), r, fm(fm(T[0], T[6]), r)));
                        const float cyp = ff(fm(T[5], T[8]), -r, ff(fm(T[4], T[7]), r, fm(fm(T[3], T[6]), r)));
                        const float nqx = ff(fm(T[2], T[2]), r, -ff(fm(T[1], T[1]), r, fm(fm(T[0], T[0]), r)));
                        const float nqy = ff(fm(T[5], T[5]), r, -ff(fm(T[4], T[4]), r, fm(fm(T[3], T[3]), r)));
                        const float ex = __fsqrt_rn(fmaxf(0.0f, ff(cxp, cxp, nqx)));
                        const float ey = __fsqrt_rn(fmaxf(0.0f, ff(cyp, cyp, nqy)));
                        // forward.cu:239 -- FilterSize is a double literal: max / *3 / ceil happen in double
                        double e = (double)fmaxf(ex, ey);
                        e = fmax(e, 0.7071067811865476);
                        const float radius = (float)ceil(3.0 * e);
                        const int ri = (int)radius;
                        uint2 rmin, rmax;
                        get_rect(cxp, cyp, ri, c.tiles_x, c.tiles_y, rmin, rmax);
                        const uint32_t area = (rmax.x - rmin.x) * (rmax.y - rmin.y);
                        if (area != 0) {
                            uint32_t cl = 0;
                            float3 rgb;
                            if (use_sh) {
                                rgb = sh_to_rgb(c.D, c.M, make_float3(px, py, pz), c.campos, shbuf + threadIdx.x * stride, cl);
                            } else {
                                const float* cp = fr(colors_precomp, fs.colors, f) + 3 * (size_t)idx;
                                rgb = make_float3(__ldg(cp), __ldg(cp + 1), __ldg(cp + 2));
                            }
                            if (fs.opac != 0) opac = __ldg(fr(opacities, fs.opac, f) + idx);
                            uint32_t bx, by;
                            cull_bbox(T, cxp, cyp, opac, c.W, c.H, bx, by);
                            float4* o = fr(srec, fs.geom, f) + (size_t)idx * 5;
                            o[0] = make_float4(T[0], T[1], T[2], T[3]);
                            o[1] = make_float4(T[4], T[5], T[6], T[7]);
                            o[2] = make_float4(T[8], cxp, cyp, opac);
                            o[3] = make_float4(tn.x, tn.y, tn.z, rgb.x);
                            o[4] = make_float4(rgb.y, rgb.z, __uint_as_float(bx), __uint_as_float(by));
                            fr(depths, fs.geom, f)[idx] = depth;
                            fr(clamped_out, fs.geom, f)[idx] = (uint8_t)cl;
                            radius_i = ri;
                            touched = area;
                        }
                    }
                }
            } else if (prefiltered) {
                atomicOr(fr(status, fs.nr, f), 4u);   // the reference __trap()s here (auxiliary.h:177-181)
            }
            fr(radii, fs.radii, f)[idx] = radius_i;
            fr(tiles_touched, fs.geom, f)[idx] = touched;
        }
        // block sum of this frame's tiles_touched -> block_sums[blockIdx.x] of the frame.  Thread 0 reads wsum[f & 1]
        // before it reaches the next frame's barrier, and nobody writes that half again until the frame after.
        uint32_t v = touched;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((threadIdx.x & 31) == 0) wsum[f & 1][threadIdx.x >> 5] = v;
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t tot = 0;
#pragma unroll
            for (int i = 0; i < 8; i++) tot += wsum[f & 1][i];
            fr(block_sums, fs.geom, f)[blockIdx.x] = tot;
        }
    }
}

// exclusive scan of block_sums[0..nb) in place; block_sums[nb] = total; publishes R and the overflow flag
__global__ void __launch_bounds__(1024)
scan_block_sums_kernel(const FrameStrides fs, uint32_t* __restrict__ block_sums, int nb, uint32_t* __restrict__ num_rendered,
                       long long capacity) {
    block_sums = fr(block_sums, fs.geom, (int)blockIdx.x);          // one block per frame
    num_rendered = fr(num_rendered, fs.nr, (int)blockIdx.x);
    __shared__ uint32_t wtot[32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    for (int base = 0; base < nb; base += 1024) {
        const int i = base + threadIdx.x;
        const uint32_t v = i < nb ? block_sums[i] : 0u;
        uint32_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= o) inc += n; }
        if ((threadIdx.x & 31) == 31) wtot[threadIdx.x >> 5] = inc;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = wtot[threadIdx.x], winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, winc, o); if (threadIdx.x >= o) winc += n; }
            wtot[threadIdx.x] = winc - w;   // exclusive
        }
        __syncthreads();
        const uint32_t carry = carry_s;
        const uint32_t excl = carry + wtot[threadIdx.x >> 5] + inc - v;
        if (i < nb) block_sums[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        const uint32_t R = carry_s;
        block_sums[nb] = R;
        num_rendered[0] = R;
        if ((long long)R > capacity) atomicOr(num_rendered + 1, SR_STATUS_OVERFLOW);
    }
}

// duplicateWithKeys: offsets come from the block prefix + an in-block scan; same emission order as the
// reference (ascending surfel id, row-major over the tile rectangle) so that the stable sort ties agree.
__global__ void __launch_bounds__(256)
emit_keys_kernel(const CamParams c, const FrameStrides fs, const float4* __restrict__ srec, const float* __restrict__ depths,
                 const int* __restrict__ radii, const uint32_t* __restrict__ tiles_touched,
                 const uint32_t* __restrict__ block_sums, uint32_t* __restrict__ point_offsets,
                 uint64_t* __restrict__ keys, uint32_t* __restrict__ values, long long capacity) {
    const int f = blockIdx.y;
    srec = fr(srec, fs.geom, f); depths = fr(depths, fs.geom, f); radii = fr(radii, fs.radii, f);
    tiles_touched = fr(tiles_touched, fs.geom, f); block_sums = fr(block_sums, fs.geom, f);
    point_offsets = fr(point_offsets, fs.geom, f); keys = fr(keys, fs.bin, f); values = fr(values, fs.bin, f);
    const int idx = blockIdx.x * 256 + threadIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t total = block_sums[gridDim.x];
    const uint32_t touched = idx < c.P ? tiles_touched[idx] : 0u;
    __shared__ uint32_t wtot[8];
    uint32_t inc = touched;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    uint32_t wbase = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) wbase += i < warp ? wtot[i] : 0u;
    uint32_t off = block_sums[blockIdx.x] + wbase + inc - touched;
    if (idx < c.P) point_offsets[idx] = off + touched;
    if ((long long)total > capacity) return;    // overflow: the frame is abandoned (status already set)

    uint2 rmin = make_uint2(0, 0), rmax = make_uint2(0, 0);
    uint32_t dbits = 0;
    if (touched) {
        const float4 r2 = __ldg(srec + (size_t)idx * 5 + 2);   // (Tw.z, xy.x, xy.y, opacity)
        get_rect(r2.y, r2.z, radii[idx], c.tiles_x, c.tiles_y, rmin, rmax);
        dbits = __float_as_uint(depths[idx]);
    }
    const uint32_t BIG = 32;
    if (touched && touched <= BIG) {
        for (uint32_t y = rmin.y; y < rmax.y; y++)
            for (uint32_t x = rmin.x; x < rmax.x; x++) {
                keys[off] = ((uint64_t)(y * (uint32_t)c.tiles_x + x) << 32) | dbits;
                values[off] = (uint32_t)idx;
                off++;
            }
    }
    // large footprints: the whole warp emits one surfel's rectangle cooperatively
    uint32_t bigmask = __ballot_sync(0xffffffffu, touched > BIG);
    while (bigmask) {
        const int src = __ffs(bigmask) - 1;
        bigmask &= bigmask - 1;
        const uint32_t n = __shfl_sync(0xffffffffu, touched, src);
        const uint32_t o0 = __shfl_sync(0xffffffffu, off, src);
        const uint32_t x0 = __shfl_sync(0xffffffffu, rmin.x, src), y0 = __shfl_sync(0xffffffffu, rmin.y, src);
        const uint32_t wdt = __shfl_sync(0xffffffffu, rmax.x, src) - x0;
        const uint32_t db = __shfl_sync(0xffffffffu, dbits, src);
        const uint32_t id = (uint32_t)(blockIdx.x * 256 + warp * 32 + src);
        for (uint32_t t = lane; t < n; t += 32) {
            const uint32_t y = y0 + t / wdt, x = x0 + t % wdt;
            keys[o0 + t] = ((uint64_t)(y * (uint32_t)c.tiles_x + x) << 32) | db;
            values[o0 + t] = id;
        }
    }
}

__global__ void mark_visible_kernel(int P, const float* __restrict__ means3D, const float* __restrict__ vm, uint8_t* __restrict__ present) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= P) return;
    const View V = load_view(vm);
    const float z = view_z(V, means3D[3 * (size_t)idx], means3D[3 * (size_t)idx + 1], means3D[3 * (size_t)idx + 2]);
    present[idx] = z > 0.2f;
}

}  // namespace

cudaError_t launch_preprocess_fwd(const FwdArgs& a) {
    const int nb = a.gl.nblocks;
    const size_t smem = a.colors_precomp ? 0 : (size_t)256 * (3 * a.cam.M + 1) * sizeof(float);
    if (cudaError_t e = sr_opt_in_smem(preprocess_fwd_kernel, smem)) return e;
    ProfileScope ps("preprocess_fwd", a.stream);
    preprocess_fwd_kernel<<<nb, 256, smem, a.stream>>>(
        a.cam, a.fs, a.means3D, a.shs, a.colors_precomp, a.opacities, (const float2*)a.scales, (const float4*)a.rotations,
        a.radii, (float4*)(a.geom + a.gl.surfel_rec), (float*)(a.geom + a.gl.depths),
        (uint32_t*)(a.geom + a.gl.tiles_touched), (uint8_t*)(a.geom + a.gl.clamped),
        (uint32_t*)(a.geom + a.gl.block_sums), a.num_rendered_dev + 1, a.prefiltered);
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_scan_emit(const FwdArgs& a) {
    const int nb = a.gl.nblocks;
    uint32_t* bs = (uint32_t*)(a.geom + a.gl.block_sums);
    { ProfileScope ps("scan_block_sums", a.stream);
      scan_block_sums_kernel<<<a.fs.frames, 1024, 0, a.stream>>>(a.fs, bs, nb, a.num_rendered_dev, (long long)a.bl.capacity); }
    ProfileScope ps("emit_keys", a.stream);
    emit_keys_kernel<<<dim3(nb, a.fs.frames), 256, 0, a.stream>>>(
        a.cam, a.fs, (const float4*)(a.geom + a.gl.surfel_rec), (const float*)(a.geom + a.gl.depths), a.radii,
        (const uint32_t*)(a.geom + a.gl.tiles_touched), bs, (uint32_t*)(a.geom + a.gl.point_offsets),
        (uint64_t*)(a.bin + a.bl.keys[0]), (uint32_t*)(a.bin + a.bl.values[0]), (long long)a.bl.capacity);
    sr_count_launch(2);
    return cudaGetLastError();
}

cudaError_t launch_mark_visible(int P, const float* means3D, const float* vm, uint8_t* present, cudaStream_t s) {
    mark_visible_kernel<<<(P + 255) / 256, 256, 0, s>>>(P, means3D, vm, present);
    sr_count_launch();
    return cudaGetLastError();
}
