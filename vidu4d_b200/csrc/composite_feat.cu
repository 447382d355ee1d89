// composite_feat.cu -- per-surfel feature channels composited with the colour's weights, forward and backward.
//
// The reference's Stage-3 code builds a per-surfel feature vector (registration feature, flow, normal, mask) and
// renders it next to the SH colour (lab4d/nnutils/deformable_gaussian.py:1182-1207); its rasterizer composites three
// channels only, so the vector is dropped there.  Here plane f of a pixel is
//     sum_i T_i alpha_i feat[i, f]  +  T_final bg_f
// over exactly the contributors, weights and FMA order of the colour planes.
//
// Design (DESIGN.md "feature channels"):
//   * a separate pass after the composite forward / backward; the pinned composite kernels are untouched.  It reads
//     what either composite forward leaves behind: the instance records, the per-(stage, pixel) contribution masks,
//     final_T and each 8x4 sub-tile's deepest contributor (sub_last);
//   * work item = (tile, 8x4 sub-tile) = one warp = one CTA, lane = pixel; the tile's records stream through the
//     warp-private 2-stage ring of 32 records that composite_fwd.cu uses (comp::Ring).  Every lane
//     walks only its own recorded contributors -- no cull or alpha test is repeated -- and re-evaluates alpha with the
//     forward's arithmetic (comp::pair_alpha), so each plane is bit-identical to a colour plane of the same values;
//   * a CTA owns SR_FEAT_CHUNK = 8 channels (gridDim.y = ceil(F/8)): 8 accumulators (forward) or 8 accumulators + 8
//     incoming gradients (backward) bound the register use for any F <= 32; the row of a surfel's features is read
//     with 16-, 8- or 4-byte vector loads depending on F and alignment (F = 22: rows of 88 B -> float2);
//   * backward: reverse walk from final_T as in comp::BwdPixel; dL/dfeat = T alpha dL/dplane leaves by vector
//     reductions into the zeroed dL/dfeatures; dL/dalpha of the chunk goes through the colour path's geometry
//     vector-Jacobian product (comp::pair_geom_vjp, dL/dz = 0) into the per-surfel accumulator's dT / dopacity /
//     low-pass dmean2D slots, which surfel_bwd then chains to means3D / scales / rotations / opacities / means2D.
#include "composite_common.cuh"

namespace {
using namespace comp;
constexpr int FC = SR_FEAT_CHUNK;

template <int V>
__device__ __forceinline__ void red_chunk(float* row, int c0, int F, const float (&g)[FC]) {
#pragma unroll
    for (int k = 0; k < FC; k += V) {
        if (c0 + k < F) {
            if constexpr (V == 4)
                asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" :: "l"(row + c0 + k), "f"(g[k]), "f"(g[k + 1]), "f"(g[k + 2]), "f"(g[k + 3]) : "memory");
            else if constexpr (V == 2)
                asm volatile("red.global.v2.f32.add [%0], {%1, %2};" :: "l"(row + c0 + k), "f"(g[k]), "f"(g[k + 1]) : "memory");
            else
                atomicAdd(row + c0 + k, g[k]);
        }
    }
}

// ------------------------------------------------------------------------------------------------ forward
template <int V>
__global__ void __launch_bounds__(32, 32)
feature_fwd_kernel(const FrameStrides fs, const FeatArgs ft, const uint2* __restrict__ ranges,
                   const uint32_t* __restrict__ tile_order, int n_items, int tiles_x, const float4* __restrict__ irec,
                   int W, int H, const uint32_t* __restrict__ sub_last, const uint32_t* __restrict__ contrib_masks) {
    __shared__ __align__(128) float4 st[NST][WB * REC4];
    __shared__ __align__(8) uint64_t bar[NST];
    const int lane = threadIdx.x;
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    const int item = (int)(blockIdx.x / (unsigned)fs.frames);
    if (item >= n_items) return;
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    sub_last = fr(sub_last, fs.img, f); contrib_masks = fr(contrib_masks, fs.bin, f);
    const float* feat = fr(ft.feat, ft.feat_stride, f);
    float* out = fr(ft.out, ft.out_stride, f);
    const int F = ft.F, c0 = (int)blockIdx.y * FC;

    const int warp = item & 7;
    const int tile = (int)tile_order[item >> 3];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const int len = min((int)(range.y - range.x), (int)sub_last[tile * 8 + warp]);   // nothing deeper contributed
    const int nb = (len + WB - 1) / WB;
    const SubPixel sp = sub_pixel(tile_x, tile_y, warp, lane);

    Ring ring{st, bar, irec + (size_t)range.x * REC4, len};
    if (lane == 0) {
        ring.init();
        for (int b = 0; b < NST && b < nb; b++) ring.issue(b, b);
    }
    __syncwarp();

    float T = 1.0f, acc[FC];
#pragma unroll
    for (int k = 0; k < FC; k++) acc[k] = 0.f;
    const uint32_t* cm_in = contrib_masks + contrib_word(range.x, tile, warp, lane);
    uint32_t next = nb > 0 ? __ldg(cm_in) : 0u;
    for (int b = 0; b < nb; b++) {
        uint32_t own = next;
        if (b + 1 < nb) next = __ldg(cm_in + (size_t)(b + 1) * SR_CONTRIB_STAGE_WORDS);
        const float4* S = ring.wait(b);
        while (own != 0u) {                               // front to back over this pixel's contributors only
            const int jj = __ffs(own) - 1;
            own &= own - 1u;
            const float4* R = S + jj * REC4;
            PairAlpha q;
            pair_alpha(R[0], R[1], R[2], sp.pixx, sp.pixy, q);
            float x[FC];
            load_chunk<V>(feat + (size_t)__float_as_uint(R[4].z) * F, c0, F, x);
#pragma unroll
            for (int k = 0; k < FC; k++) acc[k] = ff(T, fm(q.alpha, x[k]), acc[k]);   // == the colour planes' update
            T = fm(T, fa(1.0f, -q.alpha));
        }
        __syncwarp();                                     // every lane is done reading stage b
        if (lane == 0 && b + NST < nb) ring.issue(b + NST, b + NST);
    }

    if (sp.inside(W, H)) {
        const size_t N = (size_t)W * H, pid = (size_t)W * sp.pix_y + sp.pix_x;
#pragma unroll
        for (int k = 0; k < FC; k++)
            if (c0 + k < F) out[(size_t)(c0 + k) * N + pid] = ft.bg ? ff(T, __ldg(ft.bg + c0 + k), acc[k]) : ff(T, 0.0f, acc[k]);
    }
}

// ------------------------------------------------------------------------------------------------ backward
template <int V>
__global__ void __launch_bounds__(32, 24)      // <= 85 registers: the scalar-row variant otherwise takes 125
feature_bwd_kernel(const FrameStrides fs, const FeatArgs ft, const uint2* __restrict__ ranges,
                   const uint32_t* __restrict__ tile_order, int n_items, int tiles_x, const float4* __restrict__ irec,
                   int W, int H, const float* __restrict__ final_Ts, const uint32_t* __restrict__ sub_last,
                   const uint32_t* __restrict__ contrib_masks, float* __restrict__ sgrad) {
    __shared__ __align__(128) float4 st[NST][WB * REC4];
    __shared__ __align__(8) uint64_t bar[NST];
    const int lane = threadIdx.x;
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    const int item = (int)(blockIdx.x / (unsigned)fs.frames);
    if (item >= n_items) return;
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_Ts = fr(final_Ts, fs.img, f); sub_last = fr(sub_last, fs.img, f);
    contrib_masks = fr(contrib_masks, fs.bin, f); sgrad = fr(sgrad, fs.geom, f);
    const float* feat = fr(ft.feat, ft.feat_stride, f);
    const float* dout = fr(ft.dout, ft.dout_stride, f);
    float* dfeat = fr(ft.dfeat, ft.dfeat_stride, f);
    const int F = ft.F, c0 = (int)blockIdx.y * FC;

    const int warp = item & 7;
    const int tile = (int)tile_order[item >> 3];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const int len = min((int)(range.y - range.x), (int)sub_last[tile * 8 + warp]);
    const int nb = (len + WB - 1) / WB;
    if (nb == 0) return;
    const SubPixel sp = sub_pixel(tile_x, tile_y, warp, lane);

    // the k-th consumed batch is b = nb-1-k
    Ring ring{st, bar, irec + (size_t)range.x * REC4, len};
    if (lane == 0) {
        ring.init();
        for (int k = 0; k < NST && k < nb; k++) ring.issue(k, nb - 1 - k);
    }
    __syncwarp();

    // per-pixel state (comp::BwdPixel::load, feature planes only)
    const bool inside = sp.inside(W, H);
    const size_t N = (size_t)W * H, pid = (size_t)W * sp.pix_y + sp.pix_x;
    const float T_final = inside ? final_Ts[pid] : 0.f;
    float T = T_final, g[FC], accum[FC], bg_dot = 0.f;
    const float gs = ft.grad_scale ? __ldg(ft.grad_scale) : 1.0f;
#pragma unroll
    for (int k = 0; k < FC; k++) {
        g[k] = (inside && c0 + k < F) ? dout[(size_t)(c0 + k) * N + pid] * gs : 0.f;
        if (ft.bg && c0 + k < F) bg_dot += __ldg(ft.bg + c0 + k) * g[k];
        accum[k] = 0.f;
    }

    const uint32_t* cm_in = contrib_masks + contrib_word(range.x, tile, warp, lane);
    uint32_t next = __ldg(cm_in + (size_t)(nb - 1) * SR_CONTRIB_STAGE_WORDS);
    for (int k = 0; k < nb; k++) {
        const int b = nb - 1 - k;
        uint32_t own = next;
        if (b > 0) next = __ldg(cm_in + (size_t)(b - 1) * SR_CONTRIB_STAGE_WORDS);
        const float4* S = ring.wait(k);
        while (own != 0u) {                               // back to front over this pixel's contributors only
            const int jj = 31 - __clz(own);
            own &= ~(1u << jj);
            const float4* R = S + jj * REC4;
            const float4 r1 = R[1], r2 = R[2];
            PairAlpha q;
            pair_alpha(R[0], r1, r2, sp.pixx, sp.pixy, q);
            const float alpha = q.alpha;
            const float r1ma = rcp_approx(1.f - alpha);   // as comp::BwdPixel::pair_scalars
            T = T * r1ma;
            const float aT = alpha * T;
            const uint32_t id = __float_as_uint(R[4].z);
            float x[FC], d[FC];
            load_chunk<V>(feat + (size_t)id * F, c0, F, x);
            float dL_dalpha = 0.f;
            const float oma = 1.f - alpha;
#pragma unroll
            for (int c = 0; c < FC; c++) {
                dL_dalpha += (x[c] - accum[c]) * g[c];
                d[c] = aT * g[c];
                accum[c] = alpha * x[c] + oma * accum[c];
            }
            red_chunk<V>(dfeat + (size_t)id * F, c0, F, d);
            dL_dalpha *= T;
            dL_dalpha += (-T_final * r1ma) * bg_dot;
            float v[16];
            float m2x = 0.f, m2y = 0.f;
            bool lowpass = false;
            pair_geom_vjp(q, r1, r2.w, sp.pixx, sp.pixy, dL_dalpha, 0.f, v, m2x, m2y, lowpass);
            float* gp = sgrad + (size_t)id * SR_GRAD_FLOATS;
            if (!lowpass) {
                asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" :: "l"(gp + SR_G_T), "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3]) : "memory");
                asm volatile("red.global.v4.f32.add [%0], {%1, %2, %3, %4};" :: "l"(gp + SR_G_T + 4), "f"(v[4]), "f"(v[5]), "f"(v[6]), "f"(v[7]) : "memory");
                asm volatile("red.global.v2.f32.add [%0], {%1, %2};" :: "l"(gp + SR_G_T + 8), "f"(v[8]), "f"(v[9]) : "memory");
            } else {
                // dL/dz = 0 for features: only dopacity and the low-pass dmean2D
                atomicAdd(gp + SR_G_OPAC, v[9]);
                asm volatile("red.global.v2.f32.add [%0], {%1, %2};" :: "l"(gp + SR_G_M2D), "f"(m2x), "f"(m2y) : "memory");
            }
        }
        __syncwarp();
        if (lane == 0 && k + NST < nb) ring.issue(k + NST, nb - 1 - (k + NST));
    }
}
static_assert(SR_G_T + 9 == SR_G_OPAC && (SR_G_T + 8) % 2 == 0 && SR_G_M2D % 2 == 0, "feature_bwd's vector reductions");

}  // namespace

cudaError_t launch_feature_fwd(const FwdArgs& a, const FeatArgs& ft) {
    ProfileScope ps("feature_fwd", a.stream);
    const dim3 grid((unsigned)(a.il.tiles * 8) * (unsigned)a.fs.frames, (unsigned)((ft.F + FC - 1) / FC));
    auto launch = [&](auto kern) {
        kern<<<grid, 32, 0, a.stream>>>(a.fs, ft, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order),
                                        a.il.tiles * 8, a.il.tiles_x, (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H,
                                        (const uint32_t*)(a.img + a.il.tile_last), (const uint32_t*)(a.bin + a.bl.contrib));
    };
    if (ft.vec == 4) launch(feature_fwd_kernel<4>);
    else if (ft.vec == 2) launch(feature_fwd_kernel<2>);
    else launch(feature_fwd_kernel<1>);
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_feature_bwd(const BwdArgs& a, const FeatArgs& ft) {
    ProfileScope ps("feature_bwd", a.stream);
    const dim3 grid((unsigned)(a.il.tiles * 8) * (unsigned)a.fs.frames, (unsigned)((ft.F + FC - 1) / FC));
    auto launch = [&](auto kern) {
        kern<<<grid, 32, 0, a.stream>>>(a.fs, ft, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order),
                                        a.il.tiles * 8, a.il.tiles_x, (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H,
                                        (const float*)(a.img + a.il.final_T), (const uint32_t*)(a.img + a.il.tile_last),
                                        (const uint32_t*)(a.bin + a.bl.contrib), (float*)(a.geom + a.gl.sgrad));
    };
    if (ft.vec == 4) launch(feature_bwd_kernel<4>);
    else if (ft.vec == 2) launch(feature_bwd_kernel<2>);
    else launch(feature_bwd_kernel<1>);
    sr_count_launch();
    return cudaGetLastError();
}
