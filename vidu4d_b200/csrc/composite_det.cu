// composite_det.cu -- the deterministic rasterizer backward's feature pass, slot zeroing and per-surfel gather
// (include/surfel_deterministic.h, DESIGN.md 3.4b).  The colour pass is composite_tile_bwd_kernel<true>.
//
// Every (instance, tile) owns one slot per frame, indexed by the instance's emission index (emit_keys' order: surfel
// id, then the tile's row-major position in the surfel's rectangle), so a surfel's slots are contiguous:
//   det.slots   20 floats, accumulator layout SR_G_*: the colour pass STORES the (instance, tile) sum, the feature pass
//               adds its geometry terms to it (the CTA that owns a tile is the only writer of its instances' slots);
//   det.fslots  F floats: the feature pass stores dL/dfeatures of the (instance, tile).
// det_gather_kernel then sums each surfel's slots in emission order into the per-surfel accumulator (which surfel_bwd
// reads unchanged) and into dL/dfeatures, adding frames in order where the frames share the features.  No float
// atomic touches a gradient, so every sum has an order fixed by the data.
//
// feature_bwd_det_kernel is the colour backward's two-phase scheme (composite_tile.cu) for the feature planes:
//   1. pixel phase (lane = pixel, 8 warps = 8 sub-tiles): the reverse walk over the recorded contributors with all F
//      channels (accum[NCH] in registers, the pixel's dL/dplane staged in shared memory), reduced per pair to
//      G dL/dalpha and alpha T (sign = branch), which go to a shared pair buffer at the pixel's scan slot;
//   2. instance phase (thread = instance of the chunk): dL/dfeat_f = sum over its pixels of alpha T dL/dplane_f and the
//      geometry vector-Jacobian product from the stored scalars (pair_geom_vjp_stored, dL/dz = 0), in ascending pixel
//      order.  A chunk with more pairs than FCAP runs in passes of whole pixels, as the colour pass does.
#include "composite_common.cuh"

namespace {
using namespace comp;

constexpr int FCAP = 3072;         // pair-buffer slots, 8 B each
struct FdSmem {
    static constexpr size_t masks = (size_t)BWD_NSLOT * BWD_CH * REC4 * sizeof(float4);
    static constexpr size_t g = masks + (size_t)BWD_NSTG * BWD_NPIX * sizeof(uint32_t);          // dL/dplane [channel][pixel]
    static constexpr size_t buf = g + (size_t)SR_FEAT_MAX * BWD_NPIX * sizeof(float);            // pair buffer, 2 x FCAP
    static constexpr size_t sfx = buf + 2 * (size_t)FCAP * sizeof(float);                        // slot table [stage][pixel]
    static constexpr size_t full = sfx + (size_t)BWD_NSTG * BWD_NPIX * sizeof(uint16_t);
    static constexpr size_t wsum = full + BWD_NSLOT * sizeof(uint64_t);
    static constexpr size_t total = wsum + BWD_WARPS * sizeof(uint32_t);
};
static_assert(FdSmem::full % 8 == 0, "mbarrier alignment");
static_assert(2 * (FdSmem::total + 1024) <= 233472, "two CTAs per SM (228 KB, 1 KB reserved per CTA)");

// NCH = the channel count F rounded up to a multiple of SR_FEAT_CHUNK (register arrays of compile-time size)
template <int NCH>
__global__ void __launch_bounds__(BWD_NPIX, 2)
feature_bwd_det_kernel(const FrameStrides fs, const FeatArgs ft, const uint2* __restrict__ ranges,
                       const uint32_t* __restrict__ tile_order, int tiles_x, const float4* __restrict__ irec, int W, int H,
                       const float* __restrict__ final_Ts, const uint32_t* __restrict__ sub_last,
                       const uint32_t* __restrict__ contrib_masks, const DetArgs det) {
    using SM = FdSmem;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint32_t* cm_all = reinterpret_cast<uint32_t*>(smem_raw + SM::masks);
    float* gsm = reinterpret_cast<float*>(smem_raw + SM::g);
    float* buf_a = reinterpret_cast<float*>(smem_raw + SM::buf);     // G times dL/dalpha (times T, with the background term)
    float* buf_t = buf_a + FCAP;                                      // alpha T, negated on the low-pass branch
    uint16_t* sfx = reinterpret_cast<uint16_t*>(smem_raw + SM::sfx);
    uint32_t* wsum = reinterpret_cast<uint32_t*>(smem_raw + SM::wsum);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_Ts = fr(final_Ts, fs.img, f); sub_last = fr(sub_last, fs.img, f); contrib_masks = fr(contrib_masks, fs.bin, f);
    const float* feat = fr(ft.feat, ft.feat_stride, f);
    const float* dout = fr(ft.dout, ft.dout_stride, f);
    float* slots = fr(det.slots, det.slots_stride, f);
    float* fslots = fr(det.fslots, det.fslots_stride, f);
    const uint32_t* point_offsets = fr(det.point_offsets, fs.geom, f);
    const int* radii = fr(det.radii, fs.radii, f);
    const int F = ft.F;
    const int tile = (int)tile_order[blockIdx.x / (unsigned)fs.frames];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const BwdTile bt = bwd_tile(range, sub_last, tile);
    if (bt.nchunks == 0) return;                   // CTA-uniform
    const int nb_w = bt.nb_w();
    const ChunkRing ring{reinterpret_cast<float4*>(smem_raw), reinterpret_cast<uint64_t*>(smem_raw + SM::full),
                         irec + (size_t)range.x * REC4, bt.len, bt.nchunks};
    if (threadIdx.x == 0) ring.init();

    // per-pixel state (as feature_bwd_kernel's, all channels at once); thread == pixel == warp * 32 + lane
    const SubPixel sp = sub_pixel(tile_x, tile_y, warp, lane);
    const bool inside = sp.inside(W, H);
    const size_t N = (size_t)W * H, pid = (size_t)W * sp.pix_y + sp.pix_x;
    const float T_final = inside ? final_Ts[pid] : 0.f;
    float T = T_final, accum[NCH], bg_dot = 0.f;
    const float gs = ft.grad_scale ? __ldg(ft.grad_scale) : 1.0f;
#pragma unroll
    for (int c = 0; c < NCH; c++) {
        accum[c] = 0.f;
        if (c < F) {
            const float g = inside ? dout[(size_t)c * N + pid] * gs : 0.f;
            gsm[c * BWD_NPIX + threadIdx.x] = g;
            if (ft.bg) bg_dot += __ldg(ft.bg + c) * g;
        }
    }

    PixelMasks masks{cm_all + warp * BWD_NSTG * 32 + lane, contrib_masks + contrib_word(range.x, tile, warp, lane),
                     nb_w};
    masks.fetch(bt.nchunks - 1);

    for (int k = 0; k < bt.nchunks; k++) {
        const int c = bt.nchunks - 1 - k, s = k % BWD_NSLOT;
        int np, total = 0;
        const uint32_t nz = masks.install(np);
        const int base = masks.scan(np, wsum, sfx);            // its barrier also orders dL/dplane before the first chunk
#pragma unroll 1                                               // rolled: fewer registers beside the channel arrays
        for (int w = 0; w < BWD_WARPS; w++) total += (int)wsum[w];
        const DetPasses dp(total, FCAP, BWD_CH);
        if (c > 0) masks.fetch(c - 1);
        const float4* S = ring.wait(k, s);

        for (int pass = 0; pass < dp.npass; pass++) {
            if (pass > 0) __syncthreads();         // the previous pass's phase 2 is done with the buffer
            const int off = dp.offset(pass);
            // ---- phase 1: lane = pixel, back to front over its contributors
            uint32_t nzp = dp.of(base) == pass ? nz : 0u;
            if (__any_sync(0xffffffffu, nzp != 0u)) {
                int st = 0, slot = base;
                uint32_t mym = 0u;
                for (;;) {
                    if (mym == 0u && nzp) { st = 31 - __clz(nzp); nzp &= ~(1u << st); mym = masks.cm[st * 32]; }
                    const bool act = mym != 0u;
                    if (!__any_sync(0xffffffffu, act)) break;
                    if (!act) continue;
                    const int jj = 31 - __clz(mym);
                    mym &= ~(1u << jj);
                    const float4* R = S + (st * 32 + jj) * REC4;
                    PairAlpha q;
                    pair_alpha(R[0], R[1], R[2], sp.pixx, sp.pixy, q);
                    const float alpha = q.alpha;
                    const float r1ma = rcp_approx(1.f - alpha);
                    T = T * r1ma;
                    const float aT = alpha * T;
                    const float* row = feat + (size_t)__float_as_uint(R[4].z) * F;
                    const float oma = 1.f - alpha;
                    float dL_dalpha = 0.f;
#pragma unroll
                    for (int ch = 0; ch < NCH; ch++) {
                        if (ch < F) {
                            const float x = __ldg(row + ch);
                            dL_dalpha += (x - accum[ch]) * gsm[ch * BWD_NPIX + threadIdx.x];
                            accum[ch] = alpha * x + oma * accum[ch];
                        }
                    }
                    dL_dalpha *= T;
                    dL_dalpha += (-T_final * r1ma) * bg_dot;
                    buf_a[slot - off] = q.G_ * dL_dalpha;
                    buf_t[slot - off] = (q.rho3d <= q.rho2d) ? aT : -aT;
                    slot++;
                }
            }
            __syncthreads();                       // pair buffer complete

            // ---- phase 2: thread = instance warp * 32 + lane of the chunk
            const InstancePixels ip(cm_all);
            if (ip.any) {
                const float4* R = S + threadIdx.x * REC4;
                const float4 r0 = R[0], r1 = R[1], r2 = R[2];
                const uint32_t e = sr_emission_index(point_offsets, radii, __float_as_uint(R[4].z), r2.y, r2.z, tile_x, tile_y,
                                                     tiles_x, det.tiles_y);
                float* gslot = slots + (size_t)e * SR_GRAD_FLOATS;
                float* fslot = fslots + (size_t)e * F;
                float acc[16], df[NCH], a2x = 0.f, a2y = 0.f;
                bool any_in = false;
#pragma unroll
                for (int i = 0; i < 16; i++) acc[i] = 0.f;
#pragma unroll
                for (int ch = 0; ch < NCH; ch++) df[ch] = 0.f;
                ip.walk(cm_all, sfx, dp, pass, [&](int p, int sw, int l, int b) {
                    if (!any_in) {
                        // first pair of this pass: start from what the slot holds -- the colour pass's sum, and the
                        // partial sums of earlier passes
                        slot_load(gslot, acc, a2x, a2y);
                        if (pass > 0) {
#pragma unroll
                            for (int ch = 0; ch < NCH; ch++) if (ch < F) df[ch] = fslot[ch];
                        }
                        any_in = true;
                    }
                    const SubPixel pp = sub_pixel(tile_x, tile_y, sw, l);
                    const float t = buf_t[b];
                    pair_geom_vjp_stored(r0, r1, r2, pp.pixx, pp.pixy, buf_a[b], 0.f, t < 0.f, acc, a2x, a2y);
                    const float aT = fabsf(t);
#pragma unroll
                    for (int ch = 0; ch < NCH; ch++) if (ch < F) df[ch] += aT * gsm[ch * BWD_NPIX + p];
                });
                if (any_in) {
                    slot_store(gslot, acc, a2x, a2y);
#pragma unroll
                    for (int ch = 0; ch < NCH; ch++) if (ch < F) fslot[ch] = df[ch];
                }
            }
        }
        __syncthreads();                           // ring slot, masks, pair buffer and slot table are free again
        if (threadIdx.x == 0 && k + BWD_NSLOT < bt.nchunks) ring.issue(k + BWD_NSLOT);
    }
}

// the instances a frame emitted, or 0 for a frame the forward abandoned (more instances than the capacity)
__device__ __forceinline__ uint32_t frame_instances(const DetArgs& d, const FrameStrides& fs, int f, int P, long long capacity) {
    const uint32_t R = __ldg(fr(d.point_offsets, fs.geom, f) + (P - 1));
    return (long long)R > capacity ? 0u : R;
}

// zeroes the slots of the instances each frame emitted (blockIdx.y = frame)
__global__ void __launch_bounds__(256)
det_zero_kernel(const FrameStrides fs, int P, long long capacity, const DetArgs d, int F) {
    const int f = blockIdx.y;
    const size_t R = frame_instances(d, fs, f, P, capacity);
    float4* s4 = reinterpret_cast<float4*>(fr(d.slots, d.slots_stride, f));
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < R * (SR_GRAD_FLOATS / 4); i += stride) s4[i] = z;
    if (d.fslots) {
        float* fs1 = fr(d.fslots, d.fslots_stride, f);
        for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < R * (size_t)F; i += stride) fs1[i] = 0.f;
    }
}

// One thread per surfel, frames looped inside (as surfel_bwd): the surfel's slots, summed in emission order, become
// its per-surfel accumulator of each frame and its dL/dfeatures -- per frame, or summed over the frames in order when
// the frames share the features (dfeat_stride 0).  Every element of both is written.
constexpr int GB = 128;
__global__ void __launch_bounds__(GB)
det_gather_kernel(const FrameStrides fs, int P, long long capacity, const DetArgs d, float* __restrict__ sgrad, int F,
                  float* __restrict__ dfeat, long long dfeat_stride) {
    const int idx = blockIdx.x * GB + threadIdx.x;
    if (idx >= P) return;
    for (int f = 0; f < fs.frames; f++) {
        const uint32_t* po = fr(d.point_offsets, fs.geom, f);
        const bool live = frame_instances(d, fs, f, P, capacity) != 0u;
        const uint32_t e0 = (live && idx > 0) ? __ldg(po + idx - 1) : 0u, e1 = live ? __ldg(po + idx) : 0u;
        const float4* s4 = reinterpret_cast<const float4*>(fr(d.slots, d.slots_stride, f));
        float4 a[5];
#pragma unroll
        for (int q = 0; q < 5; q++) a[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (uint32_t e = e0; e < e1; e++) {
#pragma unroll
            for (int q = 0; q < 5; q++) {
                const float4 v = s4[(size_t)e * 5 + q];
                a[q].x += v.x; a[q].y += v.y; a[q].z += v.z; a[q].w += v.w;
            }
        }
        float4* o = reinterpret_cast<float4*>(fr(sgrad, fs.geom, f)) + (size_t)idx * 5;
#pragma unroll
        for (int q = 0; q < 5; q++) o[q] = a[q];
    }
    if (!dfeat) return;
    // SR_FEAT_CHUNK channels at a time in registers: each slot row is read once per chunk, and every channel's sum runs
    // over the frames in order and the slots in emission order
    const bool shared = dfeat_stride == 0;
    constexpr int FC = SR_FEAT_CHUNK;
    for (int c0 = 0; c0 < F; c0 += FC) {
        float tot[FC];
#pragma unroll
        for (int j = 0; j < FC; j++) tot[j] = 0.f;
        for (int f = 0; f < fs.frames; f++) {
            const uint32_t* po = fr(d.point_offsets, fs.geom, f);
            const bool live = frame_instances(d, fs, f, P, capacity) != 0u;
            const uint32_t e0 = (live && idx > 0) ? __ldg(po + idx - 1) : 0u, e1 = live ? __ldg(po + idx) : 0u;
            const float* fsl = fr(d.fslots, d.fslots_stride, f);
            float s[FC];
#pragma unroll
            for (int j = 0; j < FC; j++) s[j] = 0.f;
            for (uint32_t e = e0; e < e1; e++) {
                const float* row = fsl + (size_t)e * F + c0;
#pragma unroll
                for (int j = 0; j < FC; j++) if (c0 + j < F) s[j] += row[j];
            }
            float* out = fr(dfeat, dfeat_stride, f) + (size_t)idx * F + c0;
#pragma unroll
            for (int j = 0; j < FC; j++) {
                if (c0 + j < F) {
                    if (shared) tot[j] += s[j];
                    else out[j] = s[j];
                }
            }
        }
        if (shared) {
#pragma unroll
            for (int j = 0; j < FC; j++) if (c0 + j < F) dfeat[(size_t)idx * F + c0 + j] = tot[j];
        }
    }
}

}  // namespace

cudaError_t launch_det_zero(const BwdArgs& a, const DetArgs& d, int F) {
    ProfileScope ps("det_zero", a.stream);
    det_zero_kernel<<<dim3(512, (unsigned)a.fs.frames), 256, 0, a.stream>>>(a.fs, a.cam.P, (long long)a.bl.capacity, d, F);
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_feature_bwd_det(const BwdArgs& a, const FeatArgs& ft, const DetArgs& d) {
    ProfileScope ps("feature_bwd_det", a.stream);
    auto launch = [&](auto kern) -> cudaError_t {
        if (cudaError_t e = sr_opt_in_smem(kern, FdSmem::total)) return e;
        kern<<<a.il.tiles * a.fs.frames, BWD_NPIX, FdSmem::total, a.stream>>>(
            a.fs, ft, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles_x,
            (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, (const float*)(a.img + a.il.final_T),
            (const uint32_t*)(a.img + a.il.tile_last), (const uint32_t*)(a.bin + a.bl.contrib), d);
        return cudaSuccess;
    };
    cudaError_t e;
    if (ft.F <= 8) e = launch(feature_bwd_det_kernel<8>);
    else if (ft.F <= 16) e = launch(feature_bwd_det_kernel<16>);
    else if (ft.F <= 24) e = launch(feature_bwd_det_kernel<24>);
    else e = launch(feature_bwd_det_kernel<32>);
    if (e != cudaSuccess) return e;
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_det_gather(const BwdArgs& a, const DetArgs& d, const FeatArgs* ft) {
    ProfileScope ps("det_gather", a.stream);
    det_gather_kernel<<<(a.cam.P + GB - 1) / GB, GB, 0, a.stream>>>(
        a.fs, a.cam.P, (long long)a.bl.capacity, d, (float*)(a.geom + a.gl.sgrad), ft ? ft->F : 0, ft ? ft->dfeat : nullptr,
        ft ? ft->dfeat_stride : 0);
    sr_count_launch();
    return cudaGetLastError();
}
