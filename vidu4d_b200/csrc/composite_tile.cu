// composite_tile.cu -- forward and backward composite with one CTA per 16x16 tile and a shared TMA chunk ring.
//
// Replaces (behaviour, not code) of the reference's renderCUDA forward / backward,
// RAST/cuda_rasterizer/forward.cu:265-463 and backward.cu:143-449.  The backward here is the only one; the forward is
// an alternative to composite_fwd.cu (the one-warp-per-CTA forward, the default) with the same per-pixel state,
// per-pair arithmetic and outputs (comp::FwdPixel) and contribution masks.  What changes is how the instance list
// reaches the lanes and how the kernel stops early:
//
//   * CTA = one tile = 8 warps (one per 8x4 sub-tile, lane = pixel).  The tile's sorted 80-byte instance records
//     stream through ONE ring of NSLOT chunks of CH instances, filled by cp.async.bulk (TMA 1-D) and shared by the 8
//     warps -- 8x less shared memory per warp than a private ring, which is what makes CH = 256 affordable.
//   * Inside a chunk every LANE walks its own list (cull masks forward, recorded contribution masks backward) without
//     any stage lock-step: the warp only re-converges at chunk boundaries.  With ~2 contributions per pixel and
//     32-instance stage, lock-step at stage granularity evaluates 12.5 pairs per 32-lane iteration on the headline
//     frame (Poisson noise: the warp waits for its busiest lane every stage); at 256 instances it is 18
//     (replay of the recorded masks).
//   * Forward: no CTA-wide barrier after start-up.  A ring slot is released by an shared-memory counter; the warp whose
//     release is the eighth issues the next bulk copy into it, so there is no producer warp to wait on.  A warp may
//     run NSLOT-1 chunks ahead of the slowest warp of its tile.
//   * Backward: two phases per chunk between CTA barriers (pixel walk -> shared pair buffer -> per-instance sums), so
//     that gradients reach L2 once per (instance, tile); see composite_tile_bwd_kernel.
//   * Forward early termination is per lane (T < 1e-4), per warp (all 32 pixels done: the warp only waits for and
//     releases the remaining chunks) and per CTA (all 8 warps done: no further chunk is requested).
#include <cstdlib>

#include "composite_common.cuh"

namespace {
using namespace comp;

constexpr int TWARPS = 8;      // 8x4 sub-tiles of a 16x16 tile

// ------------------------------------------------------------------------------------------------ forward
constexpr int FWD_CH = 256;        // instances per chunk
constexpr int FWD_NSLOT = 2;       // ring slots
struct FwdSmem {
    static constexpr int NSTG = FWD_CH / 32;                                     // 32-instance stages per chunk
    static constexpr size_t ring = (size_t)FWD_NSLOT * FWD_CH * REC4 * sizeof(float4);
    static constexpr size_t masks = (size_t)TWARPS * NSTG * 32 * sizeof(uint32_t);
    static constexpr size_t total = ring + masks + FWD_NSLOT * sizeof(uint64_t) + (FWD_NSLOT + 4) * sizeof(uint32_t);
};

__global__ void __launch_bounds__(32 * TWARPS, 4)
composite_tile_fwd_kernel(const FrameStrides fs, const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, int tiles_x,
                          const float4* __restrict__ irec, int W, int H, const float* __restrict__ bg,
                          float* __restrict__ final_T, uint32_t* __restrict__ n_contrib, float* __restrict__ out_color,
                          float* __restrict__ out_others, uint32_t* __restrict__ sub_last,
                          uint32_t* __restrict__ contrib_masks) {
    using SM = FwdSmem;
    constexpr int CH = FWD_CH, NSLOT = FWD_NSLOT, NSTG = SM::NSTG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4* ring = reinterpret_cast<float4*>(smem_raw);
    uint32_t* cm_all = reinterpret_cast<uint32_t*>(smem_raw + SM::ring);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + SM::ring + SM::masks);
    uint32_t* rel = reinterpret_cast<uint32_t*>(full + NSLOT);
    volatile uint32_t* ctl = rel + NSLOT;      // [0] warps with all 32 pixels finished, [1] first chunk that is NOT requested

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    // frames are interleaved in blockIdx.x: the longest tiles of EVERY frame of the batch start first
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_T = fr(final_T, fs.img, f); n_contrib = fr(n_contrib, fs.img, f); out_color = fr(out_color, fs.out_color, f);
    out_others = fr(out_others, fs.out_others, f); sub_last = fr(sub_last, fs.img, f); contrib_masks = fr(contrib_masks, fs.bin, f);
    const int tile = (int)tile_order[blockIdx.x / (unsigned)fs.frames];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const int len = (int)(range.y - range.x);
    const int nchunks = (len + CH - 1) / CH;
    const SubPixel sp = sub_pixel(tile_x, tile_y, warp, lane);     // warp -> 8x4 sub-tile, lane -> pixel

    const float4* src = irec + (size_t)range.x * REC4;
    auto issue = [&](int c) {   // one thread
        const int s = c % NSLOT;
        const uint32_t bytes = (uint32_t)min(CH, len - c * CH) * 80u;
        fence_proxy_async();                       // the slot's previous readers (generic proxy) are done: see release below
        mbar_expect_tx(&full[s], bytes);
        bulk_g2s(ring + (size_t)s * CH * REC4, src + (size_t)c * CH * REC4, bytes, &full[s]);
    };
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < NSLOT; s++) { mbar_init(&full[s], 1); rel[s] = 0u; }
        ctl[0] = 0u; ctl[1] = (uint32_t)nchunks;
        fence_mbar_init();
        for (int c = 0; c < NSLOT && c < nchunks; c++) issue(c);
    }
    __syncthreads();                               // the only CTA-wide barrier

    FwdPixel px;
    bool done = !sp.inside(W, H);
    bool counted = false;                          // (warp-uniform) this warp is in ctl[0]
    uint32_t* cm = cm_all + warp * NSTG * 32 + lane;          // this lane's column: cm[st * 32]
    uint32_t* cm_out = contrib_masks + contrib_word(range.x, tile, warp, lane);

    for (int c = 0; c < nchunks; c++) {
        const int s = c % NSLOT;
        {   // wait until chunk c has landed -- or learn that it was never requested (every warp finished earlier)
            const uint32_t parity = (uint32_t)((c / NSLOT) & 1);
            bool have = true;
            while (!mbar_try_wait(&full[s], parity)) {
                if ((int)ctl[1] <= c) { have = false; break; }
            }
            if (!__all_sync(0xffffffffu, have)) break;
        }
        const int cnt = min(CH, len - c * CH);
        const int nst = (cnt + 31) >> 5;
        const float4* S = ring + (size_t)s * CH * REC4;
        const bool skip = __all_sync(0xffffffffu, done);      // nothing left to do for this sub-tile
        uint32_t entered = 0u;
        if (!skip) {
            // lane = instance: cull rectangles of every stage of the chunk -> per-pixel candidate masks (lane = pixel)
            uint32_t nz = 0u;
#pragma unroll
            for (int st = 0; st < NSTG; st++) {
                if (st < nst) {
                    const int i = st * 32 + lane;
                    const uint32_t cull = i < cnt ? __float_as_uint(S[i * REC4 + 4].w) : 0u;
                    const uint32_t m = group_survivors(cull, sp.sx0, sp.sy0, lane);
                    cm[st * 32] = m;
                    if (m) nz |= 1u << st;
                }
            }
            if (done) nz = 0u;
            int st = -1;
            uint32_t mym = 0u, cmask = 0u;
            for (;;) {
                if (mym == 0u) {
                    // leave the stage (its candidate mask is replaced by the contribution mask), enter the next one
                    if (st >= 0) { cm[st * 32] = cmask; cmask = 0u; st = -1; }
                    if (nz) { st = __ffs(nz) - 1; nz &= nz - 1u; mym = cm[st * 32]; entered |= 1u << st; }
                }
                const bool act = mym != 0u;
                if (!__any_sync(0xffffffffu, act)) break;
                if (!act) continue;
                const int jj = __ffs(mym) - 1;
                mym &= mym - 1u;
                const float4* R = S + (st * 32 + jj) * REC4;
                if (px.blend(R, sp.pixx, sp.pixy, cull_rho_cut(__float_as_uint(R[4].w)), c * CH + st * 32, jj, cmask)) {
                    done = true; mym = 0u; nz = 0u;
                }
            }
            // contribution masks of the chunk (zero for the stages this pixel never reached): one 128-B store per stage
#pragma unroll
            for (int st2 = 0; st2 < NSTG; st2++)
                if (st2 < nst) cm_out[(size_t)(c * NSTG + st2) * SR_CONTRIB_STAGE_WORDS] = ((entered >> st2) & 1u) ? cm[st2 * 32] : 0u;
        }
        // release the slot; the warp whose release is the last one requests the next chunk into it
        const bool wdone = __all_sync(0xffffffffu, done);
        __syncwarp();
        if (lane == 0) {
            if (wdone && !counted) atomicAdd(const_cast<uint32_t*>(&ctl[0]), 1u);
            __threadfence_block();
            if (atomicAdd(&rel[s], 1u) == TWARPS - 1) {
                rel[s] = 0u;
                __threadfence_block();
                const int nc = c + NSLOT;
                if (nc < nchunks) {
                    if (ctl[0] == TWARPS) atomicMin(const_cast<uint32_t*>(&ctl[1]), (uint32_t)nc);
                    else issue(nc);
                }
            }
        }
        counted = counted || wdone;
    }

    // deepest list position any pixel of this sub-tile used: the backward starts its reverse walk there
    uint32_t wmax = px.last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) sub_last[tile * 8 + warp] = wmax;
    px.store(sp, W, H, bg, final_T, n_contrib, out_color, out_others);
}

// ------------------------------------------------------------------------------------------------ backward
// Every chunk is processed in two phases separated by CTA barriers, so that each (instance, tile) sends its gradient
// to L2 as ONE set of vector reductions instead of one set per contributing pixel (12 pairs per (instance, tile) on
// average on the headline frame; the per-pair reductions were what bounded this kernel):
//   1. pixel phase (lane = pixel): the reverse walk over the recorded contribution masks, reduced to three scalars per
//      pair (BwdPixel::pair_scalars) that go to a shared pair buffer.  A pair's slot is its pixel's base -- a CTA-wide
//      exclusive scan of the per-pixel pair counts of the chunk -- plus its rank in the pixel's back-to-front list.
//   2. instance phase (thread = instance of the chunk; warp w = stage w): the instance's pixel set is the transpose of
//      its stage's 32 x 32 (pixel x instance) masks.  For each of its pixels the thread runs pair_geom_vjp_stored on
//      the stored scalars -- G dL/dalpha, and the low-pass branch in the sign of alpha T, so neither G nor alpha is
//      evaluated again -- and sums the 16 + 2 components in registers; one red.v4 x 4 (+ one v2) per instance leaves.
// A pair whose slot lies beyond the buffer (a dense chunk) takes the direct path in phase 1 -- full VJP and per-pair
// reductions -- and phase 2 skips it: the capacity changes the order of the float sums and the rounding of a pair's
// terms (the direct path keeps the correctly rounded quotients), never which terms are summed.
constexpr int BWD_CAP = 4608;      // pair-buffer slots, 12 B each; headline chunks: 2,200 pairs average, 5,500 p99
struct BwdSmem {
    // offsets of the regions that follow the ring
    static constexpr size_t masks = (size_t)BWD_NSLOT * BWD_CH * REC4 * sizeof(float4);      // masks [warp][stage][lane]
    static constexpr size_t pd4 = masks + (size_t)BWD_NSTG * BWD_NPIX * sizeof(uint32_t);     // per pixel: dpix0..2, dn0
    static constexpr size_t pd2 = pd4 + BWD_NPIX * sizeof(float4);                              // per pixel: dn1, dn2
    static constexpr size_t buf = pd2 + BWD_NPIX * sizeof(float2);                              // pair buffer, 3 x BWD_CAP
    static constexpr size_t sfx = buf + 3 * (size_t)BWD_CAP * sizeof(float);                   // slot table [stage][pixel]
    static constexpr size_t full = sfx + (size_t)BWD_NSTG * BWD_NPIX * sizeof(uint16_t);       // mbarriers
    static constexpr size_t wsum = full + BWD_NSLOT * sizeof(uint64_t);                         // pair count per warp
    static constexpr size_t total = wsum + BWD_WARPS * sizeof(uint32_t);
};
static_assert(BwdSmem::full % 8 == 0, "mbarrier alignment");
static_assert(2 * (BwdSmem::total + 1024) <= 233472, "two CTAs per SM (228 KB, 1 KB reserved per CTA)");
// Deterministic instantiation (DET = true, include/surfel_deterministic.h):
//   * the (instance, tile) sum is STORED into the instance's slot det.slots[emission index] instead of reduced into the
//     per-surfel accumulator; launch_det_gather sums a surfel's slots in emission order;
//   * there is no direct path: a chunk with more pairs than BWD_CAP runs phases 1 and 2 in passes of whole pixels
//     (comp::DetPasses).  Phase 2 of pass k > 0 resumes from the partial sum pass k-1 stored in the slot.  Phase 2 adds
//     an instance's pixels in ascending pixel order whatever the passes, so the sum is the one a single pass would
//     form, and no pair takes the full VJP.

template <bool DET>
__global__ void __launch_bounds__(BWD_NPIX, 2)
composite_tile_bwd_kernel(const FrameStrides fs, const float* __restrict__ grad_scale, const uint2* __restrict__ ranges,
                          const uint32_t* __restrict__ tile_order, int tiles_x,
                          const float4* __restrict__ irec, int W, int H, const float* __restrict__ bg,
                          const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib,
                          const uint32_t* __restrict__ sub_last, const float* __restrict__ dL_dpixels,
                          const float* __restrict__ dL_dothers, const uint32_t* __restrict__ contrib_masks,
                          float* __restrict__ sgrad, const DetArgs det) {
    using SM = BwdSmem;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    uint32_t* cm_all = reinterpret_cast<uint32_t*>(smem_raw + SM::masks);
    float4* pd4 = reinterpret_cast<float4*>(smem_raw + SM::pd4);
    float2* pd2 = reinterpret_cast<float2*>(smem_raw + SM::pd2);
    float* buf_a = reinterpret_cast<float*>(smem_raw + SM::buf);     // G times dL/dalpha (times T, with the background term)
    float* buf_z = buf_a + BWD_CAP;                                   // dL/dz
    float* buf_t = buf_z + BWD_CAP;                                   // alpha T, negated on the low-pass branch
    uint16_t* sfx = reinterpret_cast<uint16_t*>(smem_raw + SM::sfx);  // first slot of (stage, pixel)'s pairs
    uint32_t* wsum = reinterpret_cast<uint32_t*>(smem_raw + SM::wsum);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_Ts = fr(final_Ts, fs.img, f); n_contrib = fr(n_contrib, fs.img, f); sub_last = fr(sub_last, fs.img, f);
    dL_dpixels = fr(dL_dpixels, fs.dcolor, f); dL_dothers = fr(dL_dothers, fs.dothers, f);
    contrib_masks = fr(contrib_masks, fs.bin, f); sgrad = fr(sgrad, fs.geom, f);
    float* slots = nullptr;
    const uint32_t* point_offsets = nullptr;
    const int* radii = nullptr;
    if constexpr (DET) {
        slots = fr(det.slots, det.slots_stride, f); point_offsets = fr(det.point_offsets, fs.geom, f); radii = fr(det.radii, fs.radii, f);
    }
    const int tile = (int)tile_order[blockIdx.x / (unsigned)fs.frames];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const BwdTile bt = bwd_tile(range, sub_last, tile);
    if (bt.nchunks == 0) return;                   // CTA-uniform
    const int nb_w = bt.nb_w();
    const ChunkRing ring{reinterpret_cast<float4*>(smem_raw), reinterpret_cast<uint64_t*>(smem_raw + SM::full),
                         irec + (size_t)range.x * REC4, bt.len, bt.nchunks};
    if (threadIdx.x == 0) ring.init();

    BwdPixel px;
    px.load(sub_pixel(tile_x, tile_y, warp, lane), W, H, bg, final_Ts, n_contrib, dL_dpixels, dL_dothers, grad_scale);
    pd4[threadIdx.x] = make_float4(px.dpix0, px.dpix1, px.dpix2, px.dn0);      // thread == pixel == warp * 32 + lane
    pd2[threadIdx.x] = make_float2(px.dn1, px.dn2);

    PixelMasks masks{cm_all + warp * BWD_NSTG * 32 + lane, contrib_masks + contrib_word(range.x, tile, warp, lane),
                     nb_w};
    masks.fetch(bt.nchunks - 1);

    for (int k = 0; k < bt.nchunks; k++) {
        const int c = bt.nchunks - 1 - k, s = k % BWD_NSLOT;
        int np, total = 0;
        const uint32_t nz = masks.install(np);
        const int base = masks.scan(np, wsum, sfx);
        if constexpr (DET) for (int w = 0; w < BWD_WARPS; w++) total += (int)wsum[w];
        const DetPasses dp(total, BWD_CAP, BWD_CH);                // one pass unless DET
        const int my_pass = dp.of(base);
        if (c > 0) masks.fetch(c - 1);
        const float4* S = ring.wait(k, s);

        for (int pass = 0; pass < dp.npass; pass++) {
            if (pass > 0) __syncthreads();         // the previous pass's phase 2 is done with the buffer
            const int off = dp.offset(pass);
            // ---- phase 1: lane = pixel, back to front over its contributors
            uint32_t nzp = my_pass == pass ? nz : 0u;
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
                    const int idx = st * 32 + jj;
                    PairAlpha q;
                    float dL_dalpha, dL_dz, aT;
                    px.pair_scalars(S + idx * REC4, c * BWD_CH + idx, q, dL_dalpha, dL_dz, aT);
                    if (DET || slot < BWD_CAP) {
                        // aT > 0: a recorded contributor has alpha >= 1/255, and T >= T_final >= 1e-4 (the walk back
                        // multiplies T by 1/(1 - alpha) > 1), so aT's sign bit is free to carry the low-pass branch
                        const int b = slot - off;
                        buf_a[b] = q.G_ * dL_dalpha; buf_z[b] = dL_dz; buf_t[b] = (q.rho3d <= q.rho2d) ? aT : -aT;
                    } else {
                        float v[16];
#pragma unroll
                        for (int i = 0; i < 10; i++) v[i] = 0.f;
                        float m2x = 0.f, m2y = 0.f;
                        bool lowpass = false;
                        px.pair_vjp(S + idx * REC4, q, dL_dalpha, dL_dz, aT, v, m2x, m2y, lowpass);
                        red_pixel(sgrad, S + idx * REC4, v, m2x, m2y, lowpass);
                    }
                    slot++;
                }
            }
            __syncthreads();                       // pair buffer and slot table complete

            // ---- phase 2: thread = instance warp * 32 + lane of the chunk
            const InstancePixels ip(cm_all);
            if (ip.any) {
                const float4* R = S + threadIdx.x * REC4;
                const float4 r0 = R[0], r1 = R[1], r2 = R[2];
                float acc[16];
#pragma unroll
                for (int i = 0; i < 16; i++) acc[i] = 0.f;
                float a2x = 0.f, a2y = 0.f;
                bool lowpass_any = false, any_in = false;
                float* gslot = nullptr;
                if constexpr (DET) {
                    gslot = slots + (size_t)sr_emission_index(point_offsets, radii, __float_as_uint(R[4].z), r2.y, r2.z, tile_x,
                                                              tile_y, tiles_x, det.tiles_y) * SR_GRAD_FLOATS;
                    if (pass > 0) slot_load(gslot, acc, a2x, a2y);     // resume the partial sum of the earlier passes
                }
                ip.walk(cm_all, sfx, dp, pass, [&](int p, int sw, int l, int b) {
                    if (!DET && b >= BWD_CAP) return;      // went out directly in phase 1
                    const SubPixel pp = sub_pixel(tile_x, tile_y, sw, l);
                    const float t = buf_t[b];
                    const bool lowpass = t < 0.f;
                    pair_geom_vjp_stored(r0, r1, r2, pp.pixx, pp.pixy, buf_a[b], buf_z[b], lowpass, acc, a2x, a2y);
                    const float aT = fabsf(t);
                    const float4 d4 = pd4[p];
                    const float2 d2 = pd2[p];
                    acc[10] += aT * d4.x; acc[11] += aT * d4.y; acc[12] += aT * d4.z;
                    acc[13] += aT * d4.w; acc[14] += aT * d2.x; acc[15] += aT * d2.y;
                    lowpass_any |= lowpass;
                    any_in = true;
                });
                if constexpr (DET) {
                    if (any_in) slot_store(gslot, acc, a2x, a2y);
                } else if (any_in) {
                    float* gp = sgrad + (size_t)__float_as_uint(R[4].z) * SR_GRAD_FLOATS;
                    red_add<16>(gp, acc);
                    if (lowpass_any) {
                        const float w2[16] = {a2x, a2y};
                        red_add<2>(gp + SR_G_M2D, w2);
                    }
                }
            }
        }
        __syncthreads();                           // ring slot, masks, pair buffer and slot table are free again
        if (threadIdx.x == 0 && k + BWD_NSLOT < bt.nchunks) ring.issue(k + BWD_NSLOT);
    }
}

}  // namespace

// Which composite forward runs: SURFEL_COMPOSITE_FWD (or SURFEL_COMPOSITE) = tile|warp.  Default: one-warp CTAs with
// private rings (composite_fwd.cu).  On the headline 8-frame batch the tile forward is faster, with 1 frame per call
// slower (DESIGN.md 3.3).
bool sr_composite_tile_fwd() {
    static const bool tile = [] {
        const char* e = getenv("SURFEL_COMPOSITE_FWD");
        if (!e) e = getenv("SURFEL_COMPOSITE");
        return e && e[0] == 't';
    }();
    return tile;
}

cudaError_t launch_composite_tile_fwd(const FwdArgs& a) {
    ProfileScope ps("composite_fwd", a.stream);
    cudaError_t err = sr_opt_in_smem(composite_tile_fwd_kernel, FwdSmem::total);
    if (err != cudaSuccess) return err;
    composite_tile_fwd_kernel<<<a.il.tiles * a.fs.frames, 32 * TWARPS, FwdSmem::total, a.stream>>>(
        a.fs, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles_x,
        (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
        (float*)(a.img + a.il.final_T), (uint32_t*)(a.img + a.il.n_contrib), a.out_color, a.out_others,
        (uint32_t*)(a.img + a.il.tile_last), (uint32_t*)(a.bin + a.bl.contrib));
    sr_count_launch();
    return cudaGetLastError();
}

template <bool DET>
static cudaError_t launch_tile_bwd(const BwdArgs& a, const DetArgs& d) {
    if (!DET) {
        cudaError_t e = sr_memset_frames(a.geom + a.gl.sgrad, (size_t)a.fs.geom, (size_t)(a.cam.P > 0 ? a.cam.P : 1) * SR_GRAD_FLOATS * 4,
                                         a.fs.frames, a.stream);
        if (e != cudaSuccess) return e;
    }
    ProfileScope ps(DET ? "composite_bwd_det" : "composite_bwd", a.stream);
    cudaError_t e = sr_opt_in_smem(composite_tile_bwd_kernel<DET>, BwdSmem::total);
    if (e != cudaSuccess) return e;
    composite_tile_bwd_kernel<DET><<<a.il.tiles * a.fs.frames, BWD_NPIX, BwdSmem::total, a.stream>>>(
        a.fs, a.grad_scale, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles_x,
        (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
        (const float*)(a.img + a.il.final_T), (const uint32_t*)(a.img + a.il.n_contrib),
        (const uint32_t*)(a.img + a.il.tile_last), a.dL_dcolor, a.dL_dothers,
        (const uint32_t*)(a.bin + a.bl.contrib), (float*)(a.geom + a.gl.sgrad), d);
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_composite_tile_bwd(const BwdArgs& a) { return launch_tile_bwd<false>(a, DetArgs{}); }
cudaError_t launch_composite_tile_bwd_det(const BwdArgs& a, const DetArgs& d) { return launch_tile_bwd<true>(a, d); }
