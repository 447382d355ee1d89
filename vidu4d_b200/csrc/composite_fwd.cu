// composite_fwd.cu -- per-tile front-to-back alpha composite of colour / depth / normal / distortion.
//
// Replaces (behaviour, not code) of the reference's forward renderCUDA, RAST/cuda_rasterizer/forward.cu:265-463.
//
// Design (DESIGN.md "composite"):
//   * work item = (tile, 8x4 sub-tile) = one warp = one CTA, launched longest-tile-first; each warp streams the
//     tile's sorted instance records (80 B each, contiguous) through its own double-buffered shared-memory ring
//     (comp::Ring: cp.async.bulk, TMA 1-D, on its own mbarriers) -- no CTA-wide synchronisation;
//   * one pixel per lane.  Per 32-record stage, lane = instance turns the instance's conservative cull rectangle into
//     column and row masks of the sub-tile (group_survivors); then each lane walks its own survivor list, so up to 32
//     different instances are evaluated per warp iteration.  With ~5x5-pixel footprints a whole-warp 8x4 block
//     wastes most lanes;
//   * per stage and pixel the kernel records which instances contributed (one 128-B store per warp): the backward
//     walks exactly those;
//   * culling and the rho_cut early-out never change a result: a skipped pair provably has alpha < 1/255;
//   * the per-pixel state, per-pair arithmetic and output words are comp::FwdPixel's, shared with the tile forward
//     (composite_tile.cu): the two differ only in how records reach the lanes and how they stop early;
//   * two instantiations (DESIGN.md "forward-only render").  TRAIN records the contribution masks, sub_last, final_T and
//     n_contrib for the backward; the forward-only one (sr_render_forward) records none of them and composites up to NF
//     feature channels inside the same walk, through FwdPixel::blend's per-pair hook: acc[k] = ff(T, fm(alpha, x[k]),
//     acc[k]) over the same contributors, weights and order as feature_fwd, so every plane has feature_fwd's bits;
//   * STATS (sr_render_forward_contrib, DESIGN.md "contribution statistics"): the same hook also gathers each surfel's
//     blending weight w = ff(T, alpha, 0) -- the feature plane of a feature equal to 1 -- into per-warp shared slots, one
//     per instance of the stage, with integer shared atomics; after the stage lane i adds slot i to its surfel with one
//     global integer atomic each.  Integer sums and an unsigned max are exact and order-independent: the totals have
//     the same bits whatever the order of the pairs, frames, chunks or ranks;
//   * MASKED statistics (sr_render_forward_contrib_masked): each lane reads its pixel's foreground byte once, before
//     the walk, and adds its pairs into a foreground or a background set of slots.  The flush adds both sets into the
//     three words above, which get the unmasked walk's bits, and the background set alone into weight_bg_q and
//     pixels_bg;
//   * LIFT (sr_render_forward_lift, DESIGN.md "lifting maps"): the WEIGHTS words, plus each surfel's weighted sum of
//     C <= LW caller-supplied per-pixel values.  Each lane reads its pixel's C values once, before the walk; per pair and
//     channel q = rn(fm(fm(w, v), 2^s)) is added into per-warp shared slots with two native 32-bit shared atomics, and
//     after the stage lane i adds its instance's non-zero slots to lift[surfel * C + c] with 64-bit global atomics.
//     Colour only (NF = 0): the staged values take the feature accumulator's registers.
//   * ANCHORS (sr_render_forward_anchors, DESIGN.md "anchors"): each lane keeps its pixel's KA heaviest contributing pairs
//     in registers as (surfel id, w, u, v), w the statistics' weight and (u, v) where the pixel's ray hits the disc, and
//     writes them after the walk.  No atomics and no cross-lane traffic; colour only (NF = 0).
#include "composite_common.cuh"

namespace {
using namespace comp;

constexpr int WPC = 1;      // independent warps per CTA (2 measured slower: register pressure)

// What the forward-only walk gathers besides its outputs: nothing, the contribution statistics, the statistics and
// their share on the frame's background pixels, the statistics and the lifted per-pixel values, or each pixel's
// heaviest pairs alone
enum class Stats { OFF, WEIGHTS, MASKED, LIFT, ANCHORS };

// A stage's statistics slots, per warp and instance jj: lo[jj] sums the low 16 bits of q = rn(w 2^32), hc[jj] the high
// 16 bits plus 2^21 per pair.  q < 2^32 (w <= 0.99) and a stage has at most 32 pairs per instance, so neither word
// overflows (32 (2^16 - 1) < 2^21, 32 < 2^11) and the stage's sum is (hc mod 2^21) 2^16 + lo, its pair count hc >> 21.
struct StatSlots {
    uint32_t lo[WB], hc[WB], mx[WB];
};
__device__ __forceinline__ void stat_pair(StatSlots* ss, int jj, float T, float alpha) {
    const float w = ff(T, alpha, 0.0f);
    const uint32_t q = __float2uint_rn(fm(w, 4294967296.0f));
    atomicAdd(&ss->lo[jj], q & 0xffffu);
    atomicAdd(&ss->hc[jj], (q >> 16) + (1u << 21));
    atomicMax(&ss->mx[jj], __float_as_uint(w));
}
// MASKED: two such sets, [0] for the pairs on foreground pixels and [1] for those on background pixels.  A lane's pixel
// is one or the other for the whole walk, so each lane adds into one set with stat_pair's three atomics; the flush adds
// both sets into weight_q / max_weight / pixels and set [1] alone into weight_bg_q / pixels_bg.
struct MaskedSlots {
    StatSlots set[2];
};
// LIFT: a stage's channel sums, per warp, channel c and instance jj, as q = hi 2^16 + lo: lo[c][jj] sums the low 16 bits
// of each q, hi[c][jj] the rest (q >> 16, arithmetic).  sm_90 has no native 64-bit shared add (atomicAdd on a 64-bit
// shared word is a compare-and-swap loop); two 32-bit adds are.  |q| <= 2^32 and a stage has at most 32 pairs per
// instance, so neither word overflows (32 (2^16 - 1) < 2^21, 32 (2^16 + 1) < 2^31).  Channel-major, so that the
// flush's lanes (lane = instance) read consecutive words.
template <int LW>
struct LiftSlots {
    uint32_t lo[LW][WB];
    int32_t hi[LW][WB];
};
// One pair's C <= LW channels: q = rn(fm(fm(w, v), scale)), scale = 2^s, clamped to +-2^32 (each clamp counts in sat).
// v holds the lane's staged values, 0 for a non-finite one, and nbad the number of those, which count once per pair:
// they contribute 0.  fm(p, 2^s) is exact unless it leaves float's normal range; below it the exact product rounds to
// 0 as well, above it is clamped.  A zero q skips its atomics (padding channels are always 0).
template <int LW>
__device__ __forceinline__ void lift_pair(LiftSlots<LW>* ls, int jj, float w, const float (&v)[LW], float scale,
                                          uint32_t nbad, uint32_t& sat) {
    sat += nbad;
#pragma unroll
    for (int c = 0; c < LW; c++) {
        const float x = fm(fm(w, v[c]), scale);
        long long q;
        if (fabsf(x) > 4294967296.0f) {
            q = x > 0.0f ? (1ll << 32) : -(1ll << 32);
            sat++;
        } else {
            q = __float2ll_rn(x);
        }
        if (q != 0) {
            atomicAdd(&ls->lo[c][jj], (uint32_t)q & 0xffffu);
            atomicAdd(&ls->hi[c][jj], (int32_t)(q >> 16));
        }
    }
}

// ANCHORS: a pixel's KA heaviest pairs so far, sorted by w descending; among equal weights the earlier pair (the
// front-most: the walk's order is fixed) stays ahead.  Empty slots hold id -1, w 0 and uv (0, 0); every contributing
// pair has w > 0 (T >= 1e-4, alpha >= 1/255), so it enters an empty slot.
template <int KA>
struct AnchorSlots {
    int32_t id[KA];
    float w[KA], u[KA], v[KA];
    __device__ __forceinline__ void clear() {
#pragma unroll
        for (int k = 0; k < KA; k++) { id[k] = -1; w[k] = 0.f; u[k] = 0.f; v[k] = 0.f; }
    }
    // A pair enters if its w is strictly larger than the last slot's: it takes the first slot of smaller weight and
    // every slot from there on takes its predecessor's content (selects only: the slots stay in registers).
    __device__ __forceinline__ void add(int32_t pid, float pw, float pu, float pv) {
        bool shift = false;
#pragma unroll
        for (int k = 0; k < KA; k++) {
            const bool take = shift || pw > w[k];
            const int32_t ti = id[k]; const float tw = w[k], tu = u[k], tv = v[k];
            if (take) { id[k] = pid; w[k] = pw; u[k] = pu; v[k] = pv; pid = ti; pw = tw; pu = tu; pv = tv; }
            shift = take;
        }
    }
};

// TRAIN: the training forward (V, NF, STATS, LW unused).  Otherwise forward-only with F <= NF feature channels (NF = 0:
// none), rows gathered V floats per load, and with STATS != OFF the contribution statistics added into cs; with
// STATS == LIFT (NF = 0) also the lift of cs.lift_C <= LW channels.  With STATS == ANCHORS (NF = 0) LW is the slot
// count KA instead, and nothing is added into the statistics.
template <bool TRAIN, int V, int NF, Stats STATS = Stats::OFF, int LW = 0>
__global__ void __launch_bounds__(32 * WPC)
composite_fwd_kernel(const FrameStrides fs, const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, int n_items, int tiles_x,
                     const float4* __restrict__ irec, int W, int H,
                     const float* __restrict__ bg, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                     float* __restrict__ out_color, float* __restrict__ out_others, uint32_t* __restrict__ sub_last,
                     uint32_t* __restrict__ contrib_masks, const FeatArgs ft, const ContribArgs cs) {
    static_assert(STATS != Stats::LIFT || (NF == 0 && LW > 0 && LW <= 32), "a lift is a colour-only walk of 1..32 channels");
    static_assert(STATS != Stats::ANCHORS || (NF == 0 && (LW == 1 || LW == 2 || LW == 4 || LW == 8)),
                  "anchors are a colour-only walk of 1, 2, 4 or 8 slots");
    // WPC independent warps per CTA (the SM holds at most 32 CTAs): work item = (tile, 8x4 sub-tile), tiles in
    // longest-list-first order; the warps of a CTA share nothing
    __shared__ __align__(128) float4 st_all[WPC][NST][WB * REC4];
    __shared__ __align__(8) uint64_t bar_all[WPC][NST];
    float4 (*st)[WB * REC4] = st_all[threadIdx.x >> 5];
    uint64_t* bar = bar_all[threadIdx.x >> 5];

    const int lane = threadIdx.x & 31;
    // frames are interleaved in blockIdx.x: the longest tiles of EVERY frame of the batch start first
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    const int item = (int)(blockIdx.x / (unsigned)fs.frames) * WPC + (threadIdx.x >> 5);
    if (item >= n_items) return;
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_T = fr(final_T, fs.img, f); n_contrib = fr(n_contrib, fs.img, f); out_color = fr(out_color, fs.out_color, f);
    out_others = fr(out_others, fs.out_others, f); sub_last = fr(sub_last, fs.img, f); contrib_masks = fr(contrib_masks, fs.bin, f);
    const int warp = item & 7;
    const int tile = (int)tile_order[item >> 3];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const int len = (int)(range.y - range.x);
    const int nb = (len + WB - 1) / WB;
    const SubPixel sp = sub_pixel(tile_x, tile_y, warp, lane);     // warp -> 8x4 sub-tile, lane -> pixel

    Ring ring{st, bar, irec + (size_t)range.x * REC4, len};
    if (lane == 0) {
        ring.init();
        for (int b = 0; b < NST && b < nb; b++) ring.issue(b, b);
    }
    StatSlots* ss = nullptr;
    if constexpr (STATS == Stats::WEIGHTS || STATS == Stats::LIFT) {
        __shared__ StatSlots ss_all[WPC];
        ss = &ss_all[threadIdx.x >> 5];
        ss->lo[lane] = 0u; ss->hc[lane] = 0u; ss->mx[lane] = 0u;
    }
    // LIFT: the warp's channel slots, and this lane's pixel's values in frame f, read once here (0 outside the image, for
    // the padding channels c >= C and for a non-finite value, which nbad counts)
    constexpr int LS = LW > 0 ? LW : 1;
    LiftSlots<LS>* ls = nullptr;
    float lv[LS];
    uint32_t nbad = 0u, sat = 0u;
    if constexpr (STATS == Stats::LIFT) {
        __shared__ LiftSlots<LW> ls_all[WPC];
        ls = &ls_all[threadIdx.x >> 5];
        const bool in = sp.inside(W, H);
        const size_t N = (size_t)W * H;
        const float* v = fr(cs.lift_values, cs.lift_stride, f) + (in ? (size_t)W * sp.pix_y + sp.pix_x : 0);
#pragma unroll
        for (int c = 0; c < LW; c++) {
            ls->lo[c][lane] = 0u; ls->hi[c][lane] = 0;
            const float x = (in && c < cs.lift_C) ? __ldg(v + (size_t)c * N) : 0.0f;
            const bool ok = isfinite(x);
            nbad += ok ? 0u : 1u;
            lv[c] = ok ? x : 0.0f;
        }
    }
    // MASKED: the warp's two sets, and the one this lane's pairs add into, chosen by its pixel's mask byte in frame f,
    // read once here (a pixel outside the image has no pairs)
    MaskedSlots* sm = nullptr;
    if constexpr (STATS == Stats::MASKED) {
        __shared__ MaskedSlots sm_all[WPC];
        sm = &sm_all[threadIdx.x >> 5];
        for (int k = 0; k < 2; k++) { sm->set[k].lo[lane] = 0u; sm->set[k].hc[lane] = 0u; sm->set[k].mx[lane] = 0u; }
        const bool bg_pixel =
            sp.inside(W, H) && __ldg(fr(cs.mask, cs.mask_stride, f) + (size_t)W * sp.pix_y + sp.pix_x) == 0;
        ss = &sm->set[bg_pixel ? 1 : 0];
    }
    __syncwarp();
    // ANCHORS: this lane's pixel's slots
    constexpr int KA = STATS == Stats::ANCHORS ? LW : 1;
    AnchorSlots<KA> anc;
    if constexpr (STATS == Stats::ANCHORS) anc.clear();

    FwdPixel px;
    bool done = !sp.inside(W, H);
    // instances of the current stage that contributed to this lane's pixel, kept for the backward: a warp's 32 words
    // are one 128-B store
    uint32_t cmask = 0u;
    uint32_t* cm_out = contrib_masks + contrib_word(range.x, tile, warp, lane);
    // forward-only: this lane's feature planes, composited as feature_fwd composites them
    const int F = ft.F;
    const float* feat = fr(ft.feat, ft.feat_stride, f);
    float facc[NF > 0 ? NF : 1];
#pragma unroll
    for (int k = 0; k < (NF > 0 ? NF : 1); k++) facc[k] = 0.f;
    auto feat_pair = [&](float T, float alpha, const float4* __restrict__ R) {
        if constexpr (NF > 0) {
            float x[NF];
            load_chunk<V>(feat + (size_t)__float_as_uint(R[4].z) * F, 0, F, x);
#pragma unroll
            for (int k = 0; k < NF; k++) facc[k] = ff(T, fm(alpha, x[k]), facc[k]);
        }
    };

    for (int b = 0; b < nb; b++) {
        const float4* S = ring.wait(b);
        const int cnt = min(WB, len - b * WB);
        uint32_t cull = 0;
        if (lane < cnt) cull = __float_as_uint(S[lane * REC4 + 4].w);
        // lane = instance: which pixels does this instance's cull rectangle touch?
        uint32_t mym = group_survivors(cull, sp.sx0, sp.sy0, lane);
        {   // a finished pixel must not keep the warp iterating over its survivors
            const uint32_t db = __ballot_sync(0xffffffffu, done);
            if ((db >> lane) & 1u) mym = 0u;
        }
        while (__any_sync(0xffffffffu, mym != 0u)) {
            const bool act = mym != 0u;
            const int jj = act ? __ffs(mym) - 1 : 0;
            mym &= mym - 1;                              // no-op when mym == 0
            const float rho_cut = cull_rho_cut(__shfl_sync(0xffffffffu, cull, jj));   // before any divergence
            if (!act || done) continue;
            if constexpr (TRAIN) {
                if (px.blend(S + jj * REC4, sp.pixx, sp.pixy, rho_cut, b * WB, jj, cmask)) done = true;
            } else if constexpr (STATS == Stats::OFF) {
                if (px.blend(S + jj * REC4, sp.pixx, sp.pixy, rho_cut, b * WB, jj, cmask, feat_pair)) done = true;
            } else if constexpr (STATS == Stats::ANCHORS) {
                // the screen-space filter branch blends the centre's depth: its anchor is the centre, (0, 0)
                auto pair = [&](float T, float alpha, const float4* __restrict__ R, float sx, float sy, bool disc) {
                    anc.add((int32_t)__float_as_uint(R[4].z), ff(T, alpha, 0.0f), disc ? sx : 0.0f, disc ? sy : 0.0f);
                };
                if (px.blend(S + jj * REC4, sp.pixx, sp.pixy, rho_cut, b * WB, jj, cmask, pair)) done = true;
            } else {
                auto pair = [&](float T, float alpha, const float4* __restrict__ R) {
                    feat_pair(T, alpha, R);
                    stat_pair(ss, jj, T, alpha);
                    if constexpr (STATS == Stats::LIFT) lift_pair(ls, jj, ff(T, alpha, 0.0f), lv, cs.lift_scale, nbad, sat);
                };
                if (px.blend(S + jj * REC4, sp.pixx, sp.pixy, rho_cut, b * WB, jj, cmask, pair)) done = true;
            }
        }
        __syncwarp();                                   // every lane is done reading stage b
        if constexpr (STATS == Stats::WEIGHTS || STATS == Stats::LIFT) {
            // lane = instance: its stage totals go to its surfel, and its slot is cleared for the next stage
            const uint32_t hc = ss->hc[lane];
            if (hc != 0u) {
                const uint32_t id = __float_as_uint(S[lane * REC4 + 4].z);
                atomicAdd(cs.weight_q + id, ((unsigned long long)(hc & 0x1fffffu) << 16) + ss->lo[lane]);
                atomicMax(cs.max_weight + id, ss->mx[lane]);
                atomicAdd(cs.pixels + id, (unsigned long long)(hc >> 21));
                ss->lo[lane] = 0u; ss->hc[lane] = 0u; ss->mx[lane] = 0u;
                if constexpr (STATS == Stats::LIFT) {
                    // and its non-zero channel sums to lift[id * C + c] (two's complement: an unsigned add)
                    unsigned long long* dst = reinterpret_cast<unsigned long long*>(cs.lift_sums) + (size_t)id * cs.lift_C;
#pragma unroll
                    for (int c = 0; c < LW; c++) {
                        const uint32_t lo = ls->lo[c][lane];
                        const int32_t hi = ls->hi[c][lane];
                        if ((lo | (uint32_t)hi) != 0u) {
                            const long long q = (long long)hi * 65536 + (long long)lo;
                            if (q != 0) atomicAdd(dst + c, (unsigned long long)q);
                            ls->lo[c][lane] = 0u; ls->hi[c][lane] = 0;
                        }
                    }
                }
            }
        }
        if constexpr (STATS == Stats::MASKED) {
            // the same, with both sets' totals in the three words and the background set's in its two
            StatSlots& fg = sm->set[0];
            StatSlots& bk = sm->set[1];
            const uint32_t hf = fg.hc[lane], hb = bk.hc[lane];
            if ((hf | hb) != 0u) {
                const uint32_t id = __float_as_uint(S[lane * REC4 + 4].z);
                const unsigned long long qf = ((unsigned long long)(hf & 0x1fffffu) << 16) + fg.lo[lane];
                const unsigned long long qb = ((unsigned long long)(hb & 0x1fffffu) << 16) + bk.lo[lane];
                atomicAdd(cs.weight_q + id, qf + qb);
                atomicMax(cs.max_weight + id, max(fg.mx[lane], bk.mx[lane]));
                atomicAdd(cs.pixels + id, (unsigned long long)((hf >> 21) + (hb >> 21)));
                if (hb != 0u) {
                    atomicAdd(cs.weight_bg_q + id, qb);
                    atomicAdd(cs.pixels_bg + id, (unsigned long long)(hb >> 21));
                }
                for (int k = 0; k < 2; k++) { sm->set[k].lo[lane] = 0u; sm->set[k].hc[lane] = 0u; sm->set[k].mx[lane] = 0u; }
            }
        }
        if constexpr (STATS != Stats::OFF && STATS != Stats::ANCHORS) {
            __syncwarp();                               // slots cleared and stage b read before its slot is refilled
        }
        if constexpr (TRAIN) cm_out[(size_t)b * SR_CONTRIB_STAGE_WORDS] = cmask;
        cmask = 0u;
        if (__all_sync(0xffffffffu, done)) {
            // drain the copies still in flight before this warp (and its CTA's smem) goes away
            for (int b2 = b + 1; b2 < nb && b2 < b + NST; b2++) ring.wait(b2);
            break;
        }
        if (lane == 0 && b + NST < nb) ring.issue(b + NST, b + NST);
    }

    if constexpr (TRAIN) {
        // deepest list position any pixel of this sub-tile used: the backward starts its reverse walk there
        uint32_t wmax = px.last_contributor;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
        if (lane == 0) sub_last[tile * 8 + warp] = wmax;
        px.store(sp, W, H, bg, final_T, n_contrib, out_color, out_others);
    } else {
        if constexpr (STATS == Stats::LIFT) {
            // the warp's clamped and non-finite (pair, channel) count: one global atomic per warp, when non-zero
            unsigned long long n = sat;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
            if (lane == 0 && n != 0ull) atomicAdd(cs.lift_saturated, n);
        }
        px.store(sp, W, H, bg, out_color, out_others);
        if constexpr (STATS == Stats::ANCHORS) {
            // every slot, empty ones included, unless the frame overflowed (its walk saw no pairs; the caller re-runs it)
            if (sp.inside(W, H) && !(__ldg(fr(cs.anchor_status, fs.nr, f)) & SR_STATUS_OVERFLOW)) {
                const size_t N = (size_t)W * H, pid = (size_t)W * sp.pix_y + sp.pix_x;
                int32_t* ids = fr(cs.anchor_ids, cs.anchor_stride * 4, f) + pid;
                float* ws = fr(cs.anchor_w, cs.anchor_stride * 4, f) + pid;
                float* uv = fr(cs.anchor_uv, cs.anchor_stride * 8, f) + pid;
#pragma unroll
                for (int k = 0; k < KA; k++) {
                    ids[k * N] = anc.id[k];
                    ws[k * N] = anc.w[k];
                    uv[2 * k * N] = anc.u[k];
                    uv[(2 * k + 1) * N] = anc.v[k];
                }
            }
        }
        if constexpr (NF > 0) {
            if (sp.inside(W, H)) {
                const size_t N = (size_t)W * H, pid = (size_t)W * sp.pix_y + sp.pix_x;
                float* out = fr(ft.out, ft.out_stride, f);
#pragma unroll
                for (int k = 0; k < NF; k++)
                    if (k < F) out[(size_t)k * N + pid] = ft.bg ? ff(px.T, __ldg(ft.bg + k), facc[k]) : ff(px.T, 0.0f, facc[k]);
            }
        }
    }
}

// the forward-only instantiation for F channels (NF = F rounded up to a multiple of 8), vector width ft.vec and, with
// STATS != OFF, the statistics cs
template <int NF, Stats STATS, int LW = 0>
void launch_render(const FwdArgs& a, const FeatArgs& ft, const ContribArgs& cs, unsigned grid) {
    auto launch = [&](auto kern) {
        kern<<<grid, 32 * WPC, 0, a.stream>>>(
            a.fs, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles * 8, a.il.tiles_x,
            (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg, nullptr, nullptr, a.out_color, a.out_others,
            nullptr, nullptr, ft, cs);
    };
    if constexpr (NF == 0) launch(composite_fwd_kernel<false, 1, 0, STATS, LW>);
    else if (ft.vec == 4) launch(composite_fwd_kernel<false, 4, NF, STATS>);
    else if (ft.vec == 2) launch(composite_fwd_kernel<false, 2, NF, STATS>);
    else launch(composite_fwd_kernel<false, 1, NF, STATS>);
}
template <Stats STATS>
void launch_render_f(const FwdArgs& a, const FeatArgs& ft, const ContribArgs& cs, unsigned grid) {
    if (ft.F == 0) launch_render<0, STATS>(a, ft, cs, grid);
    else if (ft.F <= 8) launch_render<8, STATS>(a, ft, cs, grid);
    else if (ft.F <= 16) launch_render<16, STATS>(a, ft, cs, grid);
    else if (ft.F <= 24) launch_render<24, STATS>(a, ft, cs, grid);
    else launch_render<32, STATS>(a, ft, cs, grid);
}
// the lift's instantiation for C channels (LW = C rounded up to a multiple of 8); no feature channels
void launch_lift(const FwdArgs& a, const ContribArgs& cs, unsigned grid) {
    const FeatArgs ft{};
    if (cs.lift_C <= 8) launch_render<0, Stats::LIFT, 8>(a, ft, cs, grid);
    else if (cs.lift_C <= 16) launch_render<0, Stats::LIFT, 16>(a, ft, cs, grid);
    else if (cs.lift_C <= 24) launch_render<0, Stats::LIFT, 24>(a, ft, cs, grid);
    else launch_render<0, Stats::LIFT, 32>(a, ft, cs, grid);
}
// the anchors' instantiation for K slots; no feature channels
void launch_anchors(const FwdArgs& a, const ContribArgs& cs, unsigned grid) {
    const FeatArgs ft{};
    if (cs.anchor_K == 1) launch_render<0, Stats::ANCHORS, 1>(a, ft, cs, grid);
    else if (cs.anchor_K == 2) launch_render<0, Stats::ANCHORS, 2>(a, ft, cs, grid);
    else if (cs.anchor_K == 4) launch_render<0, Stats::ANCHORS, 4>(a, ft, cs, grid);
    else launch_render<0, Stats::ANCHORS, 8>(a, ft, cs, grid);
}

}  // namespace

cudaError_t launch_composite_fwd(const FwdArgs& a) {
    const unsigned grid = (unsigned)((a.il.tiles * 8 + WPC - 1) / WPC) * (unsigned)a.fs.frames;
    if (a.forward_only) {
        ProfileScope ps("composite_render", a.stream);
        const FeatArgs ft = a.feat ? *a.feat : FeatArgs{};
        if (!a.contrib) launch_render_f<Stats::OFF>(a, ft, ContribArgs{}, grid);
        else if (a.contrib->anchors) launch_anchors(a, *a.contrib, grid);
        else if (a.contrib->lift) launch_lift(a, *a.contrib, grid);
        else if (a.contrib->mask) launch_render_f<Stats::MASKED>(a, ft, *a.contrib, grid);
        else launch_render_f<Stats::WEIGHTS>(a, ft, *a.contrib, grid);
        sr_count_launch();
        return cudaGetLastError();
    }
    ProfileScope ps("composite_fwd", a.stream);
    composite_fwd_kernel<true, 1, 0><<<((a.il.tiles * 8 + WPC - 1) / WPC) * a.fs.frames, 32 * WPC, 0, a.stream>>>(
        a.fs, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles * 8, a.il.tiles_x,
        (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
        (float*)(a.img + a.il.final_T), (uint32_t*)(a.img + a.il.n_contrib), a.out_color, a.out_others,
        (uint32_t*)(a.img + a.il.tile_last), (uint32_t*)(a.bin + a.bl.contrib), FeatArgs{}, ContribArgs{});
    sr_count_launch();
    return cudaGetLastError();
}
