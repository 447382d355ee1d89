// composite_fwd.cu -- per-tile front-to-back alpha composite of colour / depth / normal / distortion.
//
// Replaces (behaviour, not code) of the reference's forward renderCUDA, RAST/cuda_rasterizer/forward.cu:265-463.
//
// Design (DESIGN.md "composite"):
//   * work item = (tile, 8x4 sub-tile) = one warp = one CTA, launched longest-tile-first; each warp streams the
//     tile's sorted instance records (80 B each, contiguous) through its own double-buffered shared-memory ring
//     with cp.async.bulk (TMA 1-D) on its own mbarriers -- no CTA-wide synchronisation;
//   * one pixel per lane.  Per 32-record stage, lane = instance turns the instance's conservative cull rectangle into
//     column and row masks of the sub-tile (group_survivors); then each lane walks its own survivor list, so up to 32
//     different instances are evaluated per warp iteration.  With ~5x5-pixel footprints a whole-warp 8x4 block
//     wastes most lanes;
//   * per stage and pixel the kernel records which instances contributed (one 128-B store per warp): the backward
//     walks exactly those;
//   * culling and the rho_cut early-out never change a result: a skipped pair provably has alpha < 1/255;
//   * per-pair arithmetic uses explicit-rounding intrinsics in the contraction pattern of the reference's
//     sm_100a SASS, so colour/depth/alpha/normal/median planes are bit-identical to the reference build.
#include "composite_common.cuh"

namespace {
using namespace comp;

constexpr int WPC = 1;      // independent warps per CTA (2 measured slower: register pressure)

__global__ void __launch_bounds__(32 * WPC)
composite_fwd_kernel(const FrameStrides fs, const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, int n_items, int tiles_x,
                     const float4* __restrict__ irec, int W, int H,
                     const float* __restrict__ bg, float* __restrict__ final_T, uint32_t* __restrict__ n_contrib,
                     float* __restrict__ out_color, float* __restrict__ out_others, uint32_t* __restrict__ sub_last,
                     uint32_t* __restrict__ contrib_masks) {
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

    // warp -> 8x4 sub-tile, lane -> pixel (slot lane = ly * 8 + lx of the contribution-mask layout)
    const int sx0 = (warp & 1) * 8, sy0 = (warp >> 1) * 4;
    const int bx0 = sx0 + lane % 8, by0 = sy0 + lane / 8;      // tile-local pixel
    const int pix_x = tile_x * SR_TILE + bx0, pix_y = tile_y * SR_TILE + by0;
    const bool inside = pix_x < W && pix_y < H;
    const float pixx = (float)pix_x + 0.5f, pixy = (float)pix_y + 0.5f;

    const float4* src = irec + (size_t)range.x * REC4;
    auto issue = [&](int b) {   // lane 0 only
        const int s = b % NST;
        const uint32_t bytes = (uint32_t)min(WB, len - b * WB) * 80u;
        mbar_expect_tx(&bar[s], bytes);
        bulk_g2s(st[s], src + (size_t)b * WB * REC4, bytes, &bar[s]);
    };
    if (lane == 0) {
#pragma unroll
        for (int s = 0; s < NST; s++) mbar_init(&bar[s], 1);
        fence_mbar_init();
        for (int b = 0; b < NST && b < nb; b++) issue(b);
    }
    __syncwarp();

    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
    float dist1 = 0.f, dist2 = 0.f, distortion = 0.f, median_depth = 0.f, median_weight = 0.f;
    uint32_t median_contributor = 0, last_contributor = 0;
    bool done = !inside;
    // instances of the current stage that contributed to this lane's pixel, kept for the backward (common.cuh
    // bin_layout: contrib); slot = pixel index inside the 8x4 sub-tile, so a warp's 32 words are one 128-B store
    uint32_t cmask = 0u;
    uint32_t* cm_out = contrib_masks + (((size_t)(range.x >> 5) + tile) * 8 + warp) * 32 + ((by0 - sy0) * 8 + (bx0 - sx0));

    for (int b = 0; b < nb; b++) {
        const int s = b % NST;
        mbar_wait(&bar[s], (uint32_t)((b / NST) & 1));
        const int cnt = min(WB, len - b * WB);
        const float4* S = st[s];
        uint32_t cull = 0;
        if (lane < cnt) cull = __float_as_uint(S[lane * REC4 + 4].w);
        // lane = instance: which pixels does this instance's cull rectangle touch?
        uint32_t mym = group_survivors(cull, sx0, sy0, lane);
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
            const float4 r0 = S[jj * REC4], r1 = S[jj * REC4 + 1], r2 = S[jj * REC4 + 2];
            // T rows: Tu=(r0.x,r0.y,r0.z) Tv=(r0.w,r1.x,r1.y) Tw=(r1.z,r1.w,r2.x); xy=(r2.y,r2.z); opac=r2.w
            const float kx = ff(pixx, r1.z, -r0.x), ky = ff(pixx, r1.w, -r0.y), kz = ff(pixx, r2.x, -r0.z);
            const float lx_ = ff(pixy, r1.z, -r0.w), ly_ = ff(pixy, r1.w, -r1.x), lz_ = ff(pixy, r2.x, -r1.y);
            const float pz = ff(kx, ly_, -fm(ky, lx_));
            if (pz == 0.0f) continue;
            const float ppx = ff(ky, lz_, -fm(kz, ly_));
            const float ppy = ff(kz, lx_, -fm(kx, lz_));
            float sx, sy;
            div2_rn(ppx, ppy, pz, sx, sy);
            const float rho3d = ff(sx, sx, fm(sy, sy));
            const float dx = fa(r2.y, -pixx), dy = fa(r2.z, -pixy);
            const float q2 = ff(dx, dx, fm(dy, dy));
            const float rho2d = fa(q2, q2);
            const float rho = fminf(rho3d, rho2d);
            if (rho > rho_cut) continue;                 // alpha < 1/255 guaranteed: same outcome as below, no expf
            const float depth = (rho3d <= rho2d) ? fa(r2.x, ff(r1.z, sx, fm(r1.w, sy))) : r2.x;
            if (depth < 0.2f) continue;
            const float power = fm(rho, -0.5f);
            if (power > 0.0f) continue;
            const float alpha = fminf(0.99f, fm(r2.w, expf(power)));
            if (alpha < 1.0f / 255.0f) continue;
            const float test_T = fm(T, fa(1.0f, -alpha));
            if (test_T < 0.0001f) { done = true; continue; }
            const float4 r3 = S[jj * REC4 + 3], r4 = S[jj * REC4 + 4];
            const uint32_t contributor = (uint32_t)(b * WB + jj + 1);
            const float A = fa(1.0f, -T);
            const float mdep = map_depth(depth);
            const float mm = fm(mdep, mdep);
            const float error = ff(-dist1, fa(mdep, mdep), ff(A, mm, dist2));
            distortion = ff(T, fm(alpha, error), distortion);
            if (T > 0.5f) { median_depth = depth; median_weight = fm(T, alpha); median_contributor = contributor; }
            N0 = ff(T, fm(r3.x, alpha), N0);
            N1 = ff(T, fm(r3.y, alpha), N1);
            N2 = ff(T, fm(r3.z, alpha), N2);
            D = ff(T, fm(depth, alpha), D);
            dist1 = ff(T, fm(alpha, mdep), dist1);
            dist2 = ff(T, fm(alpha, mm), dist2);
            C0 = ff(T, fm(alpha, r3.w), C0);
            C1 = ff(T, fm(alpha, r4.x), C1);
            C2 = ff(T, fm(alpha, r4.y), C2);
            T = test_T;
            last_contributor = contributor;
            cmask |= 1u << jj;
        }
        __syncwarp();                                   // every lane is done reading stage s
        cm_out[(size_t)b * SR_CONTRIB_STAGE_WORDS] = cmask;
        cmask = 0u;
        if (__all_sync(0xffffffffu, done)) {
            // drain the copies still in flight before this warp (and its CTA's smem) goes away
            for (int b2 = b + 1; b2 < nb && b2 < b + NST; b2++) mbar_wait(&bar[b2 % NST], (uint32_t)((b2 / NST) & 1));
            break;
        }
        if (lane == 0 && b + NST < nb) issue(b + NST);
    }

    // deepest list position any pixel of this sub-tile used: the backward starts its reverse walk there
    uint32_t wmax = last_contributor;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) wmax = max(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
    if (lane == 0) sub_last[tile * 8 + warp] = wmax;

    if (inside) {
        const size_t N = (size_t)W * H, pid = (size_t)W * pix_y + pix_x;
        final_T[pid] = T;
        final_T[pid + N] = dist1;
        final_T[pid + 2 * N] = dist2;
        n_contrib[pid] = last_contributor;
        n_contrib[pid + N] = median_contributor;
        out_color[pid] = ff(T, __ldg(bg), C0);
        out_color[pid + N] = ff(T, __ldg(bg + 1), C1);
        out_color[pid + 2 * N] = ff(T, __ldg(bg + 2), C2);
        out_others[pid] = D;
        out_others[pid + N] = fa(1.0f, -T);
        out_others[pid + 2 * N] = N0;
        out_others[pid + 3 * N] = N1;
        out_others[pid + 4 * N] = N2;
        out_others[pid + 5 * N] = median_depth;
        out_others[pid + 6 * N] = distortion;
        out_others[pid + 7 * N] = median_weight;
    }
}

}  // namespace

cudaError_t launch_composite_fwd(const FwdArgs& a) {
    ProfileScope ps("composite_fwd", a.stream);
    composite_fwd_kernel<<<((a.il.tiles * 8 + WPC - 1) / WPC) * a.fs.frames, 32 * WPC, 0, a.stream>>>(
        a.fs, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles * 8, a.il.tiles_x,
        (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
        (float*)(a.img + a.il.final_T), (uint32_t*)(a.img + a.il.n_contrib), a.out_color, a.out_others,
        (uint32_t*)(a.img + a.il.tile_last), (uint32_t*)(a.bin + a.bl.contrib));
    sr_count_launch();
    return cudaGetLastError();
}
