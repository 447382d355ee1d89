// composite_tile.cu -- forward and backward composite with one CTA per 16x16 tile and a shared TMA chunk ring.
//
// Replaces (behaviour, not code) of the reference's renderCUDA forward / backward,
// RAST/cuda_rasterizer/forward.cu:265-463 and backward.cu:143-449.  Same per-pair arithmetic, contribution
// masks, accumulator layout and outputs as composite_fwd.cu / composite_bwd.cu (the one-warp-per-CTA kernels);
// what changes is how the instance list reaches the lanes:
//
//   * CTA = one tile = 8 warps (one per 8x4 sub-tile, lane = pixel).  The tile's sorted 80-byte instance records
//     stream through ONE ring of NSLOT chunks of CH instances, filled by cp.async.bulk (TMA 1-D) and shared by the 8
//     warps -- 8x less shared memory per warp than a private ring, which is what makes CH = 256 affordable.
//   * Inside a chunk every LANE walks its own list (cull masks forward, recorded contribution masks backward) without
//     any stage lock-step: the warp only re-converges at chunk boundaries.  With ~2 contributions per pixel and
//     32-instance stage, lock-step at stage granularity evaluates 12.5 pairs per 32-lane iteration on the headline
//     frame (Poisson noise: the warp waits for its busiest lane every stage); at 256 instances it is 18
//     (replay of the recorded masks).
//   * No CTA-wide barrier after start-up.  A ring slot is released by an shared-memory counter; the warp whose
//     release is the eighth issues the next bulk copy into it, so there is no producer warp to wait on.  A warp may
//     run NSLOT-1 chunks ahead of the slowest warp of its tile.
//   * Forward early termination is per lane (T < 1e-4), per warp (all 32 pixels done: the warp only waits for and
//     releases the remaining chunks) and per CTA (all 8 warps done: no further chunk is requested).
#include "composite_common.cuh"

namespace {
using namespace comp;

constexpr int TWARPS = 8;      // 8x4 sub-tiles of a 16x16 tile

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n"     // suspend-time hint: the warp sleeps in hardware
        "selp.u32 %0, 1, 0, p;\n"                                          // instead of spinning (r2a ncu: 8 % of the
        "}\n" : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity), "r"(20000u) : "memory");   // forward's issue slots were the spin loop)
    return ok != 0;
}

template <int CH, int NSLOT>
struct TileSmem {
    static constexpr int NSTG = CH / 32;                                         // 32-instance stages per chunk
    static constexpr size_t ring = (size_t)NSLOT * CH * REC4 * sizeof(float4);
    static constexpr size_t masks = (size_t)TWARPS * NSTG * 32 * sizeof(uint32_t);
    static constexpr size_t total = ring + masks + NSLOT * sizeof(uint64_t) + (NSLOT + 4) * sizeof(uint32_t);
};

// ------------------------------------------------------------------------------------------------ forward
template <int CH, int NSLOT, int MINB>
__global__ void __launch_bounds__(32 * TWARPS, MINB)
composite_tile_fwd_kernel(const FrameStrides fs, const uint2* __restrict__ ranges, const uint32_t* __restrict__ tile_order, int tiles_x,
                          const float4* __restrict__ irec, int W, int H, const float* __restrict__ bg,
                          float* __restrict__ final_T, uint32_t* __restrict__ n_contrib, float* __restrict__ out_color,
                          float* __restrict__ out_others, uint32_t* __restrict__ sub_last,
                          uint32_t* __restrict__ contrib_masks) {
    using SM = TileSmem<CH, NSLOT>;
    constexpr int NSTG = SM::NSTG;
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

    // warp -> 8x4 sub-tile, lane -> pixel (slot lane = ly * 8 + lx of the contribution-mask layout)
    const int sx0 = (warp & 1) * 8, sy0 = (warp >> 1) * 4;
    const int pix_x = tile_x * SR_TILE + sx0 + (lane & 7), pix_y = tile_y * SR_TILE + sy0 + (lane >> 3);
    const bool inside = pix_x < W && pix_y < H;
    const float pixx = (float)pix_x + 0.5f, pixy = (float)pix_y + 0.5f;

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

    float T = 1.0f, C0 = 0.f, C1 = 0.f, C2 = 0.f, D = 0.f, N0 = 0.f, N1 = 0.f, N2 = 0.f;
    float dist1 = 0.f, dist2 = 0.f, distortion = 0.f, median_depth = 0.f, median_weight = 0.f;
    uint32_t median_contributor = 0, last_contributor = 0;
    bool done = !inside;
    bool counted = false;                          // (warp-uniform) this warp is in ctl[0]
    uint32_t* cm = cm_all + warp * NSTG * 32 + lane;          // this lane's column: cm[st * 32]
    uint32_t* cm_out = contrib_masks + (((size_t)(range.x >> 5) + tile) * 8 + warp) * 32 + lane;

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
                    const uint32_t m = group_survivors<32>(cull, sx0, sy0, lane);
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
                const float4 r0 = R[0], r1 = R[1], r2 = R[2], r4 = R[4];
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
                if (rho > cull_rho_cut(__float_as_uint(r4.w))) continue;   // alpha < 1/255 guaranteed: no expf
                const float depth = (rho3d <= rho2d) ? fa(r2.x, ff(r1.z, sx, fm(r1.w, sy))) : r2.x;
                if (depth < 0.2f) continue;
                const float power = fm(rho, -0.5f);
                if (power > 0.0f) continue;
                const float alpha = fminf(0.99f, fm(r2.w, expf(power)));
                if (alpha < 1.0f / 255.0f) continue;
                const float test_T = fm(T, fa(1.0f, -alpha));
                if (test_T < 0.0001f) { done = true; mym = 0u; nz = 0u; continue; }
                const float4 r3 = R[3];
                const uint32_t contributor = (uint32_t)(c * CH + st * 32 + jj + 1);
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

// ------------------------------------------------------------------------------------------------ backward
template <int CH, int NSLOT, int MINB>
__global__ void __launch_bounds__(32 * TWARPS, MINB)
composite_tile_bwd_kernel(const FrameStrides fs, const float* __restrict__ grad_scale, const uint2* __restrict__ ranges,
                          const uint32_t* __restrict__ tile_order, int tiles_x,
                          const float4* __restrict__ irec, int W, int H, const float* __restrict__ bg,
                          const float* __restrict__ final_Ts, const uint32_t* __restrict__ n_contrib,
                          const uint32_t* __restrict__ sub_last, const float* __restrict__ dL_dpixels,
                          const float* __restrict__ dL_dothers, const uint32_t* __restrict__ contrib_masks,
                          float* __restrict__ sgrad) {
    using SM = TileSmem<CH, NSLOT>;
    constexpr int NSTG = SM::NSTG;
    extern __shared__ __align__(128) unsigned char smem_raw[];
    float4* ring = reinterpret_cast<float4*>(smem_raw);
    uint32_t* cm_all = reinterpret_cast<uint32_t*>(smem_raw + SM::ring);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw + SM::ring + SM::masks);
    uint32_t* rel = reinterpret_cast<uint32_t*>(full + NSLOT);

    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int f = (int)(blockIdx.x % (unsigned)fs.frames);
    ranges = fr(ranges, fs.img, f); tile_order = fr(tile_order, fs.img, f); irec = fr(irec, fs.bin, f);
    final_Ts = fr(final_Ts, fs.img, f); n_contrib = fr(n_contrib, fs.img, f); sub_last = fr(sub_last, fs.img, f);
    dL_dpixels = fr(dL_dpixels, fs.dcolor, f); dL_dothers = fr(dL_dothers, fs.dothers, f);
    contrib_masks = fr(contrib_masks, fs.bin, f); sgrad = fr(sgrad, fs.geom, f);
    const int tile = (int)tile_order[blockIdx.x / (unsigned)fs.frames];
    const int tile_x = tile % tiles_x, tile_y = tile / tiles_x;
    const uint2 range = ranges[tile];
    const int rlen = (int)(range.y - range.x);
    // nothing beyond a sub-tile's deepest contributor matters to it; the CTA streams up to the deepest of the eight
    const uint32_t my_last = sub_last[tile * 8 + (lane & 7)];
    uint32_t cta_last = my_last;
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) cta_last = max(cta_last, __shfl_xor_sync(0xffffffffu, cta_last, o));
    const int len = min(rlen, (int)cta_last);
    const int len_w = min(rlen, (int)__shfl_sync(0xffffffffu, my_last, warp));
    const int nchunks = (len + CH - 1) / CH;
    if (nchunks == 0) return;
    const int nb_w = (len_w + 31) >> 5;            // stages this sub-tile reads

    const int sx0 = (warp & 1) * 8, sy0 = (warp >> 1) * 4;
    const float4* src = irec + (size_t)range.x * REC4;
    // the k-th consumed chunk (k = 0, 1, ..) is c = nchunks-1-k; it lives in slot k % NSLOT
    auto issue = [&](int k) {   // one thread
        const int c = nchunks - 1 - k, s = k % NSLOT;
        const uint32_t bytes = (uint32_t)min(CH, len - c * CH) * 80u;
        fence_proxy_async();
        mbar_expect_tx(&full[s], bytes);
        bulk_g2s(ring + (size_t)s * CH * REC4, src + (size_t)c * CH * REC4, bytes, &full[s]);
    };
    if (threadIdx.x == 0) {
#pragma unroll
        for (int s = 0; s < NSLOT; s++) { mbar_init(&full[s], 1); rel[s] = 0u; }
        fence_mbar_init();
        for (int k = 0; k < NSLOT && k < nchunks; k++) issue(k);
    }
    __syncthreads();                               // the only CTA-wide barrier

    BwdPixel px;
    px.load(tile_x * SR_TILE + sx0 + (lane & 7), tile_y * SR_TILE + sy0 + (lane >> 3), W, H, bg, final_Ts, n_contrib,
            dL_dpixels, dL_dothers, grad_scale);

    uint32_t* cm = cm_all + warp * NSTG * 32 + lane;
    const uint32_t* cm_in = contrib_masks + (((size_t)(range.x >> 5) + tile) * 8 + warp) * 32 + lane;
    uint32_t pre[NSTG];                            // the next chunk's masks, in flight while this one is walked
    auto fetch = [&](int c) {
#pragma unroll
        for (int st = 0; st < NSTG; st++) {
            const int g = c * NSTG + st;
            pre[st] = g < nb_w ? __ldg(cm_in + (size_t)g * SR_CONTRIB_STAGE_WORDS) : 0u;
        }
    };
    fetch(nchunks - 1);

    for (int k = 0; k < nchunks; k++) {
        const int c = nchunks - 1 - k, s = k % NSLOT;
        uint32_t nz = 0u;
#pragma unroll
        for (int st = 0; st < NSTG; st++) { cm[st * 32] = pre[st]; if (pre[st]) nz |= 1u << st; }
        if (c > 0) fetch(c - 1);
        const bool any = __any_sync(0xffffffffu, nz != 0u);
        {
            const uint32_t parity = (uint32_t)((k / NSLOT) & 1);
            while (!mbar_try_wait(&full[s], parity)) { }
        }
        if (any) {
            const float4* S = ring + (size_t)s * CH * REC4;
            int st = 0;
            uint32_t mym = 0u;
            for (;;) {
                if (mym == 0u && nz) { st = 31 - __clz(nz); nz &= ~(1u << st); mym = cm[st * 32]; }
                const bool act = mym != 0u;
                if (!__any_sync(0xffffffffu, act)) break;
                if (!act) continue;
                const int jj = 31 - __clz(mym);
                mym &= ~(1u << jj);
                const int idx = st * 32 + jj;
                float v[16];
#pragma unroll
                for (int i = 0; i < 16; i++) v[i] = 0.f;
                float m2x = 0.f, m2y = 0.f;
                bool lowpass = false;
                px.pair(S + idx * REC4, c * CH + idx, v, m2x, m2y, lowpass);
                red_pixel(sgrad, S + idx * REC4, v, m2x, m2y, lowpass);
            }
        }
        __syncwarp();
        if (lane == 0) {
            __threadfence_block();
            if (atomicAdd(&rel[s], 1u) == TWARPS - 1) {
                rel[s] = 0u;
                __threadfence_block();
                if (k + NSLOT < nchunks) issue(k + NSLOT);
            }
        }
    }
}

template <typename K>
cudaError_t opt_in_smem(K kern, size_t bytes) {
    // per device: cudaFuncSetAttribute applies to the current device's context only
    static bool set[64] = {};
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64 || !set[dev]) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
        if (e != cudaSuccess) return e;
        if (dev >= 0 && dev < 64) set[dev] = true;
    }
    return cudaSuccess;
}

}  // namespace

// Which composite kernels run: SURFEL_COMPOSITE=tile|warp sets both directions, SURFEL_COMPOSITE_FWD / _BWD one of them.
// Defaults (measured on the headline batch): forward = one-warp CTAs with private rings (fewer
// instructions per iteration; the forward is issue bound), backward = tile CTAs with the shared chunk ring (25 % fewer
// instructions thanks to the per-lane free walk; the backward is bound by L2 reductions and latency).
bool sr_composite_tile_mode(bool backward) {
    static const int mode = [] {
        auto pick = [](const char* name, int dflt) {
            const char* e = getenv(name);
            if (!e) e = getenv("SURFEL_COMPOSITE");
            return e ? (e[0] == 't' ? 1 : 0) : dflt;
        };
        return pick("SURFEL_COMPOSITE_FWD", 0) | (pick("SURFEL_COMPOSITE_BWD", 1) << 1);
    }();
    return backward ? (mode >> 1) & 1 : mode & 1;
}

int comp::tile_cfg_from_env() {
    static const int cfg = [] {
        const char* e = getenv("SURFEL_TILE_CFG");
        const int v = e ? atoi(e) : 2562;
        return (v == 2562 || v == 2563 || v == 1283 || v == 1284 || v == 5122 || v == 1282) ? v : 2562;
    }();
    return cfg;
}

cudaError_t launch_composite_tile_fwd(const FwdArgs& a) {
    ProfileScope ps("composite_fwd", a.stream);
    cudaError_t err = cudaSuccess;
    auto launch = [&](auto kern, size_t smem) {
        err = opt_in_smem(kern, smem);
        if (err != cudaSuccess) return;
        kern<<<a.il.tiles * a.fs.frames, 32 * TWARPS, smem, a.stream>>>(
            a.fs, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles_x,
            (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
            (float*)(a.img + a.il.final_T), (uint32_t*)(a.img + a.il.n_contrib), a.out_color, a.out_others,
            (uint32_t*)(a.img + a.il.tile_last), (uint32_t*)(a.bin + a.bl.contrib));
    };
    switch (comp::tile_cfg_from_env()) {
        case 2563: launch(composite_tile_fwd_kernel<256, 3, 3>, TileSmem<256, 3>::total); break;
        case 1282: launch(composite_tile_fwd_kernel<128, 2, 4>, TileSmem<128, 2>::total); break;
        case 1283: launch(composite_tile_fwd_kernel<128, 3, 4>, TileSmem<128, 3>::total); break;
        case 1284: launch(composite_tile_fwd_kernel<128, 4, 4>, TileSmem<128, 4>::total); break;
        case 5122: launch(composite_tile_fwd_kernel<512, 2, 2>, TileSmem<512, 2>::total); break;
        default: launch(composite_tile_fwd_kernel<256, 2, 4>, TileSmem<256, 2>::total); break;
    }
    if (err != cudaSuccess) return err;
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_composite_tile_bwd(const BwdArgs& a) {
    cudaError_t e = sr_memset_frames(a.geom + a.gl.sgrad, (size_t)a.fs.geom, (size_t)(a.cam.P > 0 ? a.cam.P : 1) * SR_GRAD_FLOATS * 4,
                                     a.fs.frames, a.stream);
    if (e != cudaSuccess) return e;
    ProfileScope ps("composite_bwd", a.stream);
    cudaError_t err = cudaSuccess;
    auto launch = [&](auto kern, size_t smem) {
        err = opt_in_smem(kern, smem);
        if (err != cudaSuccess) return;
        kern<<<a.il.tiles * a.fs.frames, 32 * TWARPS, smem, a.stream>>>(
            a.fs, a.grad_scale, (const uint2*)(a.img + a.il.ranges), (const uint32_t*)(a.img + a.il.tile_order), a.il.tiles_x,
            (const float4*)(a.bin + a.bl.inst_rec), a.cam.W, a.cam.H, a.cam.bg,
            (const float*)(a.img + a.il.final_T), (const uint32_t*)(a.img + a.il.n_contrib),
            (const uint32_t*)(a.img + a.il.tile_last), a.dL_dcolor, a.dL_dothers,
            (const uint32_t*)(a.bin + a.bl.contrib), (float*)(a.geom + a.gl.sgrad));
    };
    switch (comp::tile_cfg_from_env()) {
        case 2563: launch(composite_tile_bwd_kernel<256, 3, 3>, TileSmem<256, 3>::total); break;
        case 1282: launch(composite_tile_bwd_kernel<128, 2, 3>, TileSmem<128, 2>::total); break;
        case 1283: launch(composite_tile_bwd_kernel<128, 3, 3>, TileSmem<128, 3>::total); break;
        case 1284: launch(composite_tile_bwd_kernel<128, 4, 3>, TileSmem<128, 4>::total); break;
        case 5122: launch(composite_tile_bwd_kernel<512, 2, 2>, TileSmem<512, 2>::total); break;
        default: launch(composite_tile_bwd_kernel<256, 2, 3>, TileSmem<256, 2>::total); break;
    }
    if (err != cudaSuccess) return err;
    sr_count_launch();
    return cudaGetLastError();
}
