// sort.cu -- stable onesweep LSD radix sort of the (tile | depth) instance keys, then tile ranges and
// the per-instance record stream.
//
// Replaces (behaviour, not code) of the reference:
//   cub::DeviceRadixSort::SortPairs(keys u64, values u32, bits [0, 32+bit))   rasterizer_impl.cu:301-309
//   cudaMemset(ranges) + identifyTileRanges                                   rasterizer_impl.cu:311-319, 116-138
//   the per-round gather of surfel attributes inside renderCUDA                forward.cu:338-349, backward.cu:256-270
//
// Design (DESIGN.md "sort"):
//   * one histogram kernel reads the keys once and builds the digit histograms of ALL passes;
//   * a plan kernel exclusive-scans them, and marks a pass as skipped when one bin holds every key
//     (e.g. the top depth byte of an object-centric scene) -- the permutation of that pass is the
//     identity, so skipping it cannot change the result;
//   * each remaining pass is ONE kernel: tiles are claimed in order through an atomic ticket, ranked
//     stably with warp match-any, chained with decoupled look-back on a (flag|count) word per bin, and
//     scattered through shared memory so the global stores are contiguous per bin.
//   The instance count R lives only on the device (no D2H sync in the forward): grids are sized from the
//   buffer CAPACITY and surplus blocks exit on the first load of R.
#include <cstdlib>
#include "composite_common.cuh"

namespace {
__device__ __forceinline__ uint32_t comp_cull_rho(float opacity) { return comp::cull_encode_rho_cut(opacity); }

enum : uint32_t { FLAG_AGG = 1u << 30, FLAG_INC = 2u << 30, FLAG_MASK = 3u << 30, VAL_MASK = ~(3u << 30) };

struct SortPlan {
    int npass;
    int shift[SR_SORT_MAX_PASSES];
    int bits[SR_SORT_MAX_PASSES];
};

__global__ void __launch_bounds__(256)
sort_histogram_kernel(const FrameStrides fs, const uint64_t* __restrict__ keys, const uint32_t* __restrict__ num_rendered,
                      long long capacity, SortPlan plan, uint32_t* __restrict__ hist) {
    const int f = blockIdx.y;
    keys = fr(keys, fs.bin, f); num_rendered = fr(num_rendered, fs.nr, f); hist = fr(hist, fs.bin, f);
    const uint32_t n = num_rendered[0];
    if ((long long)n > capacity) return;
    __shared__ uint32_t sh[SR_SORT_MAX_PASSES * SR_SORT_BINS];
    for (int i = threadIdx.x; i < plan.npass * SR_SORT_BINS; i += 256) sh[i] = 0;
    __syncthreads();
    const uint32_t per_block = 256 * 16;
    const uint32_t base = blockIdx.x * per_block;
    if (base >= n) return;
#pragma unroll 4
    for (int j = 0; j < 16; j++) {
        const uint32_t i = base + j * 256 + threadIdx.x;
        if (i < n) {
            const uint64_t k = keys[i];
            for (int p = 0; p < plan.npass; p++)
                atomicAdd(&sh[p * SR_SORT_BINS + (uint32_t)((k >> plan.shift[p]) & ((1u << plan.bits[p]) - 1u))], 1u);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < plan.npass * SR_SORT_BINS; i += 256)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// one block: exclusive-scan each pass's histogram in place, decide which passes are identities
__global__ void __launch_bounds__(256)
sort_plan_kernel(const FrameStrides fs, uint32_t* __restrict__ hist, uint32_t* __restrict__ ctl,
                 const uint32_t* __restrict__ num_rendered, long long capacity, SortPlan plan) {
    const int f = blockIdx.x;                       // one block per frame
    hist = fr(hist, fs.bin, f); ctl = fr(ctl, fs.bin, f); num_rendered = fr(num_rendered, fs.nr, f);
    const uint32_t n = num_rendered[0];
    __shared__ uint32_t wsum[8];
    __shared__ int skip_s[SR_SORT_MAX_PASSES];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x < SR_SORT_MAX_PASSES) skip_s[threadIdx.x] = 0;
    __syncthreads();
    const bool dead = (long long)n > capacity || n == 0;
    for (int p = 0; p < plan.npass; p++) {
        const uint32_t v = hist[p * SR_SORT_BINS + threadIdx.x];
        if (v == n || dead) skip_s[p] = 1;      // benign race: every writer writes 1
        uint32_t inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) wsum[warp] = inc;
        __syncthreads();
        uint32_t wb = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) wb += i < warp ? wsum[i] : 0u;
        hist[p * SR_SORT_BINS + threadIdx.x] = wb + inc - v;
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        uint32_t sel = 0;
        for (int p = 0; p < plan.npass; p++) {
            ctl[SR_CTL_SRC + p] = sel;
            ctl[SR_CTL_SKIP + p] = (uint32_t)skip_s[p];
            if (!skip_s[p]) sel ^= 1u;
        }
        ctl[SR_CTL_SORTED_SEL] = sel;
        ctl[SR_CTL_NPASS] = (uint32_t)plan.npass;
    }
}

// 3 resident blocks per SM (<= 85 registers, no spills) instead of 2: the pass is latency bound (ticket, key loads,
// look-back), r2g ncu: 24 % warps active, 15 % DRAM.
__global__ void __launch_bounds__(SR_SORT_THREADS, 3)
onesweep_pass_kernel(const FrameStrides fs, uint64_t* __restrict__ keys0, uint64_t* __restrict__ keys1,
                     uint32_t* __restrict__ vals0, uint32_t* __restrict__ vals1, const uint32_t* __restrict__ hist,
                     uint32_t* __restrict__ ctl, uint32_t* __restrict__ status, const uint32_t* __restrict__ num_rendered,
                     int pass, int shift, int bits, int sort_tiles, int interleave) {
    // Block -> (frame, slot).  Interleaved: consecutive blocks belong to different frames, so the ~300 blocks resident at
    // a time hold only ~300 / frames consecutive tiles of any one frame and the look-back chain inside a wave is that
    // short (all tiles of a 0.5 M-key frame would otherwise start together and tile t would walk back over t tiles).
    const int f = interleave ? (int)(blockIdx.x % (unsigned)fs.frames) : (int)(blockIdx.x / (unsigned)sort_tiles);
    const uint32_t slot = interleave ? blockIdx.x / (unsigned)fs.frames : blockIdx.x % (unsigned)sort_tiles;
    keys0 = fr(keys0, fs.bin, f); keys1 = fr(keys1, fs.bin, f); vals0 = fr(vals0, fs.bin, f); vals1 = fr(vals1, fs.bin, f);
    hist = fr(hist, fs.bin, f); ctl = fr(ctl, fs.bin, f); status = fr(status, fs.bin, f); num_rendered = fr(num_rendered, fs.nr, f);
    const uint32_t skip = ctl[SR_CTL_SKIP + pass];
    const uint32_t n = num_rendered[0];
    // the grid is sized from the buffer capacity: blocks beyond the tiles this frame needs leave before taking a ticket
    // (exactly ceil(n / TILE) blocks stay, so every ticket below that is handed out)
    if (skip || (unsigned long long)slot * SR_SORT_TILE >= n) return;
    __shared__ uint64_t keys_s[SR_SORT_TILE];
    __shared__ uint32_t vals_s[SR_SORT_TILE];
    __shared__ uint32_t whist[8][SR_SORT_BINS];
    __shared__ uint32_t lstart[SR_SORT_BINS];
    __shared__ uint32_t goff[SR_SORT_BINS];
    __shared__ uint32_t wsum[8];
    __shared__ uint32_t tile_s;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    if (tid == 0) tile_s = atomicAdd(&ctl[SR_CTL_TILE_COUNTER + pass], 1u);
#pragma unroll
    for (int w = 0; w < 8; w++) whist[w][tid] = 0;
    __syncthreads();
    const uint32_t tile = tile_s;
    const uint32_t tile_base = tile * SR_SORT_TILE;
    if (tile_base >= n) return;
    const uint32_t src = ctl[SR_CTL_SRC + pass];
    const uint64_t* __restrict__ kin = src ? keys1 : keys0;
    const uint32_t* __restrict__ vin = src ? vals1 : vals0;
    uint64_t* __restrict__ kout = src ? keys0 : keys1;
    uint32_t* __restrict__ vout = src ? vals0 : vals1;
    const uint32_t mask = (1u << bits) - 1u;
    const uint32_t lt_mask = (1u << lane) - 1u;

    uint64_t key[SR_SORT_ITEMS];
    uint32_t val[SR_SORT_ITEMS];
    uint32_t rank[SR_SORT_ITEMS];
    const uint32_t wbase = tile_base + warp * (32 * SR_SORT_ITEMS);
#pragma unroll
    for (int i = 0; i < SR_SORT_ITEMS; i++) {
        const uint32_t idx = wbase + i * 32 + lane;
        const bool valid = idx < n;
        key[i] = valid ? kin[idx] : ~0ull;
        val[i] = valid ? vin[idx] : 0u;
    }
    // stable ranking: items of a warp are visited in index order, lanes in lane order
#pragma unroll
    for (int i = 0; i < SR_SORT_ITEMS; i++) {
        const uint32_t idx = wbase + i * 32 + lane;
        const bool valid = idx < n;
        const uint32_t d = valid ? (uint32_t)((key[i] >> shift) & mask) : 0xffffffffu;
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const int leader = __ffs(peers) - 1;
        uint32_t old = 0;
        if (lane == leader && valid) { old = whist[warp][d]; whist[warp][d] = old + __popc(peers); }
        old = __shfl_sync(0xffffffffu, old, leader);
        rank[i] = old + __popc(peers & lt_mask);
        __syncwarp();
    }
    __syncthreads();
    // per-bin: exclusive offsets across warps, tile count
    uint32_t count = 0;
#pragma unroll
    for (int w = 0; w < 8; w++) { const uint32_t c = whist[w][tid]; whist[w][tid] = count; count += c; }
    // decoupled look-back, one thread per bin
    uint32_t* st = status + ((size_t)pass * sort_tiles) * SR_SORT_BINS;
    uint32_t excl = 0;
    if (tile == 0) {
        atomicExch(&st[(size_t)tile * SR_SORT_BINS + tid], FLAG_INC | count);
    } else {
        atomicExch(&st[(size_t)tile * SR_SORT_BINS + tid], FLAG_AGG | count);
        // windowed look-back: LB independent loads in flight per hop instead of one dependent load per
        // predecessor (all tiles of a 0.5 M-key sort run in one wave, so nobody is "long finished")
        constexpr int LB = 16;
        int t = (int)tile - 1;
        while (true) {
            uint32_t v[LB];
#pragma unroll
            for (int q = 0; q < LB; q++)
                v[q] = (t - q >= 0) ? *((volatile uint32_t*)&st[(size_t)(t - q) * SR_SORT_BINS + tid]) : FLAG_INC;
            bool fin = false;
            int q = 0;
#pragma unroll
            for (; q < LB; q++) {
                const uint32_t f = v[q] & FLAG_MASK;
                if (f == 0) break;                  // not published yet: re-read from here
                excl += v[q] & VAL_MASK;
                if (f == FLAG_INC) { fin = true; break; }
            }
            if (fin) break;
            t -= q;
        }
        atomicExch(&st[(size_t)tile * SR_SORT_BINS + tid], FLAG_INC | (excl + count));
    }
    // tile-local exclusive scan over bins
    uint32_t inc = count;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { uint32_t t2 = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t2; }
    if (lane == 31) wsum[warp] = inc;
    __syncthreads();
    uint32_t wb = 0;
#pragma unroll
    for (int i = 0; i < 8; i++) wb += i < warp ? wsum[i] : 0u;
    const uint32_t ls = wb + inc - count;
    lstart[tid] = ls;
    goff[tid] = hist[pass * SR_SORT_BINS + tid] + excl - ls;   // global position = goff[bin] + local position
    __syncthreads();
    const uint32_t tile_n = min((uint32_t)SR_SORT_TILE, n - tile_base);
#pragma unroll
    for (int i = 0; i < SR_SORT_ITEMS; i++) {
        const uint32_t idx = wbase + i * 32 + lane;
        if (idx < n) {
            const uint32_t d = (uint32_t)((key[i] >> shift) & mask);
            const uint32_t pos = lstart[d] + whist[warp][d] + rank[i];
            keys_s[pos] = key[i];
            vals_s[pos] = val[i];
        }
    }
    __syncthreads();
    for (uint32_t j = tid; j < tile_n; j += SR_SORT_THREADS) {
        const uint64_t k = keys_s[j];
        const uint32_t d = (uint32_t)((k >> shift) & mask);
        const uint32_t out = goff[d] + j;
        kout[out] = k;
        vout[out] = vals_s[j];
    }
}

// identifyTileRanges + materialise the per-instance record stream (sorted order, 80 B each) that the
// composite kernels pull into shared memory with one bulk-async (TMA) copy per chunk.
//
// The 80-byte records are moved WARP-COOPERATIVELY: lane l carries 16-byte piece (l % 5) of instance (l / 5) of a group
// of six, so one LDG.128 / STG.128 covers six whole records -- 480 contiguous bytes on the store side -- instead of 32
// lanes each touching its own record at an 80-byte stride (r2a ncu: 24 % issue, 39 % DRAM, the load/store unit spent
// 32 cycles per instruction on 32 distinct sectors).
__global__ void __launch_bounds__(256)
ranges_gather_kernel(const FrameStrides fs, const uint64_t* __restrict__ keys0, const uint64_t* __restrict__ keys1,
                     const uint32_t* __restrict__ vals0, const uint32_t* __restrict__ vals1,
                     const uint32_t* __restrict__ ctl, const uint32_t* __restrict__ num_rendered, long long capacity,
                     const float4* __restrict__ srec, float4* __restrict__ irec, uint2* __restrict__ ranges, int tiles_x) {
    const int f = blockIdx.y;
    keys0 = fr(keys0, fs.bin, f); keys1 = fr(keys1, fs.bin, f); vals0 = fr(vals0, fs.bin, f); vals1 = fr(vals1, fs.bin, f);
    ctl = fr(ctl, fs.bin, f); num_rendered = fr(num_rendered, fs.nr, f); srec = fr(srec, fs.geom, f);
    irec = fr(irec, fs.bin, f); ranges = fr(ranges, fs.img, f);
    const uint32_t n = num_rendered[0];
    if ((long long)n > capacity) return;
    const uint32_t wbase = (blockIdx.x * 256u + threadIdx.x) & ~31u;      // first instance of this warp
    if (wbase >= n) return;                                                // whole warp out of range
    const int lane = threadIdx.x & 31;
    const uint32_t i = wbase + lane;
    const bool live = i < n;
    const uint32_t sel = ctl[SR_CTL_SORTED_SEL];
    const uint64_t* __restrict__ keys = sel ? keys1 : keys0;
    const uint32_t* __restrict__ vals = sel ? vals1 : vals0;
    uint32_t tile = 0, id = 0;
    if (live) {
        const uint64_t key = keys[i];
        tile = (uint32_t)(key >> 32);
        if (i == 0) ranges[tile].x = 0;
        else {
            const uint32_t prev = (uint32_t)(keys[i - 1] >> 32);
            if (tile != prev) { ranges[prev].y = i; ranges[tile].x = i; }
        }
        if (i == n - 1) ranges[tile].y = n;
        id = vals[i];
    }
    // ---- cooperative load: pass p moves instances 6p .. 6p+5 of the warp; lane = (slot k = lane / 5, piece = lane % 5)
    const int k = lane / 5, piece = lane - 5 * k;
    float4 v[6];
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const int inst = 6 * p + k;                                        // warp-local instance this lane helps to move
        const uint32_t sid = __shfl_sync(0xffffffffu, id, inst & 31);
        const bool ok = lane < 30 && inst < 32 && wbase + inst < n;
        v[p] = ok ? __ldg(srec + (size_t)sid * 5 + piece) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    // ---- lane = instance again: its opacity (piece 2, .w) and packed pixel bbox (piece 4, .z/.w) arrive by shuffle
    const int myp = lane / 6, myk = lane - 6 * myp;
    float opac = 0.f;
    uint32_t bx = 0, by = 0;
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const float o = __shfl_sync(0xffffffffu, v[p].w, 5 * myk + 2);
        const float zx = __shfl_sync(0xffffffffu, v[p].z, 5 * myk + 4);
        const float zy = __shfl_sync(0xffffffffu, v[p].w, 5 * myk + 4);
        if (p == myp) { opac = o; bx = __float_as_uint(zx); by = __float_as_uint(zy); }
    }
    const int tx = (int)(tile % (uint32_t)tiles_x) * SR_TILE, ty = (int)(tile / (uint32_t)tiles_x) * SR_TILE;
    const int x0 = max((int)(bx & 0xffffu) - tx, 0), x1 = min((int)(bx >> 16) - tx, SR_TILE - 1);
    const int y0 = max((int)(by & 0xffffu) - ty, 0), y1 = min((int)(by >> 16) - ty, SR_TILE - 1);
    uint32_t cull = 0;
    if (live && x0 <= x1 && y0 <= y1) {
        cull = (uint32_t)x0 | ((uint32_t)x1 << 4) | ((uint32_t)y0 << 8) | ((uint32_t)y1 << 12) | (1u << 16) | comp_cull_rho(opac);
    }
    // ---- cooperative store: the lane carrying piece 4 patches in the surfel id and the cull word
#pragma unroll
    for (int p = 0; p < 6; p++) {
        const int inst = 6 * p + k;
        const uint32_t cw = __shfl_sync(0xffffffffu, cull, inst & 31);
        const uint32_t sid = __shfl_sync(0xffffffffu, id, inst & 31);
        if (lane < 30 && inst < 32 && wbase + inst < n) {
            float4 o = v[p];
            if (piece == 4) { o.z = __uint_as_float(sid); o.w = __uint_as_float(cw); }
            irec[(size_t)(wbase + inst) * 5 + piece] = o;
        }
    }
}

// Longest-processing-time-first launch order for the composite kernels: tiles bucketed by floor(log2(len)),
// longest bucket first.  The CTA scheduler hands out work in blockIdx order, so the heavy tiles of an
// object-centric frame start first and the many light / empty ones fill the tail (round r1b ncu: SM busy
// cycles ranged 152K..548K with row-major order).
__global__ void __launch_bounds__(1024)
tile_order_kernel(const FrameStrides fs, const uint2* __restrict__ ranges, int tiles, uint32_t* __restrict__ order) {
    ranges = fr(ranges, fs.img, (int)blockIdx.x);   // one block per frame
    order = fr(order, fs.img, (int)blockIdx.x);
    __shared__ uint32_t cnt[33], start[33];
    if (threadIdx.x < 33) cnt[threadIdx.x] = 0;
    __syncthreads();
    for (int t = threadIdx.x; t < tiles; t += 1024) {
        const uint2 r = ranges[t];
        const uint32_t len = r.y - r.x;
        atomicAdd(&cnt[len ? 32 - __clz(len) : 0], 1u);     // bucket 0 = empty, b = floor(log2(len)) + 1
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t acc = 0;
        for (int b = 32; b >= 0; b--) { start[b] = acc; acc += cnt[b]; }
    }
    __syncthreads();
    for (int t = threadIdx.x; t < tiles; t += 1024) {
        const uint2 r = ranges[t];
        const uint32_t len = r.y - r.x;
        order[atomicAdd(&start[len ? 32 - __clz(len) : 0], 1u)] = (uint32_t)t;
    }
}

SortPlan make_plan(int key_bits) {
    SortPlan p{};
    int np = 0;
    for (int s = 0; s < key_bits && np < SR_SORT_MAX_PASSES; s += SR_SORT_RADIX_BITS) {
        p.shift[np] = s;
        p.bits[np] = key_bits - s < SR_SORT_RADIX_BITS ? key_bits - s : SR_SORT_RADIX_BITS;
        np++;
    }
    p.npass = np;
    return p;
}

}  // namespace

cudaError_t launch_sort(const FwdArgs& a) {
    const SortPlan plan = make_plan(a.key_bits);
    uint64_t* k0 = (uint64_t*)(a.bin + a.bl.keys[0]);
    uint64_t* k1 = (uint64_t*)(a.bin + a.bl.keys[1]);
    uint32_t* v0 = (uint32_t*)(a.bin + a.bl.values[0]);
    uint32_t* v1 = (uint32_t*)(a.bin + a.bl.values[1]);
    uint32_t* ctl = (uint32_t*)(a.bin + a.bl.sort_ctl);
    uint32_t* hist = (uint32_t*)(a.bin + a.bl.hist);
    uint32_t* status = (uint32_t*)(a.bin + a.bl.status);
    const long long cap = (long long)a.bl.capacity;
    const int hblocks = (int)((cap + 4095) / 4096);
    { ProfileScope ps("sort_histogram", a.stream);
      sort_histogram_kernel<<<dim3(hblocks, a.fs.frames), 256, 0, a.stream>>>(a.fs, k0, a.num_rendered_dev, cap, plan, hist); }
    { ProfileScope ps("sort_plan", a.stream);
      sort_plan_kernel<<<a.fs.frames, 256, 0, a.stream>>>(a.fs, hist, ctl, a.num_rendered_dev, cap, plan); }
    ProfileScope ps("onesweep_passes", a.stream);
    // SURFEL_SORT_INTERLEAVE=0 keeps each frame's blocks together: on the headline batch that pass time was ~1 % lower
    // with the end-to-end rates unchanged (DESIGN.md 3.2)
    static const int inter = [] { const char* e = getenv("SURFEL_SORT_INTERLEAVE"); return e && atoi(e) == 0 ? 0 : 1; }();
    const unsigned blocks = (unsigned)a.bl.sort_tiles * (unsigned)a.fs.frames;
    for (int p = 0; p < plan.npass; p++)
        onesweep_pass_kernel<<<blocks, SR_SORT_THREADS, 0, a.stream>>>(
            a.fs, k0, k1, v0, v1, hist, ctl, status, a.num_rendered_dev, p, plan.shift[p], plan.bits[p], a.bl.sort_tiles, inter);
    sr_count_launch(2 + plan.npass);
    return cudaGetLastError();
}

cudaError_t launch_ranges_gather(const FwdArgs& a) {
    const long long cap = (long long)a.bl.capacity;
    const int blocks = (int)((cap + 255) / 256);
    ProfileScope ps("ranges_gather", a.stream);
    ranges_gather_kernel<<<dim3(blocks, a.fs.frames), 256, 0, a.stream>>>(
        a.fs, (const uint64_t*)(a.bin + a.bl.keys[0]), (const uint64_t*)(a.bin + a.bl.keys[1]),
        (const uint32_t*)(a.bin + a.bl.values[0]), (const uint32_t*)(a.bin + a.bl.values[1]),
        (const uint32_t*)(a.bin + a.bl.sort_ctl), a.num_rendered_dev, cap,
        (const float4*)(a.geom + a.gl.surfel_rec), (float4*)(a.bin + a.bl.inst_rec),
        (uint2*)(a.img + a.il.ranges), a.il.tiles_x);
    sr_count_launch();
    return cudaGetLastError();
}

cudaError_t launch_tile_order(const FwdArgs& a) {
    ProfileScope ps("tile_order", a.stream);
    tile_order_kernel<<<a.fs.frames, 1024, 0, a.stream>>>(a.fs, (const uint2*)(a.img + a.il.ranges), a.il.tiles,
                                                 (uint32_t*)(a.img + a.il.tile_order));
    sr_count_launch();
    return cudaGetLastError();
}
