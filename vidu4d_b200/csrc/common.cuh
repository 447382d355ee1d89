// common.cuh -- shared definitions for the sm_90a surfel rasterizer kernels.
//
// Vocabulary follows the reference (RAST = gs/submodules/diff-surfel-rasterization):
//   surfel    one 2D Gaussian disc (P of them)
//   instance  one (surfel, 16x16 tile) overlap; R = num_rendered of them
//   tile      16x16 pixel block (RAST/cuda_rasterizer/config.h:16-17)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include "../../include/surfel_raster.h"

#define SR_TILE 16               // BLOCK_X == BLOCK_Y == 16 in the reference
#define SR_REC_FLOATS 20         // floats per surfel / instance record (80 B = 5 x float4)
#define SR_GRAD_FLOATS 20        // floats per surfel gradient accumulator (80 B)

// ---- record layout (float index) --------------------------------------------------------
//  0..8   T   rows Tu, Tv, Tw of the tangent-plane -> pixel homography (forward.cu:117-125)
//  9,10   xy  centre of the projected 1-sigma bounding box (forward.cu:160)
//  11     opacity
//  12..14 normal (view space, flipped to face the camera)
//  15..17 rgb (after SH evaluation / clamp, or colors_precomp)
//  18     surfel record: packed conservative pixel bbox x (lo16 = x0, hi16 = x1)
//         instance record: surfel id
//  19     surfel record: packed conservative pixel bbox y
//         instance record: tile-local cull rect  lx0 | lx1<<4 | ly0<<8 | ly1<<12 | valid<<16 | rho_cut(1/1024)<<17
#define SR_R_T 0
#define SR_R_XY 9
#define SR_R_OPAC 11
#define SR_R_NORMAL 12
#define SR_R_RGB 15
#define SR_R_W18 18
#define SR_R_W19 19

// ---- gradient accumulator layout (float index), one per surfel ----------------------------
//  0..8 dL/dT   9 dL/dopacity   10..12 dL/dcolor   13..15 dL/dnormal   16,17 dL/dmean2D (low-pass branch)
//  Slots 0..15 are, in order, the 16 components of the composite backward's butterfly, so that a lane's 2 or 4
//  consecutive totals leave as ONE 8- or 16-byte vector reduction (REDG.ADD.F32x2 / x4).
#define SR_G_T 0
#define SR_G_OPAC 9
#define SR_G_COLOR 10
#define SR_G_NORMAL 13
#define SR_G_M2D 16

#define SR_CONTRIB_STAGE_WORDS 256  // 8 sub-tiles x 32 pixels, one 32-bit instance mask each (1 KB per stage)
#define SR_SORT_MAX_PASSES 8
#define SR_SORT_RADIX_BITS 8
#define SR_SORT_BINS 256
#define SR_SORT_THREADS 256
#define SR_SORT_ITEMS 12
#define SR_SORT_TILE (SR_SORT_THREADS * SR_SORT_ITEMS)

// sort_ctl words (uint32)
#define SR_CTL_SORTED_SEL 0      // which ping/pong array holds the sorted result
#define SR_CTL_NPASS 1
#define SR_CTL_SKIP 8            // [8 .. 8+MAX_PASSES): 1 = pass is an identity permutation, skipped
#define SR_CTL_SRC 16            // [16 .. 16+MAX_PASSES): source array (0/1) of pass p
#define SR_CTL_TILE_COUNTER 24   // [24 .. 24+MAX_PASSES): dynamic tile ids of pass p
#define SR_CTL_WORDS 64

static inline __host__ __device__ size_t sr_align_up(size_t x, size_t a = 256) { return (x + a - 1) / a * a; }

struct GeomLayout {
    size_t surfel_rec, depths, tiles_touched, point_offsets, clamped, block_sums, sgrad, total;
    int nblocks;
};
struct ImageLayout {
    size_t final_T, n_contrib, ranges, tile_last, tile_order, total;
    int tiles_x, tiles_y, tiles;
};
struct BinLayout {
    size_t keys[2], values[2], inst_rec, contrib, sort_ctl, hist, status, total;
    int64_t capacity;
    int sort_tiles;
};

static inline __host__ __device__ GeomLayout geom_layout(int P) {
    GeomLayout L;
    size_t Pa = P > 0 ? (size_t)P : 1, o = 0;
    L.nblocks = (int)((Pa + 255) / 256);
    L.surfel_rec = o;    o = sr_align_up(o + Pa * SR_REC_FLOATS * 4);
    L.depths = o;        o = sr_align_up(o + Pa * 4);
    L.tiles_touched = o; o = sr_align_up(o + Pa * 4);
    L.point_offsets = o; o = sr_align_up(o + Pa * 4);
    L.clamped = o;       o = sr_align_up(o + Pa);
    L.block_sums = o;    o = sr_align_up(o + ((size_t)L.nblocks + 1) * 4);
    L.sgrad = o;         o = sr_align_up(o + Pa * SR_GRAD_FLOATS * 4);
    L.total = o;
    return L;
}
static inline __host__ __device__ ImageLayout image_layout(int W, int H) {
    ImageLayout L;
    size_t N = (size_t)W * H, o = 0;
    L.tiles_x = (W + SR_TILE - 1) / SR_TILE; L.tiles_y = (H + SR_TILE - 1) / SR_TILE;
    L.tiles = L.tiles_x * L.tiles_y;
    L.final_T = o;   o = sr_align_up(o + 3 * N * 4);
    L.n_contrib = o; o = sr_align_up(o + 2 * N * 4);
    L.ranges = o;    o = sr_align_up(o + (size_t)L.tiles * 8);
    L.tile_last = o; o = sr_align_up(o + (size_t)L.tiles * 8 * 4);   // per 8x4 sub-tile: deepest contributor
    L.tile_order = o; o = sr_align_up(o + (size_t)L.tiles * 4);       // tiles, longest instance list first
    L.total = o;
    return L;
}
static inline __host__ __device__ BinLayout bin_layout(int64_t capacity, int tiles) {
    BinLayout L;
    size_t C = capacity > 0 ? (size_t)capacity : 1, o = 0;
    L.capacity = (int64_t)C;
    L.sort_tiles = (int)((C + SR_SORT_TILE - 1) / SR_SORT_TILE);
    L.keys[0] = o;   o = sr_align_up(o + C * 8);
    L.keys[1] = o;   o = sr_align_up(o + C * 8);
    L.values[0] = o; o = sr_align_up(o + C * 4);
    L.values[1] = o; o = sr_align_up(o + C * 4);
    L.inst_rec = o;  o = sr_align_up(o + C * SR_REC_FLOATS * 4);
    // contribution masks: per (32-instance stage of a tile list, 8x4 sub-tile, pixel) the instances that
    // contributed to the pixel -- written by the forward composite, walked by the backward.
    // Stage s of tile t lives at index (range.x >> 5) + t + s  (<= capacity/32 + tiles in total).
    L.contrib = o;   o = sr_align_up(o + ((C >> 5) + (size_t)(tiles > 0 ? tiles : 0) + 1) * SR_CONTRIB_STAGE_WORDS * 4);
    // the three below are zeroed together by one memset at the start of every forward
    L.sort_ctl = o;  o = sr_align_up(o + SR_CTL_WORDS * 4);
    L.hist = o;      o = sr_align_up(o + (size_t)SR_SORT_MAX_PASSES * SR_SORT_BINS * 4);
    L.status = o;    o = sr_align_up(o + (size_t)SR_SORT_MAX_PASSES * L.sort_tiles * SR_SORT_BINS * 4);
    L.total = o;
    return L;
}

// Host-side uniform parameters shared by the per-surfel kernels.
struct CamParams {
    const float* vm;       // DEVICE viewmatrix[16] as passed (column-major 4x4 in glm terms)
    const float* campos;   // DEVICE [3]
    const float* bg;       // DEVICE [3]
    float focal_x, focal_y, cx, cy;     // forward intrinsics: cx = W/2, cy = H/2 (forward.cu:208)
    float bcx, bcy;                     // backward intrinsics: focal*tanfov (backward.cu:570)
    int W, H, tiles_x, tiles_y;
    int P, D, M;
};

// getHigherMsb, rasterizer_impl.cu:35-50
static inline uint32_t sr_higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) { step /= 2; if (n >> msb) msb += step; else msb -= step; }
    if (n >> msb) msb++;
    return msb;
}

// Batched launches: every kernel of the path processes `frames` independent frames in ONE launch (frame = blockIdx.y, or
// interleaved into blockIdx.x for the composite kernels so that the longest tiles of ALL frames start first).  The
// kernels receive frame 0's pointers plus the BYTE distance between consecutive frames of each array (0 = the array
// is shared by every frame, e.g. the SH coefficients of a Stage-3 batch).
struct FrameStrides {
    int frames;
    long long geom, bin, img, nr;                                        // scratch buffers, {num_rendered, status} words
    long long means3D, shs, colors, opac, scales, rots, vm, campos;      // inputs
    long long out_color, out_others, radii;                              // forward outputs
    long long dcolor, dothers;                                           // backward inputs
    long long g_m2d, g_col, g_opac, g_m3d, g_tm, g_sh, g_scales, g_rots; // backward outputs
};

// ---- launchers implemented in the .cu files ------------------------------------------------
struct FwdArgs {
    FrameStrides fs;
    CamParams cam;
    const float* means3D; const float* shs; const float* colors_precomp; const float* opacities;
    const float* scales; const float* rotations;
    float* out_color; float* out_others; int* radii;
    char* geom; char* bin; char* img;
    GeomLayout gl; BinLayout bl; ImageLayout il;
    uint32_t* num_rendered_dev;   // [0]=R, [1]=status
    int prefiltered;
    int key_bits;                 // 32 + getHigherMsb(tiles)
    cudaStream_t stream;
    bool debug;
};
struct BwdArgs {
    FrameStrides fs;
    const float* grad_scale;      // optional DEVICE scalar multiplying dL_dcolor / dL_dothers (nullptr = 1)
    CamParams cam;
    const float* means3D; const float* shs; const float* colors_precomp;
    const float* scales; const float* rotations; const int* radii;
    const float* dL_dcolor; const float* dL_dothers;
    char* geom; char* bin; char* img;
    GeomLayout gl; BinLayout bl; ImageLayout il;
    float* dL_dmeans2D; float* dL_dcolors; float* dL_dopacity; float* dL_dmeans3D;
    float* dL_dtransMat; float* dL_dsh; float* dL_dscales; float* dL_drotations;
    cudaStream_t stream;
    bool debug;
};

cudaError_t launch_preprocess_fwd(const FwdArgs& a);      // preprocess.cu
cudaError_t launch_scan_emit(const FwdArgs& a);           // preprocess.cu
cudaError_t launch_sort(const FwdArgs& a);                // sort.cu
cudaError_t launch_ranges_gather(const FwdArgs& a);       // sort.cu
cudaError_t launch_tile_order(const FwdArgs& a);          // sort.cu
cudaError_t launch_composite_fwd(const FwdArgs& a);       // composite_fwd.cu
cudaError_t launch_composite_bwd(const BwdArgs& a);       // composite_bwd.cu
cudaError_t launch_surfel_bwd(const BwdArgs& a);          // surfel_bwd.cu
cudaError_t launch_composite_tile_fwd(const FwdArgs& a);  // composite_tile.cu (one CTA per tile, shared chunk ring)
cudaError_t launch_composite_tile_bwd(const BwdArgs& a);  // composite_tile.cu
bool sr_composite_tile_mode(bool backward);               // SURFEL_COMPOSITE[_FWD|_BWD]=tile|warp
cudaError_t launch_mark_visible(int P, const float* means3D, const float* vm, uint8_t* present, cudaStream_t s);
// clears `bytes` at p + f * pitch for every frame f of the batch (one 2-D memset)
cudaError_t sr_memset_frames(void* p, size_t pitch, size_t bytes, int frames, cudaStream_t s);

void sr_count_launch(int n = 1);

// Optional per-kernel timing (sr_set_profiling): CUDA events recorded on the launching stream around each
// kernel; read back (after a sync) with sr_get_profile().  Off by default: zero overhead on the hot path.
bool sr_profiling_on();
void sr_profile_push(const char* name, cudaEvent_t e0, cudaEvent_t e1);
struct ProfileScope {
    const char* name; cudaStream_t stream; cudaEvent_t e0 = nullptr, e1 = nullptr; bool on;
    ProfileScope(const char* n, cudaStream_t s) : name(n), stream(s), on(sr_profiling_on()) {
        if (on) { cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0, stream); }
    }
    ~ProfileScope() { if (on) { cudaEventRecord(e1, stream); sr_profile_push(name, e0, e1); } }
};

// ---- small device helpers -----------------------------------------------------------------
#ifdef __CUDACC__
// frame f's copy of an array whose frame 0 starts at p (nullptr stays nullptr)
template <class T>
__device__ __forceinline__ T* fr(T* p, long long stride_bytes, int f) {
    return p ? reinterpret_cast<T*>(reinterpret_cast<uintptr_t>(p) + (uintptr_t)((long long)f * stride_bytes)) : p;
}
__device__ __forceinline__ CamParams cam_of_frame(CamParams c, const FrameStrides& fs, int f) {
    c.vm = fr(c.vm, fs.vm, f);
    c.campos = fr(c.campos, fs.campos, f);
    return c;
}
__device__ __forceinline__ float4 ld_nc_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// mbarrier + bulk async copy (TMA 1-D) -- sm_90+
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE;\n"
        "bra WAIT_LOOP;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(smem_dst)),
                 "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}
#endif
