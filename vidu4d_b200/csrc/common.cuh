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

// forward_only (sr_render_forward's arena): the arrays only a backward reads -- the geometry's gradient accumulator
// sgrad, the binning's contribution masks, the image's final_T, n_contrib and sub_last (tile_last) -- take no bytes;
// their offsets alias the next array's and nothing touches them.
static inline __host__ __device__ GeomLayout geom_layout(int P, bool forward_only = false) {
    GeomLayout L;
    size_t Pa = P > 0 ? (size_t)P : 1, o = 0;
    L.nblocks = (int)((Pa + 255) / 256);
    L.surfel_rec = o;    o = sr_align_up(o + Pa * SR_REC_FLOATS * 4);
    L.depths = o;        o = sr_align_up(o + Pa * 4);
    L.tiles_touched = o; o = sr_align_up(o + Pa * 4);
    L.point_offsets = o; o = sr_align_up(o + Pa * 4);
    L.clamped = o;       o = sr_align_up(o + Pa);
    L.block_sums = o;    o = sr_align_up(o + ((size_t)L.nblocks + 1) * 4);
    L.sgrad = o;         if (!forward_only) o = sr_align_up(o + Pa * SR_GRAD_FLOATS * 4);
    L.total = o;
    return L;
}
static inline __host__ __device__ ImageLayout image_layout(int W, int H, bool forward_only = false) {
    ImageLayout L;
    size_t N = (size_t)W * H, o = 0;
    L.tiles_x = (W + SR_TILE - 1) / SR_TILE; L.tiles_y = (H + SR_TILE - 1) / SR_TILE;
    L.tiles = L.tiles_x * L.tiles_y;
    L.final_T = o;   if (!forward_only) o = sr_align_up(o + 3 * N * 4);
    L.n_contrib = o; if (!forward_only) o = sr_align_up(o + 2 * N * 4);
    L.ranges = o;    o = sr_align_up(o + (size_t)L.tiles * 8);
    L.tile_last = o; if (!forward_only) o = sr_align_up(o + (size_t)L.tiles * 8 * 4);   // per 8x4 sub-tile: deepest contributor
    L.tile_order = o; o = sr_align_up(o + (size_t)L.tiles * 4);       // tiles, longest instance list first
    L.total = o;
    return L;
}
static inline __host__ __device__ BinLayout bin_layout(int64_t capacity, int tiles, bool forward_only = false) {
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
    // contributed to the pixel -- written by the forward composite, walked by the backward (contrib_word).
    // Stage s of tile t lives at index (range.x >> 5) + t + s  (<= capacity/32 + tiles in total).
    L.contrib = o;
    if (!forward_only) o = sr_align_up(o + ((C >> 5) + (size_t)(tiles > 0 ? tiles : 0) + 1) * SR_CONTRIB_STAGE_WORDS * 4);
    // the three below are zeroed together by one memset at the start of every forward
    L.sort_ctl = o;  o = sr_align_up(o + SR_CTL_WORDS * 4);
    L.hist = o;      o = sr_align_up(o + (size_t)SR_SORT_MAX_PASSES * SR_SORT_BINS * 4);
    L.status = o;    o = sr_align_up(o + (size_t)SR_SORT_MAX_PASSES * L.sort_tiles * SR_SORT_BINS * 4);
    L.total = o;
    return L;
}
// Index, in words from L.contrib, of the contribution mask of slot `slot` (pixel ly * 8 + lx) of 8x4 sub-tile `sub` in
// stage 0 of tile `tile`, whose sorted list starts at instance range_x.  Stage s of the tile is
// s * SR_CONTRIB_STAGE_WORDS words further.
static inline __host__ __device__ size_t contrib_word(uint32_t range_x, int tile, int sub, int slot) {
    return (((size_t)(range_x >> 5) + tile) * 8 + sub) * 32 + slot;
}

// Host-side uniform parameters shared by the per-surfel kernels.
struct CamParams {
    const float* vm;       // DEVICE viewmatrix[16] as passed (column-major 4x4 in glm terms)
    const float* campos;   // DEVICE [3]
    const float* bg;       // DEVICE [3]
    const float* cams;     // DEVICE [frames*4] per-frame (tan_x, tan_y, cx_off, cy_off), or nullptr: the scalars below
    float focal_x, focal_y, cx, cy;     // forward intrinsics: cx = W/2 + cx_off, cy = H/2 + cy_off (forward.cu:208)
    float bcx, bcy;                     // backward intrinsics: focal*tanfov (backward.cu:570), the mean2D proxy's scale
    float kcx, kcy;                     // backward K's principal point: bcx + cx_off, bcy + cy_off
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
struct FeatArgs;
// Per-surfel contribution statistics of sr_render_forward_contrib (include/surfel_render.h), added into by every
// contributing (frame, pixel, surfel) pair of the forward-only walk, w = T alpha rounded once; or, with `anchors`, where
// sr_render_forward_anchors writes each pixel's heaviest pairs instead.  The anchors' words share the statistics' bytes
// and their flag the lift flag's padding, so that the kernel parameter keeps its size and the other walks their code.
struct ContribArgs {
    union {
        struct {
            unsigned long long* weight_q;  // [P] sum of rn(w 2^32)
            uint32_t* max_weight;          // [P] max of w, as float bits
            unsigned long long* pixels;    // [P] number of pairs
            // sr_render_forward_contrib_masked: frame m's H*W foreground bytes at mask + m*mask_stride (0 = background),
            // and the two sums over the pairs on background pixels; mask = nullptr gathers the three words above alone
            const uint8_t* mask;
            long long mask_stride;         // bytes
            unsigned long long* weight_bg_q;  // [P] sum of rn(w 2^32) over the background pairs
            unsigned long long* pixels_bg;    // [P] number of background pairs
        };
        struct {
            // sr_render_forward_anchors: each pixel's anchor_K heaviest contributing pairs, frame m's (K, H, W) ids and
            // weights at + m*anchor_stride elements, its (K, 2, H, W) hit coordinates at anchor_uv + 2m*anchor_stride; a
            // frame whose status word (anchor_status + m*fs.nr bytes) has SR_STATUS_OVERFLOW set writes none
            int32_t* anchor_ids;
            float* anchor_w;
            float* anchor_uv;
            const uint32_t* anchor_status;
            long long anchor_stride;       // elements
            int anchor_K;                  // 1, 2, 4 or 8
        };
    };
    // sr_render_forward_lift (lift = true): frame m's (C, H, W) values at lift_values + m*lift_stride, each pair's
    // rn(w v 2^s) added into lift_sums[surfel * C + c], clamped and non-finite values counted in lift_saturated
    bool lift;
    bool anchors;                  // sr_render_forward_anchors: the union holds the anchors' words, no statistics
    int lift_C;                    // 1..32
    const float* lift_values;
    long long lift_stride;         // bytes
    float lift_scale;              // 2^s
    int lift_scale_log2;           // s
    long long* lift_sums;          // [P * C]
    unsigned long long* lift_saturated;  // [1]
};
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
    // sr_render_forward: the layouts are forward_only, the composite keeps no backward state and composites the feature
    // channels `feat` (nullptr when F = 0) in its own walk
    bool forward_only;
    const FeatArgs* feat;
    const ContribArgs* contrib;   // forward-only: the statistics to add into, or nullptr
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

// Per-surfel feature channels composited with the colour's weights (composite_feat.cu).  Strides are in BYTES between
// consecutive frames (0 = shared by every frame, for `feat` and `dfeat` only).
#define SR_FEAT_MAX 32           // channels per call
#define SR_FEAT_CHUNK 8          // channels one CTA accumulates (gridDim.y = ceil(F / SR_FEAT_CHUNK))
struct FeatArgs {
    int F;                        // 1..SR_FEAT_MAX
    int vec;                      // 4, 2 or 1: floats per vector access of a feature row (F % vec == 0, aligned)
    const float* feat;  long long feat_stride;     // [P*F] per frame
    const float* bg;                               // DEVICE bg[F] of the feature planes, nullptr = 0
    float* out;         long long out_stride;      // forward: F planes of H*W per frame
    const float* dout;  long long dout_stride;     // backward: dL/d(feature planes)
    const float* grad_scale;                       // optional DEVICE scalar multiplying dout (nullptr = 1)
    float* dfeat;       long long dfeat_stride;    // backward: dL/dfeatures [P*F], zeroed by the launcher
};

// the forward's camera of an sr_frame (api.cu): intrinsics from its tangents, or its per-frame table
CamParams make_cam(const sr_frame* f, const float* vm, const float* campos, const float* bg);

cudaError_t launch_preprocess_fwd(const FwdArgs& a);      // preprocess.cu
cudaError_t launch_scan_emit(const FwdArgs& a);           // preprocess.cu
cudaError_t launch_sort(const FwdArgs& a);                // sort.cu
cudaError_t launch_ranges_gather(const FwdArgs& a);       // sort.cu
cudaError_t launch_tile_order(const FwdArgs& a);          // sort.cu
cudaError_t launch_composite_fwd(const FwdArgs& a);       // composite_fwd.cu
cudaError_t launch_surfel_bwd(const BwdArgs& a);          // surfel_bwd.cu
cudaError_t launch_composite_tile_fwd(const FwdArgs& a);  // composite_tile.cu (one CTA per tile, shared chunk ring)
cudaError_t launch_composite_tile_bwd(const BwdArgs& a);  // composite_tile.cu
bool sr_composite_tile_fwd();                             // SURFEL_COMPOSITE[_FWD]=tile|warp
cudaError_t launch_feature_fwd(const FwdArgs& a, const FeatArgs& ft);   // composite_feat.cu (after the composite forward)
cudaError_t launch_feature_bwd(const BwdArgs& a, const FeatArgs& ft);   // composite_feat.cu (after the composite backward)
// Deterministic backward (include/surfel_deterministic.h): per frame, one 20-float slot per instance (the geometry /
// colour gradient of one (instance, tile), accumulator layout SR_G_*) and F floats per instance (its dL/dfeatures), both
// indexed by the instance's emission index.  Strides in BYTES between consecutive frames.
struct DetArgs {
    float* slots;  long long slots_stride;
    float* fslots; long long fslots_stride;         // nullptr when F = 0
    const uint32_t* point_offsets;                  // the geometry buffer's (frame stride FrameStrides::geom)
    const int* radii;                               // (frame stride FrameStrides::radii)
    int tiles_y;
};
static inline size_t det_slot_bytes(int64_t capacity) { return sr_align_up((size_t)(capacity > 0 ? capacity : 1) * SR_GRAD_FLOATS * 4); }
static inline size_t det_fslot_bytes(int64_t capacity, int F) { return sr_align_up((size_t)(capacity > 0 ? capacity : 1) * (F > 0 ? F : 0) * 4); }
cudaError_t launch_det_zero(const BwdArgs& a, const DetArgs& d, int F);                      // composite_det.cu
cudaError_t launch_composite_tile_bwd_det(const BwdArgs& a, const DetArgs& d);              // composite_tile.cu
cudaError_t launch_feature_bwd_det(const BwdArgs& a, const FeatArgs& ft, const DetArgs& d); // composite_det.cu
cudaError_t launch_det_gather(const BwdArgs& a, const DetArgs& d, const FeatArgs* ft);     // composite_det.cu
cudaError_t launch_mark_visible(int P, const float* means3D, const float* vm, uint8_t* present, cudaStream_t s);
// clears `bytes` at p + f * pitch for every frame f of the batch (one 2-D memset)
cudaError_t sr_memset_frames(void* p, size_t pitch, size_t bytes, int frames, cudaStream_t s);

void sr_count_launch(int n = 1);

// ---- error reporting: every failing entry point sets the message sr_last_error() returns ---------------------------
// sets the calling thread's message (printf format) and returns `code`
int sr_fail(int code, const char* fmt, ...) __attribute__((format(printf, 2, 3)));
static inline int cuda_fail(cudaError_t e, const char* where) {
    return sr_fail(SR_ECUDA, "CUDA error in %s: %s", where, cudaGetErrorString(e));
}
// returns SR_ECUDA (naming `where`) from the enclosing function if a CUDA runtime call fails
#define CK(call, where)                                      \
    do {                                                     \
        cudaError_t e_ = (call);                             \
        if (e_ != cudaSuccess) return cuda_fail(e_, where);  \
    } while (0)
// epilogue of an entry point that launched `n` kernels: counts them, then turns a pending launch error into SR_ECUDA
int sr_launched(int n, const char* where);

// Opts `kern` in to `bytes` of dynamic shared memory.  Nothing to do up to the default 48 KB; above it the attribute
// belongs to the current device's context, so the largest size set so far is remembered per (kernel, device) and a
// request within it costs no driver call.  Safe to call from several threads.
cudaError_t sr_opt_in_smem(const void* kern, size_t bytes);
template <class K>
cudaError_t sr_opt_in_smem(K* kern, size_t bytes) { return sr_opt_in_smem((const void*)kern, bytes); }
// dynamic shared memory the bone / frame tables of the warp, reprojection and cycle kernels may take (B <= 64)
#define SR_TABLE_SMEM_MAX (200 * 1024)

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
// Frame f's camera.  With a per-frame table (c.cams), its intrinsics come from row f by make_cam's own operations (each
// one rounded on its own, as the host rounds them), then the principal-point offset is added: a row holding the launch's
// tangents and zero offsets reproduces the scalar intrinsics bit for bit.  The row is read as four scalar loads, so the
// table needs no more than float alignment.  Its values are not checked.
__device__ __forceinline__ CamParams cam_of_frame(CamParams c, const FrameStrides& fs, int f) {
    c.vm = fr(c.vm, fs.vm, f);
    c.campos = fr(c.campos, fs.campos, f);
    if (c.cams) {
        const float* r = c.cams + 4 * (size_t)f;
        const float tx = __ldg(r), ty = __ldg(r + 1), ox = __ldg(r + 2), oy = __ldg(r + 3);
        c.focal_y = __fdiv_rn((float)c.H, __fmul_rn(2.0f, ty));
        c.focal_x = __fdiv_rn((float)c.W, __fmul_rn(2.0f, tx));
        c.cx = __fadd_rn(__fmul_rn((float)c.W, 0.5f), ox);
        c.cy = __fadd_rn(__fmul_rn((float)c.H, 0.5f), oy);
        c.bcx = __fmul_rn(c.focal_x, tx);
        c.bcy = __fmul_rn(c.focal_y, ty);
        c.kcx = __fadd_rn(c.bcx, ox);
        c.kcy = __fadd_rn(c.bcy, oy);
    }
    return c;
}
// The tile rectangle [rmin, rmax) of a surfel centred at (px, py) with radius max_radius (getRect, auxiliary.h:64-74).
// The float operations are exact by construction (adds and power-of-two scaling).  emit_keys emits a surfel's instances
// row-major over this rectangle; the deterministic backward recomputes it to find an instance's emission index.
__device__ __forceinline__ void sr_tile_rect(float px, float py, int max_radius, int gx, int gy, uint2& rmin, uint2& rmax) {
    const float r = (float)max_radius;
    int x0 = (int)__fmul_rn(__fadd_rn(px, -r), 0.0625f), y0 = (int)__fmul_rn(__fadd_rn(py, -r), 0.0625f);
    int x1 = (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(px, r), 16.f), -1.f), 0.0625f);
    int y1 = (int)__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(py, r), 16.f), -1.f), 0.0625f);
    rmin.x = min((unsigned)gx, (unsigned)max(0, x0));
    rmin.y = min((unsigned)gy, (unsigned)max(0, y0));
    rmax.x = min((unsigned)gx, (unsigned)max(0, x1));
    rmax.y = min((unsigned)gy, (unsigned)max(0, y1));
}
// Emission index of surfel id's instance on tile (tx, ty): the surfel's first index (point_offsets is the inclusive scan
// of tiles_touched) plus the tile's row-major position in its rectangle
__device__ __forceinline__ uint32_t sr_emission_index(const uint32_t* __restrict__ point_offsets, const int* __restrict__ radii,
                                                      uint32_t id, float px, float py, int tx, int ty, int gx, int gy) {
    uint2 rmin, rmax;
    sr_tile_rect(px, py, __ldg(radii + id), gx, gy, rmin, rmax);
    const uint32_t first = id == 0 ? 0u : __ldg(point_offsets + id - 1);
    return first + ((uint32_t)ty - rmin.y) * (rmax.x - rmin.x) + ((uint32_t)tx - rmin.x);
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
