// api.cu -- the C ABI declared in include/surfel_raster.h: argument checking, buffer layout,
// launch orchestration.  Replaces the host side of the reference:
//   Rasterizer::forward / backward / markVisible   RAST/cuda_rasterizer/rasterizer_impl.cu:141-153,198-342,346-448
//   GeometryState/ImageState/BinningState::fromChunk, required<T>   rasterizer_impl.cu:155-194, rasterizer_impl.h:66-72
// No torch types; no host<->device synchronisation on the forward/backward path (debug mode excepted).
#include <atomic>
#include <initializer_list>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "common.cuh"
#include "../../include/surfel_camera.h"
#include "../../include/surfel_deterministic.h"
#include "../../include/surfel_render.h"

namespace {
thread_local char g_err[512] = "";
std::atomic<uint64_t> g_launches{0};

#define DBG(where)                                           \
    do {                                                     \
        if (debug) CK(cudaStreamSynchronize(stream), where); \
    } while (0)
}  // namespace

CamParams make_cam(const sr_frame* f, const float* vm, const float* campos, const float* bg) {
    CamParams c{};
    c.vm = vm; c.campos = campos; c.bg = bg;
    c.W = f->width; c.H = f->height;
    c.tiles_x = (f->width + SR_TILE - 1) / SR_TILE;
    c.tiles_y = (f->height + SR_TILE - 1) / SR_TILE;
    c.P = f->P; c.D = f->sh_degree; c.M = f->sh_coeffs;
    // rasterizer_impl.cu:223-224
    c.focal_y = f->height / (2.0f * f->tan_fovy);
    c.focal_x = f->width / (2.0f * f->tan_fovx);
    // forward.cu:208  {focal_x, focal_y, float(W)/2.0, float(H)/2.0}
    c.cx = (float)((float)f->width / 2.0);
    c.cy = (float)((float)f->height / 2.0);
    // backward.cu:570 / 683-684
    c.bcx = c.focal_x * f->tan_fovx;
    c.bcy = c.focal_y * f->tan_fovy;
    c.kcx = c.bcx; c.kcy = c.bcy;
    // SR_FRAME_CAMERAS: the kernels replace the intrinsics above with each frame's row (common.cuh cam_of_frame)
    c.cams = (f->flags & SR_FRAME_CAMERAS) ? reinterpret_cast<const sr_frame_cameras*>(f)->cameras : nullptr;
    return c;
}

namespace {

int check_frame(const sr_frame* f) {
    if (!f) return sr_fail(SR_EINVAL, "frame descriptor is NULL");
    if (f->P < 0) return sr_fail(SR_EINVAL, "P must be >= 0");
    if (f->width <= 0 || f->height <= 0) return sr_fail(SR_EINVAL, "image size must be positive");
    if (f->width > 65535 || f->height > 65535) return sr_fail(SR_EINVAL, "image side must be < 65536");
    if (f->sh_degree < 0 || f->sh_degree > 3) return sr_fail(SR_EINVAL, "sh_degree must be 0..3");
    if (f->sh_coeffs < 0) return sr_fail(SR_EINVAL, "sh_coeffs must be >= 0");
    if ((f->flags & SR_FRAME_CAMERAS) && !reinterpret_cast<const sr_frame_cameras*>(f)->cameras)
        return sr_fail(SR_EINVAL, "SR_FRAME_CAMERAS is set but the per-frame camera table is NULL");
    if (f->sh_coeffs > 0 && (f->sh_degree + 1) * (f->sh_degree + 1) > f->sh_coeffs)
        return sr_fail(SR_EINVAL, "sh_degree %d needs %d coefficients, shs has %d", f->sh_degree,
                       (f->sh_degree + 1) * (f->sh_degree + 1), f->sh_coeffs);
    return 0;
}
}  // namespace

void sr_count_launch(int n) { g_launches.fetch_add((uint64_t)n, std::memory_order_relaxed); }

int sr_fail(int code, const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
}

int sr_launched(int n, const char* where) {
    sr_count_launch(n);
    const cudaError_t e = cudaGetLastError();
    return e == cudaSuccess ? 0 : cuda_fail(e, where);
}

cudaError_t sr_opt_in_smem(const void* kern, size_t bytes) {
    if (bytes <= 48 * 1024) return cudaSuccess;
    int dev = 0;
    if (cudaError_t e = cudaGetDevice(&dev)) return e;
    static std::mutex mu;
    static std::map<std::pair<const void*, int>, size_t> done;   // largest size set per (kernel, device)
    std::lock_guard<std::mutex> lk(mu);
    size_t& have = done[{kern, dev}];
    if (bytes <= have) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) have = bytes;
    return e;
}

cudaError_t sr_memset_frames(void* p, size_t pitch, size_t bytes, int frames, cudaStream_t s) {
    if (frames == 1) return cudaMemsetAsync(p, 0, bytes, s);
    return cudaMemset2DAsync(p, pitch, 0, bytes, (size_t)frames, s);
}

namespace {
std::atomic<bool> g_profiling{false};
std::mutex g_prof_mu;
struct ProfRec { const char* name; cudaEvent_t e0, e1; };
std::vector<ProfRec> g_prof;
std::string g_prof_json;
}  // namespace
bool sr_profiling_on() { return g_profiling.load(std::memory_order_relaxed); }
void sr_profile_push(const char* name, cudaEvent_t e0, cudaEvent_t e1) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.push_back({name, e0, e1});
}

extern "C" {

int sr_abi_version(void) { return SR_ABI_VERSION; }
const char* sr_last_error(void) { return g_err; }
uint64_t sr_launch_count(void) { return g_launches.load(); }

void sr_set_profiling(int on) { g_profiling.store(on != 0); }

// Synchronises the device, then returns {"kernel": {"ms": total, "count": n}, ...} for everything recorded
// since the previous call.  The returned pointer stays valid until the next call.
const char* sr_get_profile(void) {
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> lk(g_prof_mu);
    std::map<std::string, std::pair<double, int>> acc;
    for (auto& r : g_prof) {
        float ms = 0.f;
        if (cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess) { acc[r.name].first += ms; acc[r.name].second += 1; }
        cudaEventDestroy(r.e0); cudaEventDestroy(r.e1);
    }
    g_prof.clear();
    g_prof_json = "{";
    bool first = true;
    for (auto& kv : acc) {
        char buf[256];
        snprintf(buf, sizeof(buf), "%s\"%s\": {\"ms\": %.6f, \"count\": %d}", first ? "" : ", ", kv.first.c_str(), kv.second.first, kv.second.second);
        g_prof_json += buf; first = false;
    }
    g_prof_json += "}";
    return g_prof_json.c_str();
}

size_t sr_geom_bytes(int32_t P) { return geom_layout(P).total; }
size_t sr_backward_det_bytes(int64_t capacity, int32_t F) { return det_slot_bytes(capacity) + det_fslot_bytes(capacity, F); }
size_t sr_image_bytes(int32_t width, int32_t height) { return image_layout(width, height).total; }
size_t sr_binning_bytes(int64_t capacity, int32_t width, int32_t height) {
    return bin_layout(capacity, image_layout(width > 0 ? width : 0, height > 0 ? height : 0).tiles).total;
}
size_t sr_render_bytes(int32_t P, int64_t capacity, int32_t width, int32_t height) {
    const ImageLayout i = image_layout(width > 0 ? width : 0, height > 0 ? height : 0, true);
    return geom_layout(P, true).total + bin_layout(capacity, i.tiles, true).total + i.total;
}

int sr_debug_view(int32_t P, int32_t width, int32_t height, int64_t capacity, sr_debug_layout* out) {
    if (!out) return sr_fail(SR_EINVAL, "out is NULL");
    const GeomLayout g = geom_layout(P);
    const ImageLayout i = image_layout(width, height);
    const BinLayout b = bin_layout(capacity, i.tiles);
    out->surfel_rec = g.surfel_rec; out->depths = g.depths; out->tiles_touched = g.tiles_touched;
    out->point_offsets = g.point_offsets; out->clamped = g.clamped;
    out->keys[0] = b.keys[0]; out->keys[1] = b.keys[1]; out->values[0] = b.values[0]; out->values[1] = b.values[1];
    out->sort_ctl = b.sort_ctl; out->inst_rec = b.inst_rec; out->contrib = b.contrib;
    out->final_T = i.final_T; out->n_contrib = i.n_contrib; out->ranges = i.ranges; out->sub_last = i.tile_last;
    out->tile_order = i.tile_order;
    return 0;
}

namespace {
// Feature-channel arguments of sr_forward / sr_backward with F > 0: F in [1, SR_FEAT_MAX], background length 3 or 3+F,
// and the widest vector access (4, 2 or 1 floats) that every feature row / gradient row / frame stride allows.
int check_features(const sr_frame* f, int32_t F, int32_t bg_channels, const float* features, int64_t features_stride) {
    if (!f) return sr_fail(SR_EINVAL, "frame descriptor is NULL");
    if (F < 1 || F > SR_FEAT_MAX) return sr_fail(SR_EINVAL, "features: F must be in [1, %d], got %d", SR_FEAT_MAX, F);
    if (!features && f->P > 0) return sr_fail(SR_EINVAL, "features pointer is NULL");
    if (features_stride < 0) return sr_fail(SR_EINVAL, "features: frame stride must be >= 0");
    if (bg_channels != 3 && bg_channels != 3 + F)
        return sr_fail(SR_EINVAL, "background must have 3 or 3+F = %d channels, got %d", 3 + F, bg_channels);
    return 0;
}
// F = 0: the plain rasterizer (no feature pointer, 3-channel background, packed colour)
int check_no_features(const sr_frame* f, const float* features, int32_t bg_channels, int64_t color_stride) {
    if (features) return sr_fail(SR_EINVAL, "features: F must be in [1, %d], got 0", SR_FEAT_MAX);
    if (bg_channels != 3) return sr_fail(SR_EINVAL, "background must have 3 channels when F = 0, got %d", bg_channels);
    if (f && color_stride != 0 && color_stride != (int64_t)f->width * f->height * 3)
        return sr_fail(SR_EINVAL, "F = 0: the colour planes must be packed (frame stride 0 or 3*H*W)");
    return 0;
}
int feature_vec(int32_t F, std::initializer_list<uintptr_t> addrs) {
    for (int v : {4, 2}) {
        bool ok = F % v == 0;
        for (uintptr_t p : addrs) ok = ok && (p % (uintptr_t)(4 * v)) == 0;
        if (ok) return v;
    }
    return 1;
}
}  // namespace

static int forward_batch(const sr_frame* f, const sr_batch* b, const float* background, const float* means3D, const float* shs,
                         const float* colors_precomp, const float* opacities, const float* scales, const float* rotations,
                         const float* viewmatrix, const float* campos, float* out_color, int64_t color_stride,
                         float* out_others, int32_t* radii, void* geom_buffer, void* binning_buffer, void* image_buffer,
                         int64_t capacity, uint32_t* num_rendered_dev, uint32_t* num_rendered_host, void* stream_,
                         FeatArgs* ft, bool forward_only, const ContribArgs* contrib) {
    if (int rc = check_frame(f)) return rc;
    if (!b || b->frames < 1 || b->frames > 65535) return sr_fail(SR_EINVAL, "batch descriptor: frames must be in [1, 65535]");
    cudaStream_t stream = (cudaStream_t)stream_;
    const bool debug = f->debug != 0;
    const int P = f->P, M = b->frames;
    const size_t N = (size_t)f->width * f->height;
    if (!out_color || !out_others || !num_rendered_dev) return sr_fail(SR_EINVAL, "output pointer is NULL");
    if (!background || !viewmatrix || !campos) return sr_fail(SR_EINVAL, "camera / background pointer is NULL");
    const bool stats = contrib && !contrib->anchors;   // anchors gather none of the statistics
    if (stats && contrib->mask && contrib->mask_stride < (long long)N)
        return sr_fail(SR_EINVAL, "silhouette mask frame stride must be >= H*W bytes");
    if (stats && contrib->lift) {
        if (contrib->lift_C < 1 || contrib->lift_C > SR_LIFT_MAX_CHANNELS)
            return sr_fail(SR_EINVAL, "lift: C must be in [1, %d], got %d", SR_LIFT_MAX_CHANNELS, contrib->lift_C);
        if (ft) return sr_fail(SR_EINVAL, "lift: feature channels cannot be composited in the same call (F must be 0)");
        if (contrib->lift_stride / 4 < (long long)contrib->lift_C * (long long)N)
            return sr_fail(SR_EINVAL, "lift: values frame stride must be >= C*H*W floats");
        if (contrib->lift_scale_log2 < SR_LIFT_SCALE_MIN || contrib->lift_scale_log2 > SR_LIFT_SCALE_MAX)
            return sr_fail(SR_EINVAL, "lift: scale_log2 must be in [%d, %d], got %d", SR_LIFT_SCALE_MIN, SR_LIFT_SCALE_MAX,
                           contrib->lift_scale_log2);
    }
    if (ft) {
        if (color_stride < (int64_t)(3 * N)) return sr_fail(SR_EINVAL, "out_color frame stride must be >= 3*H*W");
        if (!ft->out) return sr_fail(SR_EINVAL, "out_features pointer is NULL");
        if (ft->out_stride < (long long)(ft->F * N) * 4) return sr_fail(SR_EINVAL, "out_features frame stride must be >= F*H*W");
    }
    if (P > 0) {   // every argument is checked before any device work
        if (!means3D || !opacities || !scales || !rotations || !radii) return sr_fail(SR_EINVAL, "surfel attribute pointer is NULL");
        if ((shs == nullptr) == (colors_precomp == nullptr))
            return sr_fail(SR_EINVAL, "provide exactly one of shs / colors_precomp");
        if (shs && f->sh_coeffs == 0) return sr_fail(SR_EINVAL, "shs given but sh_coeffs == 0");
        if (forward_only) {
            if (!geom_buffer) return sr_fail(SR_EINVAL, "arena is NULL");
            if ((uintptr_t)geom_buffer & 15) return sr_fail(SR_EINVAL, "arena must be 16-byte aligned");
        } else if (!geom_buffer || !binning_buffer || !image_buffer) {
            return sr_fail(SR_EINVAL, "scratch buffer is NULL");
        }
        if (capacity <= 0 || capacity >= (1ll << 30)) return sr_fail(SR_EINVAL, "capacity must be in (0, 2^30)");
        if (stats) {
            if (!contrib->weight_q || !contrib->max_weight || !contrib->pixels)
                return sr_fail(SR_EINVAL, "contribution statistics pointer is NULL");
            if (((uintptr_t)contrib->weight_q & 7) || ((uintptr_t)contrib->pixels & 7) || ((uintptr_t)contrib->max_weight & 3))
                return sr_fail(SR_EINVAL, "contribution statistics: weight_q / pixels must be 8-byte aligned, max_weight 4-byte aligned");
            if (contrib->mask) {
                if (!contrib->weight_bg_q || !contrib->pixels_bg)
                    return sr_fail(SR_EINVAL, "silhouette statistics pointer is NULL");
                if (((uintptr_t)contrib->weight_bg_q & 7) || ((uintptr_t)contrib->pixels_bg & 7))
                    return sr_fail(SR_EINVAL, "silhouette statistics: weight_bg_q / pixels_bg must be 8-byte aligned");
            }
            if (contrib->lift) {
                if (!contrib->lift_values || !contrib->lift_sums || !contrib->lift_saturated)
                    return sr_fail(SR_EINVAL, "lift: values / sums / saturated pointer is NULL");
                if ((uintptr_t)contrib->lift_values & 3)
                    return sr_fail(SR_EINVAL, "lift: values must be 4-byte aligned");
                if (((uintptr_t)contrib->lift_sums & 7) || ((uintptr_t)contrib->lift_saturated & 7))
                    return sr_fail(SR_EINVAL, "lift: sums / saturated must be 8-byte aligned");
            }
        }
        // 128-bit / 64-bit vector loads: rotations as float4, scales as float2, SH rows as float4 when 3M % 4 == 0
        if (((uintptr_t)rotations & 15) || ((uintptr_t)scales & 7) || (shs && ((uintptr_t)shs & 15)) ||
            ((b->rotations * 4) & 15) || ((b->scales * 4) & 7) || ((b->shs * 4) & 15))
            return sr_fail(SR_EINVAL, "rotations / shs must be 16-byte aligned and scales 8-byte aligned (per frame)");
    }
    CK(cudaMemsetAsync(num_rendered_dev, 0, (size_t)M * 2 * sizeof(uint32_t), stream), "memset(num_rendered)");
    if (P == 0) {
        // rasterize_points.cu:106 -- P == 0 short-circuits to zero-filled outputs
        if (ft) {
            CK(sr_memset_frames(out_color, (size_t)color_stride * 4, 3 * N * sizeof(float), M, stream), "memset(out_color)");
            CK(sr_memset_frames(ft->out, (size_t)ft->out_stride, (size_t)ft->F * N * sizeof(float), M, stream), "memset(out_features)");
        } else {
            CK(cudaMemsetAsync(out_color, 0, (size_t)M * 3 * N * sizeof(float), stream), "memset(out_color)");
        }
        CK(cudaMemsetAsync(out_others, 0, (size_t)M * 8 * N * sizeof(float), stream), "memset(out_others)");
        if (contrib && contrib->anchors) {
            // every slot empty: id -1 (all bits set), w 0, uv (0, 0)
            const size_t K = (size_t)contrib->anchor_K, pitch = (size_t)contrib->anchor_stride * 4;
            CK(cudaMemset2DAsync(contrib->anchor_ids, pitch, 0xff, K * N * 4, (size_t)M, stream), "memset(anchor_ids)");
            CK(cudaMemset2DAsync(contrib->anchor_w, pitch, 0, K * N * 4, (size_t)M, stream), "memset(anchor_weights)");
            CK(cudaMemset2DAsync(contrib->anchor_uv, 2 * pitch, 0, 2 * K * N * 4, (size_t)M, stream), "memset(anchor_uv)");
        }
        if (num_rendered_host)
            CK(cudaMemcpyAsync(num_rendered_host, num_rendered_dev, (size_t)M * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream), "copy(num_rendered)");
        return 0;
    }

    FwdArgs a{};
    a.cam = make_cam(f, viewmatrix, campos, background);
    if (!shs) a.cam.M = 0;
    a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.opacities = opacities;
    a.scales = scales; a.rotations = rotations;
    a.out_color = out_color; a.out_others = out_others; a.radii = radii;
    a.gl = geom_layout(P, forward_only); a.il = image_layout(f->width, f->height, forward_only);
    a.bl = bin_layout(capacity, a.il.tiles, forward_only);
    a.geom = (char*)geom_buffer; a.bin = (char*)binning_buffer; a.img = (char*)image_buffer;
    if (forward_only) { a.bin = a.geom + a.gl.total; a.img = a.bin + a.bl.total; }   // frame m's arena: [geom | bin | img]
    a.num_rendered_dev = num_rendered_dev;
    a.prefiltered = f->prefiltered;
    a.key_bits = 32 + (int)sr_higher_msb((uint32_t)a.il.tiles);
    a.stream = stream; a.debug = debug;
    a.forward_only = forward_only; a.feat = ft; a.contrib = contrib;
    ContribArgs anchors{};
    if (contrib && contrib->anchors) {   // the kernel reads each frame's status word to skip an overflowed frame
        anchors = *contrib;
        anchors.anchor_status = num_rendered_dev + 1;
        a.contrib = &anchors;
    }
    FrameStrides& fs = a.fs;
    fs.frames = M;
    fs.geom = (long long)a.gl.total; fs.bin = (long long)a.bl.total; fs.img = (long long)a.il.total; fs.nr = 2 * sizeof(uint32_t);
    if (forward_only) fs.geom = fs.bin = fs.img = (long long)(a.gl.total + a.bl.total + a.il.total);
    fs.means3D = b->means3D * 4; fs.shs = b->shs * 4; fs.colors = b->colors_precomp * 4; fs.opac = b->opacities * 4;
    fs.scales = b->scales * 4; fs.rots = b->rotations * 4; fs.vm = 16 * sizeof(float); fs.campos = 3 * sizeof(float);
    fs.out_color = (long long)(3 * N * sizeof(float)); fs.out_others = (long long)(8 * N * sizeof(float));
    if (ft) fs.out_color = (long long)color_stride * 4;
    fs.radii = (long long)P * sizeof(int32_t);

    // per frame: tile state (ranges .. end of the image buffer); sort control words + digit histograms + look-back status
    CK(sr_memset_frames(a.img + a.il.ranges, (size_t)fs.img, a.il.total - a.il.ranges, M, stream), "memset(tile state)");
    CK(sr_memset_frames(a.bin + a.bl.sort_ctl, (size_t)fs.bin, a.bl.total - a.bl.sort_ctl, M, stream), "memset(sort state)");
    CK(launch_preprocess_fwd(a), "preprocess_fwd"); DBG("preprocess_fwd");
    CK(launch_scan_emit(a), "scan/emit_keys"); DBG("scan/emit_keys");
    CK(launch_sort(a), "sort"); DBG("sort");
    CK(launch_ranges_gather(a), "ranges_gather"); DBG("ranges_gather");
    CK(launch_tile_order(a), "tile_order"); DBG("tile_order");
    if (forward_only) {
        // one walk: colour, allmap and the feature channels; SURFEL_COMPOSITE_FWD is not consulted
        CK(launch_composite_fwd(a), "composite_render"); DBG("composite_render");
    } else {
        if (sr_composite_tile_fwd()) { CK(launch_composite_tile_fwd(a), "composite_tile_fwd"); }
        else { CK(launch_composite_fwd(a), "composite_fwd"); }
        DBG("composite_fwd");
        if (ft) { CK(launch_feature_fwd(a, *ft), "feature_fwd"); DBG("feature_fwd"); }
    }
    if (num_rendered_host)
        CK(cudaMemcpyAsync(num_rendered_host, num_rendered_dev, (size_t)M * 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, stream), "copy(num_rendered)");
    return 0;
}

namespace {
// sr_forward, sr_render_forward and sr_render_forward_contrib: the feature arguments, then forward_batch
int forward_entry(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels, const float* means3D,
                  const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                  const float* rotations, const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
                  const float* campos, float* out_color, int64_t out_color_stride, float* out_features,
                  int64_t out_features_stride, float* out_others, int32_t* radii, void* geom_buffer, void* binning_buffer,
                  void* image_buffer, int64_t capacity, uint32_t* num_rendered_dev, uint32_t* num_rendered_host,
                  void* stream_, bool forward_only, const ContribArgs* contrib = nullptr) {
    if (F == 0) {
        if (int rc = check_no_features(f, features, bg_channels, out_color_stride)) return rc;
        return forward_batch(f, b, background, means3D, shs, colors_precomp, opacities, scales, rotations, viewmatrix, campos,
                             out_color, 0, out_others, radii, geom_buffer, binning_buffer, image_buffer, capacity,
                             num_rendered_dev, num_rendered_host, stream_, nullptr, forward_only, contrib);
    }
    if (int rc = check_features(f, F, bg_channels, features, features_stride)) return rc;
    FeatArgs ft{};
    ft.F = F;
    ft.vec = feature_vec(F, {(uintptr_t)features, (uintptr_t)(features_stride * 4)});
    ft.feat = features; ft.feat_stride = features_stride * 4;
    ft.bg = (bg_channels == 3 + F && background) ? background + 3 : nullptr;
    ft.out = out_features; ft.out_stride = out_features_stride * 4;
    return forward_batch(f, b, background, means3D, shs, colors_precomp, opacities, scales, rotations, viewmatrix, campos,
                         out_color, out_color_stride, out_others, radii, geom_buffer, binning_buffer, image_buffer, capacity,
                         num_rendered_dev, num_rendered_host, stream_, &ft, forward_only, contrib);
}
}  // namespace

int sr_forward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels, const float* means3D,
               const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
               const float* rotations, const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
               const float* projmatrix, const float* campos, float* out_color, int64_t out_color_stride,
               float* out_features, int64_t out_features_stride, float* out_others, int32_t* radii, void* geom_buffer,
               void* binning_buffer, void* image_buffer, int64_t capacity, uint32_t* num_rendered_dev,
               uint32_t* num_rendered_host, void* stream_) {
    (void)projmatrix;   // only feeds dead code in the reference (auxiliary.h:170-172)
    return forward_entry(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations, features, F,
                         features_stride, viewmatrix, campos, out_color, out_color_stride, out_features, out_features_stride,
                         out_others, radii, geom_buffer, binning_buffer, image_buffer, capacity, num_rendered_dev,
                         num_rendered_host, stream_, false);
}

int sr_render_forward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels, const float* means3D,
                      const float* shs, const float* colors_precomp, const float* opacities, const float* scales,
                      const float* rotations, const float* features, int32_t F, int64_t features_stride,
                      const float* viewmatrix, const float* projmatrix, const float* campos, float* out_color,
                      int64_t out_color_stride, float* out_features, int64_t out_features_stride, float* out_others,
                      int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev, uint32_t* num_rendered_host,
                      void* stream_) {
    (void)projmatrix;
    return forward_entry(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations, features, F,
                         features_stride, viewmatrix, campos, out_color, out_color_stride, out_features, out_features_stride,
                         out_others, radii, arena, nullptr, nullptr, capacity, num_rendered_dev, num_rendered_host, stream_,
                         true);
}

// sr_render_forward_contrib_masked and sr_render_forward_lift: the statistics' arguments, then forward_entry
static int render_forward_stats(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                                const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                                const float* scales, const float* rotations, const float* features, int32_t F,
                                int64_t features_stride, const float* viewmatrix, const float* campos, float* out_color,
                                int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                                float* out_others, int32_t* radii, void* arena, int64_t capacity,
                                uint32_t* num_rendered_dev, uint32_t* num_rendered_host, const sr_contrib* contrib,
                                const sr_contrib_mask* mask, const sr_lift* lift, void* stream_) {
    const bool masked = mask && mask->mask;
    if (masked && !contrib) return sr_fail(SR_EINVAL, "a silhouette mask needs the contribution statistics (contrib is NULL)");
    if (lift && !contrib) return sr_fail(SR_EINVAL, "a lift needs the contribution statistics (contrib is NULL)");
    ContribArgs cs{};
    if (lift) {
        cs.lift = true;
        cs.lift_C = lift->C;
        cs.lift_values = lift->values;
        cs.lift_stride = lift->values_stride * 4;
        cs.lift_scale_log2 = lift->scale_log2;
        cs.lift_scale = ldexpf(1.0f, lift->scale_log2);
        cs.lift_sums = reinterpret_cast<long long*>(lift->sums);
        cs.lift_saturated = reinterpret_cast<unsigned long long*>(lift->saturated);
    }
    if (contrib) {
        cs.weight_q = reinterpret_cast<unsigned long long*>(contrib->weight_q);
        cs.max_weight = contrib->max_weight;
        cs.pixels = reinterpret_cast<unsigned long long*>(contrib->pixels);
    }
    if (masked) {
        cs.mask = mask->mask;
        cs.mask_stride = mask->mask_stride;
        cs.weight_bg_q = reinterpret_cast<unsigned long long*>(mask->weight_bg_q);
        cs.pixels_bg = reinterpret_cast<unsigned long long*>(mask->pixels_bg);
    }
    return forward_entry(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations, features, F,
                         features_stride, viewmatrix, campos, out_color, out_color_stride, out_features, out_features_stride,
                         out_others, radii, arena, nullptr, nullptr, capacity, num_rendered_dev, num_rendered_host, stream_,
                         true, contrib ? &cs : nullptr);
}

int sr_render_forward_contrib(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                              const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                              const float* scales, const float* rotations, const float* features, int32_t F,
                              int64_t features_stride, const float* viewmatrix, const float* projmatrix, const float* campos,
                              float* out_color, int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                              float* out_others, int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev,
                              uint32_t* num_rendered_host, const sr_contrib* contrib, void* stream_) {
    return sr_render_forward_contrib_masked(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales,
                                            rotations, features, F, features_stride, viewmatrix, projmatrix, campos,
                                            out_color, out_color_stride, out_features, out_features_stride, out_others,
                                            radii, arena, capacity, num_rendered_dev, num_rendered_host, contrib, nullptr,
                                            stream_);
}

int sr_render_forward_contrib_masked(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                                     const float* means3D, const float* shs, const float* colors_precomp,
                                     const float* opacities, const float* scales, const float* rotations,
                                     const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
                                     const float* projmatrix, const float* campos, float* out_color,
                                     int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                                     float* out_others, int32_t* radii, void* arena, int64_t capacity,
                                     uint32_t* num_rendered_dev, uint32_t* num_rendered_host, const sr_contrib* contrib,
                                     const sr_contrib_mask* mask, void* stream_) {
    (void)projmatrix;
    return render_forward_stats(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations,
                                features, F, features_stride, viewmatrix, campos, out_color, out_color_stride, out_features,
                                out_features_stride, out_others, radii, arena, capacity, num_rendered_dev, num_rendered_host,
                                contrib, mask, nullptr, stream_);
}

int sr_render_forward_lift(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                           const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                           const float* scales, const float* rotations, const float* features, int32_t F,
                           int64_t features_stride, const float* viewmatrix, const float* projmatrix, const float* campos,
                           float* out_color, int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                           float* out_others, int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev,
                           uint32_t* num_rendered_host, const sr_contrib* contrib, const sr_lift* lift, void* stream_) {
    (void)projmatrix;
    return render_forward_stats(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations,
                                features, F, features_stride, viewmatrix, campos, out_color, out_color_stride, out_features,
                                out_features_stride, out_others, radii, arena, capacity, num_rendered_dev, num_rendered_host,
                                contrib, nullptr, lift, stream_);
}

int sr_render_forward_anchors(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                              const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                              const float* scales, const float* rotations, const float* features, int32_t F,
                              int64_t features_stride, const float* viewmatrix, const float* projmatrix, const float* campos,
                              float* out_color, int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                              float* out_others, int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev,
                              uint32_t* num_rendered_host, const sr_anchors* anchors, void* stream_) {
    (void)projmatrix;
    if (!anchors) return sr_fail(SR_EINVAL, "anchors is NULL");
    const int K = anchors->K;
    if (K != 1 && K != 2 && K != 4 && K != 8) return sr_fail(SR_EINVAL, "anchors: K must be 1, 2, 4 or 8, got %d", K);
    if (F != 0) return sr_fail(SR_EINVAL, "anchors: feature channels cannot be composited in the same call (F must be 0)");
    if (f && f->width > 0 && f->height > 0 && anchors->stride < (int64_t)K * f->width * f->height)
        return sr_fail(SR_EINVAL, "anchors: frame stride must be >= K*H*W elements");
    if (!anchors->ids || !anchors->weights || !anchors->uv)
        return sr_fail(SR_EINVAL, "anchors: ids / weights / uv pointer is NULL");
    if (((uintptr_t)anchors->ids & 3) || ((uintptr_t)anchors->weights & 3) || ((uintptr_t)anchors->uv & 3))
        return sr_fail(SR_EINVAL, "anchors: ids / weights / uv must be 4-byte aligned");
    ContribArgs cs{};
    cs.anchors = true;
    cs.anchor_K = K;
    cs.anchor_stride = anchors->stride;
    cs.anchor_ids = anchors->ids;
    cs.anchor_w = anchors->weights;
    cs.anchor_uv = anchors->uv;
    return forward_entry(f, b, background, bg_channels, means3D, shs, colors_precomp, opacities, scales, rotations, features, F,
                         features_stride, viewmatrix, campos, out_color, out_color_stride, out_features, out_features_stride,
                         out_others, radii, arena, nullptr, nullptr, capacity, num_rendered_dev, num_rendered_host, stream_,
                         true, &cs);
}

static int backward_batch(const sr_frame* f, const sr_batch* b, const float* background, const float* means3D, const float* shs,
                          const float* colors_precomp, const float* scales, const float* rotations, const float* viewmatrix,
                          const float* campos, const int32_t* radii, const float* dL_dout_color, int64_t dcolor_stride,
                          const float* dL_dout_others, const float* grad_scale, void* geom_buffer, void* binning_buffer,
                          void* image_buffer, int64_t capacity, float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity,
                          float* dL_dmeans3D, float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                          void* stream_, FeatArgs* ft) {
    if (int rc = check_frame(f)) return rc;
    if (!b || b->frames < 1 || b->frames > 65535) return sr_fail(SR_EINVAL, "batch descriptor: frames must be in [1, 65535]");
    cudaStream_t stream = (cudaStream_t)stream_;
    const bool debug = f->debug != 0;
    if (f->P == 0) return 0;   // rasterize_points.cu:204
    if (!background || !means3D || !scales || !rotations || !viewmatrix || !campos || !radii || !dL_dout_color ||
        !dL_dout_others || !geom_buffer || !binning_buffer || !image_buffer)
        return sr_fail(SR_EINVAL, "input pointer is NULL");
    if (!dL_dmeans2D || !dL_dcolors || !dL_dopacity || !dL_dmeans3D || !dL_dscales || !dL_drotations)
        return sr_fail(SR_EINVAL, "gradient output pointer is NULL");
    if (!dL_dtransMat && b->frames == 1 && !(b->flags & SR_BATCH_SUM_SHARED)) return sr_fail(SR_EINVAL, "dL_dtransMat is NULL");
    if (shs && !dL_dsh) return sr_fail(SR_EINVAL, "dL_dsh is NULL");
    if (capacity <= 0) return sr_fail(SR_EINVAL, "capacity must be positive");
    // SR_BATCH_DETERMINISTIC: b is the batch member of an sr_batch_det whose scratch holds M frames' slots
    const bool det = (b->flags & SR_BATCH_DETERMINISTIC) != 0;
    const sr_batch_det* bd = reinterpret_cast<const sr_batch_det*>(b);
    if (det) {
        const size_t need = sr_backward_det_bytes(capacity, ft ? ft->F : 0) * (size_t)b->frames;
        if (!bd->scratch) return sr_fail(SR_EINVAL, "SR_BATCH_DETERMINISTIC is set but the scratch pointer is NULL");
        if (bd->scratch_bytes < 0 || (size_t)bd->scratch_bytes < need)
            return sr_fail(SR_EINVAL, "deterministic backward: scratch has %lld bytes, needs %zu (sr_backward_det_bytes x frames)",
                           (long long)bd->scratch_bytes, need);
        if ((uintptr_t)bd->scratch & 15) return sr_fail(SR_EINVAL, "deterministic backward: scratch must be 16-byte aligned");
    }
    if (ft) {
        const long long N = (long long)f->width * f->height;
        if (dcolor_stride < 3 * N) return sr_fail(SR_EINVAL, "dL_dout_color frame stride must be >= 3*H*W");
        if (!ft->dout || !ft->dfeat) return sr_fail(SR_EINVAL, "dL_dout_features / dL_dfeatures pointer is NULL");
        if (ft->dout_stride < ft->F * N * 4) return sr_fail(SR_EINVAL, "dL_dout_features frame stride must be >= F*H*W");
    }
    if (((uintptr_t)rotations & 15) || ((uintptr_t)scales & 7) || (shs && ((uintptr_t)shs & 15)) ||
        ((uintptr_t)dL_drotations & 15) || ((uintptr_t)dL_dscales & 7) || (dL_dsh && ((uintptr_t)dL_dsh & 15)) ||
        ((b->rotations * 4) & 15) || ((b->scales * 4) & 7) || ((b->shs * 4) & 15))
        return sr_fail(SR_EINVAL, "rotations / shs (and their gradients) must be 16-byte aligned, scales 8-byte aligned");

    const int P = f->P, M = b->frames;
    const size_t N = (size_t)f->width * f->height;
    BwdArgs a{};
    a.cam = make_cam(f, viewmatrix, campos, background);
    if (!shs) a.cam.M = 0;
    a.grad_scale = grad_scale;
    a.means3D = means3D; a.shs = shs; a.colors_precomp = colors_precomp; a.scales = scales; a.rotations = rotations;
    a.radii = radii; a.dL_dcolor = dL_dout_color; a.dL_dothers = dL_dout_others;
    a.geom = (char*)geom_buffer; a.bin = (char*)binning_buffer; a.img = (char*)image_buffer;
    a.gl = geom_layout(P); a.il = image_layout(f->width, f->height); a.bl = bin_layout(capacity, a.il.tiles);
    a.dL_dmeans2D = dL_dmeans2D; a.dL_dcolors = dL_dcolors; a.dL_dopacity = dL_dopacity; a.dL_dmeans3D = dL_dmeans3D;
    a.dL_dtransMat = dL_dtransMat; a.dL_dsh = dL_dsh; a.dL_dscales = dL_dscales; a.dL_drotations = dL_drotations;
    a.stream = stream; a.debug = debug;
    FrameStrides& fs = a.fs;
    fs.frames = M;
    fs.geom = (long long)a.gl.total; fs.bin = (long long)a.bl.total; fs.img = (long long)a.il.total; fs.nr = 2 * sizeof(uint32_t);
    fs.means3D = b->means3D * 4; fs.shs = b->shs * 4; fs.colors = b->colors_precomp * 4; fs.opac = b->opacities * 4;
    fs.scales = b->scales * 4; fs.rots = b->rotations * 4; fs.vm = 16 * sizeof(float); fs.campos = 3 * sizeof(float);
    fs.radii = (long long)P * sizeof(int32_t);
    fs.dcolor = (long long)(3 * N * sizeof(float)); fs.dothers = (long long)(8 * N * sizeof(float));
    if (ft) fs.dcolor = (long long)dcolor_stride * 4;
    // gradients are written per frame, (M, P, .) -- or, with SR_BATCH_SUM_SHARED, once as the sum over frames, (P, .), for
    // the inputs the frames share (surfel_bwd.cu accumulates them inside the kernel; stride 0 selects that)
    const long long Pl = P;
    const bool sum = (b->flags & SR_BATCH_SUM_SHARED) != 0 && M > 1;
    fs.g_m2d = Pl * 3 * 4; fs.g_tm = Pl * 9 * 4;
    fs.g_col = (sum && b->colors_precomp == 0) ? 0 : Pl * 3 * 4;
    fs.g_opac = (sum && b->opacities == 0) ? 0 : Pl * 4;
    fs.g_m3d = (sum && b->means3D == 0) ? 0 : Pl * 3 * 4;
    fs.g_sh = (sum && b->shs == 0) ? 0 : Pl * a.cam.M * 3 * 4;
    fs.g_scales = (sum && b->scales == 0) ? 0 : Pl * 2 * 4;
    fs.g_rots = (sum && b->rotations == 0) ? 0 : Pl * 4 * 4;
    if (ft) {
        // dL/dfeatures: (P,F) summed over the frames when the features are shared and SR_BATCH_SUM_SHARED is set,
        // else (M,P,F); zeroed here, the feature pass adds into it
        ft->dfeat_stride = (sum && ft->feat_stride == 0) ? 0 : Pl * ft->F * 4;
        const size_t rows = ft->dfeat_stride == 0 ? 1 : (size_t)M;
        if (!det) CK(cudaMemsetAsync(ft->dfeat, 0, rows * (size_t)Pl * ft->F * sizeof(float), stream), "memset(dL_dfeatures)");
    }
    if (det) {
        // per frame: [slots of capacity instances | feature slots]; det_gather writes the accumulator and dL/dfeatures whole
        DetArgs d{};
        const size_t sb = det_slot_bytes(capacity), per = sr_backward_det_bytes(capacity, ft ? ft->F : 0);
        d.slots = (float*)bd->scratch; d.slots_stride = (long long)per;
        d.fslots = ft ? (float*)((char*)bd->scratch + sb) : nullptr; d.fslots_stride = (long long)per;
        d.point_offsets = (const uint32_t*)(a.geom + a.gl.point_offsets); d.radii = radii; d.tiles_y = a.il.tiles_y;
        CK(launch_det_zero(a, d, ft ? ft->F : 0), "det_zero"); DBG("det_zero");
        CK(launch_composite_tile_bwd_det(a, d), "composite_bwd_det"); DBG("composite_bwd_det");
        if (ft) { CK(launch_feature_bwd_det(a, *ft, d), "feature_bwd_det"); DBG("feature_bwd_det"); }
        CK(launch_det_gather(a, d, ft), "det_gather"); DBG("det_gather");
        CK(launch_surfel_bwd(a), "surfel_bwd"); DBG("surfel_bwd");
        return 0;
    }
    CK(launch_composite_tile_bwd(a), "composite_bwd"); DBG("composite_bwd");
    // after composite_bwd (which zeroes the per-surfel accumulator), before surfel_bwd (which reads it)
    if (ft) { CK(launch_feature_bwd(a, *ft), "feature_bwd"); DBG("feature_bwd"); }
    CK(launch_surfel_bwd(a), "surfel_bwd"); DBG("surfel_bwd");
    return 0;
}

int sr_backward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels, const float* means3D,
                const float* shs, const float* colors_precomp, const float* scales, const float* rotations,
                const float* features, int32_t F, int64_t features_stride, const float* viewmatrix, const float* projmatrix,
                const float* campos, const int32_t* radii, const float* dL_dout_color, int64_t dL_dout_color_stride,
                const float* dL_dout_features, int64_t dL_dout_features_stride, const float* dL_dout_others,
                const float* grad_scale, const float* features_grad_scale, void* geom_buffer, void* binning_buffer,
                void* image_buffer, int64_t capacity, float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity,
                float* dL_dmeans3D, float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                float* dL_dfeatures, void* stream_) {
    (void)projmatrix;
    if (F == 0) {
        if (int rc = check_no_features(f, features, bg_channels, dL_dout_color_stride)) return rc;
        return backward_batch(f, b, background, means3D, shs, colors_precomp, scales, rotations, viewmatrix, campos, radii,
                              dL_dout_color, 0, dL_dout_others, grad_scale, geom_buffer, binning_buffer, image_buffer,
                              capacity, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh, dL_dscales,
                              dL_drotations, stream_, nullptr);
    }
    if (int rc = check_features(f, F, bg_channels, features, features_stride)) return rc;
    FeatArgs ft{};
    ft.F = F;
    ft.vec = feature_vec(F, {(uintptr_t)features, (uintptr_t)(features_stride * 4), (uintptr_t)dL_dfeatures});
    ft.feat = features; ft.feat_stride = features_stride * 4;
    ft.bg = (bg_channels == 3 + F && background) ? background + 3 : nullptr;
    ft.dout = dL_dout_features; ft.dout_stride = dL_dout_features_stride * 4;
    ft.grad_scale = features_grad_scale;
    ft.dfeat = dL_dfeatures;
    return backward_batch(f, b, background, means3D, shs, colors_precomp, scales, rotations, viewmatrix, campos, radii,
                          dL_dout_color, dL_dout_color_stride, dL_dout_others, grad_scale, geom_buffer, binning_buffer,
                          image_buffer, capacity, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh,
                          dL_dscales, dL_drotations, stream_, &ft);
}

int sr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    uint8_t* present, void* stream_) {
    (void)projmatrix;
    if (P < 0) return sr_fail(SR_EINVAL, "P must be >= 0");
    if (P == 0) return 0;
    if (!means3D || !viewmatrix || !present) return sr_fail(SR_EINVAL, "pointer is NULL");
    CK(launch_mark_visible(P, means3D, viewmatrix, present, (cudaStream_t)stream_), "mark_visible");
    return 0;
}

}  // extern "C"
