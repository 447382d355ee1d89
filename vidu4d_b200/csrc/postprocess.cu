// postprocess.cu -- fused post-processing of the rasterizer's 8-plane `allmap` (SURVEY.md section 8(f) row N1).
//
// Replaces ~35 small PyTorch kernels forward and ~60 backward per frame of the reference's render() glue:
//   gs/gaussian_renderer/__init__.py:121-162   alpha / normal rotation / nan_to_num'd median & expected depth /
//                                              surf_depth mix / surf_normal = depth_to_normal(...) * alpha.detach()
//   gs/utils/point_utils.py:9-37               depths_to_points, depth_to_normal (central differences, cross, normalise)
// One kernel forward, one backward, same values (fp32, same operation order as the torch expressions up to
// reassociation inside a dot product).  The backward is written as a GATHER (each pixel collects the stencil
// contributions of its four neighbours), so it has no atomics and is deterministic.
#include "post_common.cuh"
#include "../../include/surfel_render.h"

namespace {
using namespace post;

// sr_post_forward_frames: frame blockIdx.z of M, its camera from the optional (M,4) table, and the optional learnable
// background added into its colour planes.  FRAMES = false is sr_post_forward's one frame (Frames unused).
struct Frames {
    const float* cams;      // DEVICE (M,4) or nullptr
    const float* bkgd;      // DEVICE [3] or nullptr
    float* color;           // frame 0's colour planes (read and written only with bkgd)
    long long color_stride; // floats between frames
};
// frame f's camera: row f of the table (TABLE), else the shared tangents.  The two are separate instantiations so that
// the scalar one compiles to sr_post_forward's arithmetic, contraction for contraction.
template <bool TABLE>
__device__ __forceinline__ PostCam frame_cam(const Frames& fr, int f, const float* __restrict__ wvt, int W, int H, float tanx,
                                             float tany) {
    if constexpr (TABLE) {
        const float* r = fr.cams + 4 * (size_t)f;
        return load_cam(wvt, W, H, __ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3));
    }
    return load_cam(wvt, W, H, tanx, tany);
}

template <bool FRAMES, bool TABLE>
__global__ void __launch_bounds__(256)
post_fwd_kernel(int W, int H, float tanx, float tany, float depth_ratio, const float* __restrict__ allmap,
                const float* __restrict__ wvt, float* __restrict__ acc, float* __restrict__ rend_normal,
                float* __restrict__ rend_dist, float* __restrict__ depth_median, float* __restrict__ depth_expected,
                float* __restrict__ surf_depth, const Frames fr) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const size_t N = (size_t)W * H, p = (size_t)y * W + x;
    const int f = FRAMES ? (int)blockIdx.z : 0;
    if constexpr (FRAMES) {
        allmap += (size_t)f * 8 * N; wvt += (size_t)f * 16; acc += (size_t)f * N; rend_normal += (size_t)f * 3 * N;
        rend_dist += (size_t)f * N; depth_median += (size_t)f * N; depth_expected += (size_t)f * N; surf_depth += (size_t)f * N;
    }
    const PostCam c = frame_cam<TABLE>(fr, f, wvt, W, H, tanx, tany);
    const float a = allmap[N + p];
    if constexpr (FRAMES) {
        if (fr.bkgd) {   // deformable_gaussian.py:188-190: color[:3] + (1 - acc) * bkgd, each operation rounded
            float* col = fr.color + (size_t)f * fr.color_stride;
            const float om = __fadd_rn(1.0f, -a);
#pragma unroll
            for (int k = 0; k < 3; k++) col[k * N + p] = __fadd_rn(col[k * N + p], __fmul_rn(om, __ldg(fr.bkgd + k)));
        }
    }
    const float n0 = allmap[2 * N + p], n1 = allmap[3 * N + p], n2 = allmap[4 * N + p];
    acc[p] = a;
    rend_normal[p] = c.R[0] * n0 + c.R[1] * n1 + c.R[2] * n2;
    rend_normal[N + p] = c.R[3] * n0 + c.R[4] * n1 + c.R[5] * n2;
    rend_normal[2 * N + p] = c.R[6] * n0 + c.R[7] * n1 + c.R[8] * n2;
    rend_dist[p] = allmap[6 * N + p];
    const float med = nan_to_num00(allmap[5 * N + p]);
    const float ex = nan_to_num00(allmap[p] / a);
    depth_median[p] = med;
    depth_expected[p] = ex;
    surf_depth[p] = ex * (1.f - depth_ratio) + depth_ratio * med;
}

// surf_normal needs the neighbours' surf_depth: second (tiny) kernel
template <bool FRAMES, bool TABLE>
__global__ void __launch_bounds__(256)
post_normal_kernel(int W, int H, float tanx, float tany, const float* __restrict__ allmap, const float* __restrict__ wvt,
                   const float* __restrict__ surf_depth, float* __restrict__ surf_normal, const Frames fr) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const size_t N = (size_t)W * H, p = (size_t)y * W + x;
    const int f = FRAMES ? (int)blockIdx.z : 0;
    if constexpr (FRAMES) {
        allmap += (size_t)f * 8 * N; wvt += (size_t)f * 16; surf_depth += (size_t)f * N; surf_normal += (size_t)f * 3 * N;
    }
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    if (x >= 1 && x < W - 1 && y >= 1 && y < H - 1) {
        const PostCam c = frame_cam<TABLE>(fr, f, wvt, W, H, tanx, tany);
        float ax, ay, az, bx, by, bz, ex, ey, ez, fx, fy, fz;
        ray_dir(c, x, y + 1, ax, ay, az); ray_dir(c, x, y - 1, bx, by, bz);
        ray_dir(c, x + 1, y, ex, ey, ez); ray_dir(c, x - 1, y, fx, fy, fz);
        const float dD = surf_depth[p + W], dU = surf_depth[p - W], dR = surf_depth[p + 1], dL = surf_depth[p - 1];
        // dx = points[y+1] - points[y-1] (rows), dy = points[x+1] - points[x-1] (columns); ray origins cancel
        const float dxx = dD * ax - dU * bx, dxy = dD * ay - dU * by, dxz = dD * az - dU * bz;
        const float dyx = dR * ex - dL * fx, dyy = dR * ey - dL * fy, dyz = dR * ez - dL * fz;
        const float nx = dxy * dyz - dxz * dyy, ny = dxz * dyx - dxx * dyz, nz = dxx * dyy - dxy * dyx;
        const float inv = 1.0f / fmaxf(sqrtf(nx * nx + ny * ny + nz * nz), 1e-12f);   // F.normalize eps
        const float a = allmap[N + p];
        o0 = nx * inv * a; o1 = ny * inv * a; o2 = nz * inv * a;
    }
    surf_normal[p] = o0; surf_normal[N + p] = o1; surf_normal[2 * N + p] = o2;
}

// d(normalize(cross(dx,dy)) * a)/d(dx,dy) applied to g, for the stencil centred at (x,y); returns g_dx, g_dy
__device__ __forceinline__ bool stencil_vjp(const PostCam& c, int W, int H, int x, int y, const float* __restrict__ surf_depth,
                                            const float* __restrict__ allmap, const float* __restrict__ g_sn, size_t N,
                                            float* gdx, float* gdy) {
    if (!(x >= 1 && x < W - 1 && y >= 1 && y < H - 1)) return false;
    const size_t p = (size_t)y * W + x;
    float ax, ay, az, bx, by, bz, ex, ey, ez, fx, fy, fz;
    ray_dir(c, x, y + 1, ax, ay, az); ray_dir(c, x, y - 1, bx, by, bz);
    ray_dir(c, x + 1, y, ex, ey, ez); ray_dir(c, x - 1, y, fx, fy, fz);
    const float dD = surf_depth[p + W], dU = surf_depth[p - W], dR = surf_depth[p + 1], dL = surf_depth[p - 1];
    const float dxx = dD * ax - dU * bx, dxy = dD * ay - dU * by, dxz = dD * az - dU * bz;
    const float dyx = dR * ex - dL * fx, dyy = dR * ey - dL * fy, dyz = dR * ez - dL * fz;
    const float nx = dxy * dyz - dxz * dyy, ny = dxz * dyx - dxx * dyz, nz = dxx * dyy - dxy * dyx;
    const float len = sqrtf(nx * nx + ny * ny + nz * nz);
    const float a = allmap[N + p];                       // alpha is detached in the reference: a constant here
    const float g0 = g_sn[p] * a, g1 = g_sn[N + p] * a, g2 = g_sn[2 * N + p] * a;
    float gnx, gny, gnz;                                 // gradient w.r.t. the un-normalised cross product
    if (len > 1e-12f) {
        const float inv = 1.0f / len;
        const float ux = nx * inv, uy = ny * inv, uz = nz * inv;
        const float d = ux * g0 + uy * g1 + uz * g2;
        gnx = (g0 - ux * d) * inv; gny = (g1 - uy * d) * inv; gnz = (g2 - uz * d) * inv;
    } else {                                             // v / eps branch of F.normalize
        gnx = g0 * 1e12f; gny = g1 * 1e12f; gnz = g2 * 1e12f;
    }
    // n = dx x dy :  g_dx = dy x g_n ,  g_dy = g_n x dx
    gdx[0] = dyy * gnz - dyz * gny; gdx[1] = dyz * gnx - dyx * gnz; gdx[2] = dyx * gny - dyy * gnx;
    gdy[0] = gny * dxz - gnz * dxy; gdy[1] = gnz * dxx - gnx * dxz; gdy[2] = gnx * dxy - gny * dxx;
    return true;
}

__global__ void __launch_bounds__(256)
post_bwd_kernel(int W, int H, float tanx, float tany, float depth_ratio, const float* __restrict__ allmap,
                const float* __restrict__ wvt, const float* __restrict__ surf_depth,
                const float* __restrict__ g_acc, const float* __restrict__ g_rn, const float* __restrict__ g_dist,
                const float* __restrict__ g_med, const float* __restrict__ g_exp, const float* __restrict__ g_sd,
                const float* __restrict__ g_sn, float* __restrict__ g_allmap) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (x >= W || y >= H) return;
    const size_t N = (size_t)W * H, p = (size_t)y * W + x;
    const PostCam c = load_cam(wvt, W, H, tanx, tany);
    // ---- gather the surf_normal stencil contributions landing on this pixel's depth
    float gp0 = 0.f, gp1 = 0.f, gp2 = 0.f, gdx[3], gdy[3];
    if (stencil_vjp(c, W, H, x, y - 1, surf_depth, allmap, g_sn, N, gdx, gdy)) { gp0 += gdx[0]; gp1 += gdx[1]; gp2 += gdx[2]; }  // we are its (y+1)
    if (stencil_vjp(c, W, H, x, y + 1, surf_depth, allmap, g_sn, N, gdx, gdy)) { gp0 -= gdx[0]; gp1 -= gdx[1]; gp2 -= gdx[2]; }  // we are its (y-1)
    if (stencil_vjp(c, W, H, x - 1, y, surf_depth, allmap, g_sn, N, gdx, gdy)) { gp0 += gdy[0]; gp1 += gdy[1]; gp2 += gdy[2]; }  // we are its (x+1)
    if (stencil_vjp(c, W, H, x + 1, y, surf_depth, allmap, g_sn, N, gdx, gdy)) { gp0 -= gdy[0]; gp1 -= gdy[1]; gp2 -= gdy[2]; }  // we are its (x-1)
    float rx, ry, rz;
    ray_dir(c, x, y, rx, ry, rz);
    const float gsd = g_sd[p] + gp0 * rx + gp1 * ry + gp2 * rz;     // point = depth * ray + origin
    // ---- surf_depth = expected (1-r) + r median
    const float a = allmap[N + p], d0 = allmap[p], m5 = allmap[5 * N + p];
    const float gex = g_exp[p] + gsd * (1.f - depth_ratio);
    const float gmed = g_med[p] + gsd * depth_ratio;
    const float q = d0 / a;
    const bool qfin = isfinite(q);                       // nan_to_num passes the gradient only where its input is finite
    g_allmap[p] = qfin ? gex / a : 0.f;
    g_allmap[N + p] = g_acc[p] + (qfin ? -gex * d0 / (a * a) : 0.f);
    // ---- rend_normal = W @ n  ->  g_n = W^T g
    const float r0 = g_rn[p], r1 = g_rn[N + p], r2 = g_rn[2 * N + p];
    g_allmap[2 * N + p] = c.R[0] * r0 + c.R[3] * r1 + c.R[6] * r2;
    g_allmap[3 * N + p] = c.R[1] * r0 + c.R[4] * r1 + c.R[7] * r2;
    g_allmap[4 * N + p] = c.R[2] * r0 + c.R[5] * r1 + c.R[8] * r2;
    g_allmap[5 * N + p] = isfinite(m5) ? gmed : 0.f;
    g_allmap[6 * N + p] = g_dist[p];
    g_allmap[7 * N + p] = 0.f;
}

}  // namespace

extern "C" {

SR_API int sr_post_forward(int32_t W, int32_t H, float tanx, float tany, float depth_ratio, const float* allmap,
                           const float* world_view_transform, float* acc, float* rend_normal, float* rend_dist,
                           float* depth_median, float* depth_expected, float* surf_depth, float* surf_normal, void* stream_) {
    if (!allmap || !world_view_transform || !acc || !rend_normal || !rend_dist || !depth_median || !depth_expected || !surf_depth ||
        !surf_normal)
        return sr_fail(SR_EINVAL, "sr_post_forward: a required pointer is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    dim3 grid((W + 31) / 32, (H + 7) / 8);
    {
        ProfileScope ps("post_fwd", s);
        post_fwd_kernel<false, false><<<grid, 256, 0, s>>>(W, H, tanx, tany, depth_ratio, allmap, world_view_transform, acc,
                                                   rend_normal, rend_dist, depth_median, depth_expected, surf_depth, Frames{});
    }
    ProfileScope ps("post_normal", s);
    post_normal_kernel<false, false><<<grid, 256, 0, s>>>(W, H, tanx, tany, allmap, world_view_transform, surf_depth, surf_normal,
                                                  Frames{});
    return sr_launched(2, "sr_post_forward");
}

SR_API int sr_post_forward_frames(int32_t M, int32_t W, int32_t H, float tanx, float tany, const float* cameras,
                                  float depth_ratio, const float* allmap, const float* world_view_transform,
                                  const float* learnable_bkgd, float* color, int64_t color_stride, float* acc,
                                  float* rend_normal, float* rend_dist, float* depth_median, float* depth_expected,
                                  float* surf_depth, float* surf_normal, void* stream_) {
    if (M < 1 || M > 65535) return sr_fail(SR_EINVAL, "sr_post_forward_frames: M must be in [1, 65535], got %d", M);
    if (W <= 0 || H <= 0) return sr_fail(SR_EINVAL, "sr_post_forward_frames: image size must be positive");
    if (!allmap || !world_view_transform || !acc || !rend_normal || !rend_dist || !depth_median || !depth_expected || !surf_depth ||
        !surf_normal)
        return sr_fail(SR_EINVAL, "sr_post_forward_frames: a required pointer is NULL");
    if (learnable_bkgd && !color) return sr_fail(SR_EINVAL, "sr_post_forward_frames: learnable_bkgd is given but color is NULL");
    if (learnable_bkgd && color_stride < 3ll * W * H)
        return sr_fail(SR_EINVAL, "sr_post_forward_frames: color frame stride must be >= 3*H*W");
    cudaStream_t s = (cudaStream_t)stream_;
    const Frames fr{cameras, learnable_bkgd, color, (long long)color_stride};
    dim3 grid((W + 31) / 32, (H + 7) / 8, M);
    {
        ProfileScope ps("post_fwd_frames", s);
        auto k = cameras ? post_fwd_kernel<true, true> : post_fwd_kernel<true, false>;
        k<<<grid, 256, 0, s>>>(W, H, tanx, tany, depth_ratio, allmap, world_view_transform, acc, rend_normal, rend_dist,
                               depth_median, depth_expected, surf_depth, fr);
    }
    ProfileScope ps("post_normal_frames", s);
    auto k = cameras ? post_normal_kernel<true, true> : post_normal_kernel<true, false>;
    k<<<grid, 256, 0, s>>>(W, H, tanx, tany, allmap, world_view_transform, surf_depth, surf_normal, fr);
    return sr_launched(2, "sr_post_forward_frames");
}

SR_API int sr_post_backward(int32_t W, int32_t H, float tanx, float tany, float depth_ratio, const float* allmap,
                            const float* world_view_transform, const float* surf_depth, const float* g_acc,
                            const float* g_rend_normal, const float* g_rend_dist, const float* g_depth_median,
                            const float* g_depth_expected, const float* g_surf_depth, const float* g_surf_normal,
                            float* g_allmap, void* stream_) {
    if (!allmap || !world_view_transform || !surf_depth || !g_acc || !g_rend_normal || !g_rend_dist || !g_depth_median ||
        !g_depth_expected || !g_surf_depth || !g_surf_normal || !g_allmap)
        return sr_fail(SR_EINVAL, "sr_post_backward: a required pointer is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    dim3 grid((W + 31) / 32, (H + 7) / 8);
    ProfileScope ps("post_bwd", s);
    post_bwd_kernel<<<grid, 256, 0, s>>>(W, H, tanx, tany, depth_ratio, allmap, world_view_transform, surf_depth, g_acc,
                                        g_rend_normal, g_rend_dist, g_depth_median, g_depth_expected, g_surf_depth,
                                        g_surf_normal, g_allmap);
    return sr_launched(1, "sr_post_backward");
}

}  // extern "C"
