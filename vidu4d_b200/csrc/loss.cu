// loss.cu -- the Stage-3 image losses fused with the render() post-processing, forward AND backward in one pass
// (SURVEY.md section 8(f) row N1, second half).
//
// Replaces, per frame, ~35 + ~40 small PyTorch kernels forward and ~100 backward:
//   gs/gaussian_renderer/__init__.py:121-145   alpha / rotated normal / nan_to_num'd expected & median depth / surf_depth
//   gs/utils/point_utils.py:9-37               depth_to_normal (central differences, cross, normalise) * alpha.detach()
//   lab4d/nnutils/deformable_gaussian.py:188-190  render += (1 - acc) * learnable_bkgd           (optional)
//   lab4d/engine/model.py:674-692              masked L1 on rgb where vis2d > 0, mean over all elements
//   lab4d/engine/model.py:649-653              (acc - mask)^2 * mask_balance_wt, mean
//   lab4d/engine/model.py:817-842              lambda_n * mean(1 - <rend_normal, surf_normal>), lambda_d * mean(rend_dist)
//
// The losses are scalars whose gradient with respect to the rasterizer's outputs is analytic, so ONE kernel computes the
// four loss terms (block reduction + 4 atomics per block) and writes dL/dcolor and dL/dallmap directly; the rasterizer
// backward consumes them (times the upstream scalar, sr_backward's grad_scale).  The surf_normal stencil is
// handled as a gather: a block evaluates the stencils of its 32x8 tile plus a one-pixel ring once each into shared memory
// and every pixel picks up its four neighbours' results, so there are no atomics on image data and the result is
// deterministic.  Batched: blockIdx.z = frame.
#include "post_common.cuh"
#include "../../include/surfel_camera.h"

namespace {
using namespace post;

struct LossCfg {
    int W, H;
    const float* cams;             // DEVICE [M*4] per-frame (tan_x, tan_y, cx_off, cy_off) (surfel_camera.h), or nullptr
    float tanx, tany, depth_ratio; // tanx / tany: every frame's, when cams is nullptr
    float w_rgb, w_mask, lambda_normal, lambda_dist;
};

__global__ void __launch_bounds__(256)
loss_depth_kernel(const LossCfg g, const float* __restrict__ allmap, float* __restrict__ surf_depth) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    if (x >= g.W || y >= g.H) return;
    const size_t N = (size_t)g.W * g.H, p = (size_t)y * g.W + x;
    const float* am = allmap + (size_t)f * 8 * N;
    const float med = nan_to_num00(am[5 * N + p]);
    const float ex = nan_to_num00(am[p] / am[N + p]);
    surf_depth[(size_t)f * N + p] = ex * (1.f - g.depth_ratio) + g.depth_ratio * med;
}

// The depth_to_normal stencil centred at (X, Y) (point_utils.py:24-37), evaluated ONCE per pixel: its alpha-weighted unit
// normal `sn` (surf_normal of that pixel) and the gradient of  lambda_n * mean(1 - <rend_normal, surf_normal>)  with
// respect to its two difference vectors, gdx / gdy (alpha detached).  Everything is zero outside the image interior.
// Six divisions per evaluation (the pixel grid coordinates of the three columns and three rows the four rays use).
__device__ __forceinline__ void stencil_eval(const PostCam& c, const LossCfg& g, int X, int Y, const float* __restrict__ sd,
                                             const float* __restrict__ am, size_t N, float scale, float* sn, float* gdx,
                                             float* gdy) {
    sn[0] = sn[1] = sn[2] = 0.f;
    gdx[0] = gdx[1] = gdx[2] = 0.f;
    gdy[0] = gdy[1] = gdy[2] = 0.f;
    if (!(X >= 1 && X < g.W - 1 && Y >= 1 && Y < g.H - 1)) return;
    const size_t p = (size_t)Y * g.W + X;
    const float um = ((float)(X - 1) - c.cx) / c.fx, u0 = ((float)X - c.cx) / c.fx, up = ((float)(X + 1) - c.cx) / c.fx;
    const float vm = ((float)(Y - 1) - c.cy) / c.fy, v0 = ((float)Y - c.cy) / c.fy, vp = ((float)(Y + 1) - c.cy) / c.fy;
    // rays through (X, Y+1), (X, Y-1), (X+1, Y), (X-1, Y): A (u, v, 1)
    const float ax = c.A[0] * u0 + c.A[1] * vp + c.A[2], ay = c.A[3] * u0 + c.A[4] * vp + c.A[5], az = c.A[6] * u0 + c.A[7] * vp + c.A[8];
    const float bx = c.A[0] * u0 + c.A[1] * vm + c.A[2], by = c.A[3] * u0 + c.A[4] * vm + c.A[5], bz = c.A[6] * u0 + c.A[7] * vm + c.A[8];
    const float ex = c.A[0] * up + c.A[1] * v0 + c.A[2], ey = c.A[3] * up + c.A[4] * v0 + c.A[5], ez = c.A[6] * up + c.A[7] * v0 + c.A[8];
    const float fx = c.A[0] * um + c.A[1] * v0 + c.A[2], fy = c.A[3] * um + c.A[4] * v0 + c.A[5], fz = c.A[6] * um + c.A[7] * v0 + c.A[8];
    const float dD = sd[p + g.W], dU = sd[p - g.W], dR = sd[p + 1], dL = sd[p - 1];
    const float dx0 = dD * ax - dU * bx, dx1 = dD * ay - dU * by, dx2 = dD * az - dU * bz;
    const float dy0 = dR * ex - dL * fx, dy1 = dR * ey - dL * fy, dy2 = dR * ez - dL * fz;
    const float n0 = dx1 * dy2 - dx2 * dy1, n1 = dx2 * dy0 - dx0 * dy2, n2 = dx0 * dy1 - dx1 * dy0;
    const float len = sqrtf(n0 * n0 + n1 * n1 + n2 * n2);
    const float a = am[N + p];
    const float inv_s = a / fmaxf(len, 1e-12f);
    sn[0] = n0 * inv_s; sn[1] = n1 * inv_s; sn[2] = n2 * inv_s;
    // g_sn = scale * rend_normal (scale = -lambda_n / N), times alpha (the detached factor), back through F.normalize
    const float r0 = am[2 * N + p], r1 = am[3 * N + p], r2 = am[4 * N + p];
    const float s = scale * a;
    const float g0 = s * (c.R[0] * r0 + c.R[1] * r1 + c.R[2] * r2), g1 = s * (c.R[3] * r0 + c.R[4] * r1 + c.R[5] * r2),
                g2 = s * (c.R[6] * r0 + c.R[7] * r1 + c.R[8] * r2);
    float gn0, gn1, gn2;
    if (len > 1e-12f) {
        const float inv = 1.0f / len;
        const float w0 = n0 * inv, w1 = n1 * inv, w2 = n2 * inv;
        const float d = w0 * g0 + w1 * g1 + w2 * g2;
        gn0 = (g0 - w0 * d) * inv; gn1 = (g1 - w1 * d) * inv; gn2 = (g2 - w2 * d) * inv;
    } else {                                             // v / eps branch of F.normalize
        gn0 = g0 * 1e12f; gn1 = g1 * 1e12f; gn2 = g2 * 1e12f;
    }
    gdx[0] = dy1 * gn2 - dy2 * gn1; gdx[1] = dy2 * gn0 - dy0 * gn2; gdx[2] = dy0 * gn1 - dy1 * gn0;
    gdy[0] = gn1 * dx2 - gn2 * dx1; gdy[1] = gn2 * dx0 - gn0 * dx2; gdy[2] = gn0 * dx1 - gn1 * dx0;
}

__global__ void __launch_bounds__(256)
loss_grad_kernel(const LossCfg g, const float* __restrict__ color, const float* __restrict__ allmap,
                 const float* __restrict__ wvt, const float* __restrict__ target, const float* __restrict__ vis2d,
                 const float* __restrict__ mask_gt, const float* __restrict__ mask_wt, const float* __restrict__ bkgd,
                 const float* __restrict__ surf_depth, float* __restrict__ loss_terms, float* __restrict__ g_color,
                 float* __restrict__ g_allmap, float* __restrict__ g_bkgd) {
    const int lx = threadIdx.x & 31, ly = threadIdx.x >> 5;
    const int x = blockIdx.x * 32 + lx, y = blockIdx.y * 8 + ly, f = blockIdx.z;
    const int W = g.W, H = g.H;
    const size_t N = (size_t)W * H;
    const float invN = 1.0f / (float)N;
    const float* am = allmap + (size_t)f * 8 * N;
    const float* sd = surf_depth + (size_t)f * N;
    const float sN = g.lambda_normal * invN;
    // the stencil gradients of the 32x8 tile plus a one-pixel ring: every stencil is evaluated once (1.3 evaluations per
    // pixel) and its neighbours pick the result up from shared memory -- no atomics on image data, deterministic
    __shared__ float sg[6][10][34];
    __shared__ PostCam cam_s;
    if (threadIdx.x == 0) {
        const float* r = g.cams + 4 * (size_t)f;
        cam_s = g.cams ? load_cam(wvt + (size_t)f * 16, W, H, __ldg(r), __ldg(r + 1), __ldg(r + 2), __ldg(r + 3))
                       : load_cam(wvt + (size_t)f * 16, W, H, g.tanx, g.tany);
    }
    __syncthreads();
    const PostCam& c = cam_s;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;               // surf_normal at this pixel
    if (g.lambda_normal != 0.f) {
        float sn[3], gdx[3], gdy[3];
        stencil_eval(c, g, x, y, sd, am, N, -sN, sn, gdx, gdy);
        s0 = sn[0]; s1 = sn[1]; s2 = sn[2];
#pragma unroll
        for (int k = 0; k < 3; k++) { sg[k][ly + 1][lx + 1] = gdx[k]; sg[3 + k][ly + 1][lx + 1] = gdy[k]; }
        const int t = threadIdx.x;
        if (t < 80) {                                  // the ring (corners are never read)
            const int row = t < 32 ? 0 : (t < 64 ? 9 : (t < 72 ? t - 63 : t - 71));
            const int col = t < 32 ? t + 1 : (t < 64 ? t - 31 : (t < 72 ? 0 : 33));
            stencil_eval(c, g, (int)blockIdx.x * 32 + col - 1, (int)blockIdx.y * 8 + row - 1, sd, am, N, -sN, sn, gdx, gdy);
#pragma unroll
            for (int k = 0; k < 3; k++) { sg[k][row][col] = gdx[k]; sg[3 + k][row][col] = gdy[k]; }
        }
    }
    __syncthreads();
    float part[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};   // rgb, mask, normal, dist loss terms; dL/dbkgd
    if (x < W && y < H) {
        const size_t p = (size_t)y * W + x;
        const float a = am[N + p], d0 = am[p], m5 = am[5 * N + p];
        const float n0 = am[2 * N + p], n1 = am[3 * N + p], n2 = am[4 * N + p];
        float g_acc = 0.f;
        // ---- rgb: masked L1 (model.py:674-692), after the optional learnable-background composite
        const float v = vis2d ? (vis2d[(size_t)f * N + p] > 0.f ? 1.f : 0.f) : 1.f;
        const float s_rgb = g.w_rgb * invN * (1.0f / 3.0f);
#pragma unroll
        for (int ch = 0; ch < 3; ch++) {
            float col = color[((size_t)f * 3 + ch) * N + p];
            const float bk = bkgd ? __ldg(bkgd + ch) : 0.f;
            col += (1.f - a) * bk;
            const float d = col - target[((size_t)f * 3 + ch) * N + p];
            part[0] += fabsf(d) * v * s_rgb;
            const float gc = (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f)) * v * s_rgb;
            g_color[((size_t)f * 3 + ch) * N + p] = gc;
            part[4 + ch] = gc * (1.f - a);
            g_acc -= gc * bk;
        }
        // ---- mask: (acc - gt)^2 * balance weight (model.py:649-653)
        if (mask_gt) {
            const float wt = mask_wt ? mask_wt[(size_t)f * N + p] : 1.f;
            const float d = a - mask_gt[(size_t)f * N + p];
            part[1] = g.w_mask * d * d * wt * invN;
            g_acc += g.w_mask * 2.f * d * wt * invN;
        }
        // ---- normal consistency: lambda_n * mean(1 - <rend_normal, surf_normal>)   (model.py:817-842)
        const float r0 = c.R[0] * n0 + c.R[1] * n1 + c.R[2] * n2, r1 = c.R[3] * n0 + c.R[4] * n1 + c.R[5] * n2,
                    r2 = c.R[6] * n0 + c.R[7] * n1 + c.R[8] * n2;
        part[2] = sN * (1.f - (r0 * s0 + r1 * s1 + r2 * s2));
        // d/d rend_normal = -sN * surf_normal  ->  allmap[2..4] through W^T
        const float q0 = -sN * s0, q1 = -sN * s1, q2 = -sN * s2;
        float* ga = g_allmap + (size_t)f * 8 * N;
        ga[2 * N + p] = c.R[0] * q0 + c.R[3] * q1 + c.R[6] * q2;
        ga[3 * N + p] = c.R[1] * q0 + c.R[4] * q1 + c.R[7] * q2;
        ga[4 * N + p] = c.R[2] * q0 + c.R[5] * q1 + c.R[8] * q2;
        // d/d surf_depth[p]: gather from the four stencils this pixel takes part in (points[y+1] - points[y-1] is dx of
        // the stencil at y, so the pixel is "down" for the stencil above it and "up" for the one below; same along x)
        float gp0 = 0.f, gp1 = 0.f, gp2 = 0.f;
        if (g.lambda_normal != 0.f) {
            gp0 = sg[0][ly][lx + 1] - sg[0][ly + 2][lx + 1] + sg[3][ly + 1][lx] - sg[3][ly + 1][lx + 2];
            gp1 = sg[1][ly][lx + 1] - sg[1][ly + 2][lx + 1] + sg[4][ly + 1][lx] - sg[4][ly + 1][lx + 2];
            gp2 = sg[2][ly][lx + 1] - sg[2][ly + 2][lx + 1] + sg[5][ly + 1][lx] - sg[5][ly + 1][lx + 2];
        }
        float rx, ry, rz;
        ray_dir(c, x, y, rx, ry, rz);
        const float gsd = gp0 * rx + gp1 * ry + gp2 * rz;
        const float gex = gsd * (1.f - g.depth_ratio), gmed = gsd * g.depth_ratio;
        const float q = d0 / a;
        const bool qfin = isfinite(q);                  // nan_to_num passes the gradient only where its input is finite
        ga[p] = qfin ? gex / a : 0.f;
        ga[N + p] = g_acc + (qfin ? -gex * d0 / (a * a) : 0.f);
        ga[5 * N + p] = isfinite(m5) ? gmed : 0.f;
        // ---- distortion: lambda_d * mean(rend_dist)
        part[3] = g.lambda_dist * am[6 * N + p] * invN;
        ga[6 * N + p] = g.lambda_dist * invN;
        ga[7 * N + p] = 0.f;
    }
    // ---- block reduction of the loss terms (and dL/dbkgd): 7 atomics per block
    __shared__ float red[8][7];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 7; i++) {
        float vsum = part[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) vsum += __shfl_xor_sync(0xffffffffu, vsum, o);
        if (lane == 0) red[warp][i] = vsum;
    }
    __syncthreads();
    if (threadIdx.x < 7) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; w++) t += red[w][threadIdx.x];
        if (threadIdx.x < 4) atomicAdd(loss_terms + (size_t)f * 4 + threadIdx.x, t);
        else if (g_bkgd) atomicAdd(g_bkgd + (size_t)f * 3 + (threadIdx.x - 4), t);
    }
}

// ---- Stage-3 losses on the feature planes (DESIGN.md section 3.5a):
//   lab4d/engine/model.py:663-667   feature:        v = ||feat_r - feat_gt||_2 over the Cf target channels
//   lab4d/engine/model.py:742-745   reg_gauss_mask: v = (gauss_mask_r - acc.detach())^2
//   lab4d/engine/model.py:952-967   feature masked by the gt mask and the frame's is_detected; reg_gauss_mask unmasked
//   lab4d/engine/model.py:1000-1012 term = w * mean(v[v > 0]) over the whole batch (v.mean() = 0 when nothing is > 0)
// The denominator is a batch-wide count, known only after every pixel has been seen, so the pass is two launches:
// feat_loss_kernel writes the UNSCALED per-pixel gradient (dv/dfeat where v > 0, else 0) and per-frame block-reduced
// sums and counts; feat_loss_scale_kernel multiplies the touched planes and the sums by w_k / C_k (0 when C_k = 0).
// Every pixel's gradient is written by its own thread: no atomics on image data, deterministic planes.
struct FeatLossCfg {
    int W, H, F, Cf, gm;    // Cf = 0: no feature term; gm = -1: no Gaussian-mask term
};

__global__ void __launch_bounds__(256)
feat_loss_kernel(const FeatLossCfg g, const float* __restrict__ feat, const float* __restrict__ target,
                 const float* __restrict__ mask_gt, const float* __restrict__ is_detected, const float* __restrict__ allmap,
                 float* __restrict__ terms, uint32_t* __restrict__ counts, float* __restrict__ g_feat) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    const size_t N = (size_t)g.W * g.H;
    float part[2] = {0.f, 0.f};
    uint32_t cnt[2] = {0u, 0u};
    if (x < g.W && y < g.H) {
        const size_t p = (size_t)y * g.W + x;
        const float* fe = feat + (size_t)f * g.F * N + p;
        float* gf = g_feat + (size_t)f * g.F * N + p;
        if (g.Cf > 0) {
            const float* tg = target + (size_t)f * g.Cf * N + p;
            const float wpx = mask_gt[(size_t)f * N + p] * (is_detected ? __ldg(is_detected + f) : 1.f);
            float ss = 0.f;
            for (int c = 0; c < g.Cf; c++) {
                const float d = fe[c * N] - tg[c * N];
                ss += d * d;
            }
            const float nrm = sqrtf(ss), v = nrm * wpx;
            const bool on = v > 0.f;                     // also excludes ||d|| = 0, where torch's norm gradient is 0
            const float k = on ? wpx / nrm : 0.f;
            for (int c = 0; c < g.Cf; c++) gf[c * N] = (fe[c * N] - tg[c * N]) * k;
            part[0] = on ? v : 0.f;
            cnt[0] = on;
        }
        for (int c = g.Cf; c < g.F; c++)
            if (c != g.gm) gf[c * N] = 0.f;
        if (g.gm >= 0) {
            const float d = fe[g.gm * N] - allmap[(size_t)f * 8 * N + N + p];
            const float v = d * d;
            const bool on = v > 0.f;
            gf[g.gm * N] = on ? 2.f * d : 0.f;
            part[1] = on ? v : 0.f;
            cnt[1] = on;
        }
    }
    // block reduction as in loss_grad_kernel: 2 float + 2 integer atomics per block
    __shared__ float red[8][2];
    __shared__ uint32_t redc[8][2];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int i = 0; i < 2; i++) {
        float vs = part[i];
        uint32_t cs = cnt[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            vs += __shfl_xor_sync(0xffffffffu, vs, o);
            cs += __shfl_xor_sync(0xffffffffu, cs, o);
        }
        if (lane == 0) { red[warp][i] = vs; redc[warp][i] = cs; }
    }
    __syncthreads();
    if (threadIdx.x < 2) {
        float t = 0.f;
        uint32_t c = 0u;
#pragma unroll
        for (int w = 0; w < 8; w++) { t += red[w][threadIdx.x]; c += redc[w][threadIdx.x]; }
        if (c) {
            atomicAdd(terms + (size_t)f * 2 + threadIdx.x, t);
            atomicAdd(counts + (size_t)f * 2 + threadIdx.x, c);
        }
    }
}

__global__ void __launch_bounds__(256)
feat_loss_scale_kernel(const FeatLossCfg g, const float* __restrict__ weights, const uint32_t* __restrict__ counts,
                       float* __restrict__ terms, float* __restrict__ g_feat) {
    const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5), f = blockIdx.z;
    __shared__ float s[2];
    if (threadIdx.x < 2) {
        unsigned long long c = 0;                      // the count over the whole batch: the reference's v[v > 0].mean()
        for (int m = 0; m < (int)gridDim.z; m++) c += counts[(size_t)m * 2 + threadIdx.x];
        s[threadIdx.x] = c ? __ldg(weights + threadIdx.x) / (float)c : 0.f;
        if (blockIdx.x == 0 && blockIdx.y == 0) terms[(size_t)f * 2 + threadIdx.x] *= s[threadIdx.x];
    }
    __syncthreads();
    if (x >= g.W || y >= g.H) return;
    const size_t N = (size_t)g.W * g.H;
    float* gf = g_feat + (size_t)f * g.F * N + (size_t)y * g.W + x;
    const float s0 = s[0];
    for (int c = 0; c < g.Cf; c++) gf[c * N] *= s0;
    if (g.gm >= 0) gf[g.gm * N] *= s[1];
}

// sr_render_loss_batch and sr_render_loss_batch_cameras: `cams` (nullptr = the shared tanx / tany) is the only difference
int render_loss_batch(const char* name, int32_t M, int32_t W, int32_t H, const float* cams, float tanx, float tany,
                             float depth_ratio, const float* color, const float* allmap, const float* world_view_transform,
                             const float* target_rgb, const float* vis2d, const float* mask_gt, const float* mask_wt,
                             const float* learnable_bkgd, float w_rgb, float w_mask, float lambda_normal, float lambda_dist,
                             float* loss_terms, float* dL_dcolor, float* dL_dallmap, float* dL_dbkgd, float* surf_depth_scratch,
                             void* stream_) {
    if (M < 1 || W <= 0 || H <= 0) return sr_fail(SR_EINVAL, "%s: M, W and H must be positive", name);
    if (!color || !allmap || !world_view_transform || !target_rgb || !loss_terms || !dL_dcolor || !dL_dallmap || !surf_depth_scratch)
        return sr_fail(SR_EINVAL, "%s: a required pointer is NULL", name);
    cudaStream_t s = (cudaStream_t)stream_;
    LossCfg g{W, H, cams, tanx, tany, depth_ratio, w_rgb, w_mask, lambda_normal, lambda_dist};
    dim3 grid((W + 31) / 32, (H + 7) / 8, M);
    CK(cudaMemsetAsync(loss_terms, 0, (size_t)M * 4 * sizeof(float), s), "sr_render_loss_batch: memset(loss_terms)");
    if (dL_dbkgd) CK(cudaMemsetAsync(dL_dbkgd, 0, (size_t)M * 3 * sizeof(float), s), "sr_render_loss_batch: memset(dL_dbkgd)");
    {
        ProfileScope ps("loss_depth", s);
        loss_depth_kernel<<<grid, 256, 0, s>>>(g, allmap, surf_depth_scratch);
    }
    {
        ProfileScope ps("loss_grad", s);
        loss_grad_kernel<<<grid, 256, 0, s>>>(g, color, allmap, world_view_transform, target_rgb, vis2d, mask_gt, mask_wt,
                                             learnable_bkgd, surf_depth_scratch, loss_terms, dL_dcolor, dL_dallmap, dL_dbkgd);
    }
    return sr_launched(2, name);
}

}  // namespace

extern "C" {

SR_API int sr_render_loss_batch(int32_t M, int32_t W, int32_t H, float tanx, float tany, float depth_ratio,
                                const float* color, const float* allmap, const float* world_view_transform,
                                const float* target_rgb, const float* vis2d, const float* mask_gt, const float* mask_wt,
                                const float* learnable_bkgd, float w_rgb, float w_mask, float lambda_normal, float lambda_dist,
                                float* loss_terms, float* dL_dcolor, float* dL_dallmap, float* dL_dbkgd, float* surf_depth_scratch,
                                void* stream_) {
    return render_loss_batch("sr_render_loss_batch", M, W, H, nullptr, tanx, tany, depth_ratio, color, allmap,
                             world_view_transform, target_rgb, vis2d, mask_gt, mask_wt, learnable_bkgd, w_rgb, w_mask,
                             lambda_normal, lambda_dist, loss_terms, dL_dcolor, dL_dallmap, dL_dbkgd, surf_depth_scratch, stream_);
}

SR_API int sr_render_loss_batch_cameras(int32_t M, int32_t W, int32_t H, const float* cameras, float depth_ratio,
                                        const float* color, const float* allmap, const float* world_view_transform,
                                        const float* target_rgb, const float* vis2d, const float* mask_gt,
                                        const float* mask_wt, const float* learnable_bkgd, float w_rgb, float w_mask,
                                        float lambda_normal, float lambda_dist, float* loss_terms, float* dL_dcolor,
                                        float* dL_dallmap, float* dL_dbkgd, float* surf_depth_scratch, void* stream_) {
    if (!cameras) return sr_fail(SR_EINVAL, "sr_render_loss_batch_cameras: the per-frame camera table is NULL");
    return render_loss_batch("sr_render_loss_batch_cameras", M, W, H, cameras, 0.f, 0.f, depth_ratio, color, allmap,
                             world_view_transform, target_rgb, vis2d, mask_gt, mask_wt, learnable_bkgd, w_rgb, w_mask,
                             lambda_normal, lambda_dist, loss_terms, dL_dcolor, dL_dallmap, dL_dbkgd, surf_depth_scratch, stream_);
}

SR_API int sr_feature_loss_batch(int32_t M, int32_t W, int32_t H, int32_t F, int32_t Cf, int32_t gauss_mask_channel,
                                 const float* features, const float* target, const float* mask_gt, const float* is_detected,
                                 const float* allmap, const float* weights, float* feature_terms, uint32_t* counts,
                                 float* dL_dfeatures, void* stream_) {
    if (M < 1 || W <= 0 || H <= 0) return sr_fail(SR_EINVAL, "M, W and H must be positive");
    if (F < 1) return sr_fail(SR_EINVAL, "F must be >= 1, got %d", F);
    if (!features || !allmap || !weights || !feature_terms || !counts || !dL_dfeatures)
        return sr_fail(SR_EINVAL, "features, allmap, weights, feature_terms, counts and dL_dfeatures must not be NULL");
    if (target) {
        if (Cf < 1 || Cf > F) return sr_fail(SR_EINVAL, "Cf must be in [1, F = %d] with a target, got %d", F, Cf);
        if (!mask_gt) return sr_fail(SR_EINVAL, "the feature term needs mask_gt");
    } else if (Cf != 0) {
        return sr_fail(SR_EINVAL, "Cf must be 0 without a target, got %d", Cf);
    }
    if (gauss_mask_channel < -1 || gauss_mask_channel >= F)
        return sr_fail(SR_EINVAL, "gauss_mask_channel must be -1 or in [0, F = %d), got %d", F, gauss_mask_channel);
    if (gauss_mask_channel >= 0 && gauss_mask_channel < Cf)
        return sr_fail(SR_EINVAL, "gauss_mask_channel %d lies inside the feature target's channels [0, %d)",
                       gauss_mask_channel, Cf);
    if (!target && gauss_mask_channel < 0) return sr_fail(SR_EINVAL, "no term: neither a target nor a gauss_mask_channel");
    cudaStream_t s = (cudaStream_t)stream_;
    const FeatLossCfg g{W, H, F, Cf, gauss_mask_channel};
    dim3 grid((W + 31) / 32, (H + 7) / 8, M);
    CK(cudaMemsetAsync(feature_terms, 0, (size_t)M * 2 * sizeof(float), s), "sr_feature_loss_batch: memset(feature_terms)");
    CK(cudaMemsetAsync(counts, 0, (size_t)M * 2 * sizeof(uint32_t), s), "sr_feature_loss_batch: memset(counts)");
    {
        ProfileScope ps("feat_loss", s);
        feat_loss_kernel<<<grid, 256, 0, s>>>(g, features, target, mask_gt, is_detected, allmap, feature_terms, counts,
                                              dL_dfeatures);
    }
    {
        ProfileScope ps("feat_loss_scale", s);
        feat_loss_scale_kernel<<<grid, 256, 0, s>>>(g, weights, counts, feature_terms, dL_dfeatures);
    }
    return sr_launched(2, "sr_feature_loss_batch");
}

}  // extern "C"
