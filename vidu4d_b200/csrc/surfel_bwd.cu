// surfel_bwd.cu -- per-surfel backward: projected-AABB vjp, tangent-plane homography vjp,
// quaternion / scale vjp and SH vjp, fused into one streaming kernel.
//
// Replaces (behaviour, not code) of the reference:
//   computeAABB (bwd)        RAST/cuda_rasterizer/backward.cu:599-649
//   preprocessCUDA (bwd)     RAST/cuda_rasterizer/backward.cu:533-597
//   computeTransMat vjp      RAST/cuda_rasterizer/backward.cu:451-529
//   quat_to_rotmat_vjp       RAST/cuda_rasterizer/auxiliary.h:213-257
//   computeColorFromSH (bwd) RAST/cuda_rasterizer/backward.cu:20-139
//
// The reference runs two kernels over nine zero-filled P-sized tensors; here one kernel reads the
// 80-byte per-surfel accumulator written by the composite backward and writes every output tensor
// exactly once (including the zeros of invisible surfels), so the caller can hand in torch.empty().
#include "common.cuh"

namespace {

__constant__ float kSH_C0 = 0.28209479177387814f;
__constant__ float kSH_C1 = 0.4886025119029199f;
__constant__ float kSH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                                -1.0925484305920792f, 0.5462742152960396f};
__constant__ float kSH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                                0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                                -0.5900435899266435f};

struct V3 { float x, y, z; };
__device__ __forceinline__ V3 wmul(const float* m, V3 v) {      // W * v
    return {m[0] * v.x + m[4] * v.y + m[8] * v.z, m[1] * v.x + m[5] * v.y + m[9] * v.z, m[2] * v.x + m[6] * v.y + m[10] * v.z};
}
__device__ __forceinline__ V3 wtmul(const float* m, V3 v) {     // W^T * v
    return {m[0] * v.x + m[1] * v.y + m[2] * v.z, m[4] * v.x + m[5] * v.y + m[6] * v.z, m[8] * v.x + m[9] * v.y + m[10] * v.z};
}

// one surfel's gradients for one frame (everything except dL/dSH, which goes through the shared-memory row)
struct SurfelGrad {
    float m2d[3], col[3], op, m3d[3], tm[9], sc[2], rot[4];
};

template <bool ACC>
__device__ __forceinline__ void
surfel_bwd_body(const CamParams& c, const int idx, const int M, const float* shv, float* shg, const float* __restrict__ means3D,
                const bool has_sh, const float2* __restrict__ scales, const float4* __restrict__ rotations,
                const float4* __restrict__ srec, const uint8_t* __restrict__ clamped, const float4* __restrict__ sgrad,
                SurfelGrad& G);

// Block = 128 surfels.  The block's SH coefficients (128 x 3M floats, contiguous in HBM) are pulled into shared
// memory with coalesced 128-bit loads, each thread works on its own padded rows (stride 3M+1: conflict-free) -- one
// row of SH values, one of dL/dSH -- and the block streams the gradient rows back out coalesced, instead of 48 scalar
// loads and 48 scalar stores per thread at a 192-byte lane stride (r1a: 118 us for 175 MB).
//
// Batches: the kernel loops over the frames INSIDE the thread.  An input that is shared by the frames of a batch
// (stride 0: in Stage 3 everything except positions and orientations) gets ONE gradient, the sum over frames,
// accumulated in registers / in the shared-memory row and written once -- the (M, P, 48) dL/dSH tensor and the torch
// reduction over M that would follow never exist.  Per-frame inputs get per-frame gradients.
constexpr int SB = 128;

__device__ __forceinline__ void stage_rows_in(float* dst, const float* __restrict__ gsrc, int nrows, int M3, int stride) {
    const int total = nrows * M3;
    if ((M3 & 3) == 0) {
        const float4* g4 = reinterpret_cast<const float4*>(gsrc);
        for (int i = threadIdx.x; i < total / 4; i += SB) {
            const float4 v = __ldg(g4 + i);
            const int e = i * 4, r = e / M3, col = e - r * M3;     // 4 | M3 => the four stay in one row
            float* d = dst + r * stride + col;
            d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
        }
    } else {
        for (int i = threadIdx.x; i < total; i += SB) { const int r = i / M3; dst[r * stride + (i - r * M3)] = __ldg(gsrc + i); }
    }
}
__device__ __forceinline__ void stage_rows_out(float* __restrict__ gdst, const float* src, int nrows, int M3, int stride) {
    const int total = nrows * M3;
    if ((M3 & 3) == 0) {
        float4* g4 = reinterpret_cast<float4*>(gdst);
        for (int i = threadIdx.x; i < total / 4; i += SB) {
            const int e = i * 4, r = e / M3, col = e - r * M3;
            const float* d = src + r * stride + col;
            g4[i] = make_float4(d[0], d[1], d[2], d[3]);
        }
    } else {
        for (int i = threadIdx.x; i < total; i += SB) { const int r = i / M3; gdst[i] = src[r * stride + (i - r * M3)]; }
    }
}

// 5 blocks per SM (at most 102 registers): without the bound, the per-frame intrinsics of a camera table (common.cuh
// cam_of_frame) take the kernel to 112 registers and 4 blocks whenever shared memory does not limit it first
__global__ void __launch_bounds__(SB, 5)
surfel_bwd_kernel(const CamParams c_, const FrameStrides fs, const float* __restrict__ means3D, const float* __restrict__ shs,
                  const float2* __restrict__ scales, const float4* __restrict__ rotations, const int* __restrict__ radii,
                  const float4* __restrict__ srec, const uint8_t* __restrict__ clamped, const float4* __restrict__ sgrad,
                  float* __restrict__ dL_dmeans2D, float* __restrict__ dL_dcolors, float* __restrict__ dL_dopacity,
                  float* __restrict__ dL_dmeans3D, float* __restrict__ dL_dtransMat, float* __restrict__ dL_dsh,
                  float2* __restrict__ dL_dscales, float4* __restrict__ dL_drotations) {
    extern __shared__ float shbuf[];
    const int M = c_.M, M3 = 3 * M, stride = M3 + 1;
    const int idx = blockIdx.x * SB + threadIdx.x;
    const int base = blockIdx.x * SB;
    const int nrows = min(SB, c_.P - base);
    const bool has_sh = shs != nullptr;
    float* shv_all = shbuf;                          // SH values      [SB][stride]
    float* shg_all = shbuf + SB * stride;            // dL/dSH         [SB][stride]
    float* shv = shv_all + threadIdx.x * stride;
    float* shg = shg_all + threadIdx.x * stride;
    // which gradients are sums over the frames (their input is shared by the batch)
    const bool multi = fs.frames > 1;
    const bool sum_sh = multi && fs.g_sh == 0, sum_m3d = multi && fs.g_m3d == 0, sum_op = multi && fs.g_opac == 0;
    const bool sum_sc = multi && fs.g_scales == 0, sum_rot = multi && fs.g_rots == 0, sum_col = multi && fs.g_col == 0;
    float a_m3d[3] = {0.f, 0.f, 0.f}, a_col[3] = {0.f, 0.f, 0.f}, a_op = 0.f, a_sc[2] = {0.f, 0.f}, a_rot[4] = {0.f, 0.f, 0.f, 0.f};
    if (has_sh && sum_sh) for (int i = 0; i < M3; i++) shg[i] = 0.f;

    for (int f = 0; f < fs.frames; f++) {
        const CamParams c = cam_of_frame(c_, fs, f);
        if (has_sh && (f == 0 || fs.shs != 0)) {
            __syncthreads();                         // previous frame's readers of shv are done
            stage_rows_in(shv_all, fr(shs, fs.shs, f) + (size_t)base * M3, nrows, M3, stride);
            __syncthreads();
        }
        if (idx < c.P) {
            SurfelGrad G;
            const bool vis = fr(radii, fs.radii, f)[idx] > 0;
            if (vis) {
                if (sum_sh)
                    surfel_bwd_body<true>(c, idx, M, shv, shg, fr(means3D, fs.means3D, f), has_sh, fr(scales, fs.scales, f),
                                          fr(rotations, fs.rots, f), fr(srec, fs.geom, f), fr(clamped, fs.geom, f), fr(sgrad, fs.geom, f), G);
                else
                    surfel_bwd_body<false>(c, idx, M, shv, shg, fr(means3D, fs.means3D, f), has_sh, fr(scales, fs.scales, f),
                                           fr(rotations, fs.rots, f), fr(srec, fs.geom, f), fr(clamped, fs.geom, f), fr(sgrad, fs.geom, f), G);
            } else {
                // invisible in this frame: every gradient is zero (the reference leaves its zero-filled tensors untouched)
#pragma unroll
                for (int i = 0; i < 3; i++) { G.m2d[i] = 0.f; G.col[i] = 0.f; G.m3d[i] = 0.f; }
                G.op = 0.f; G.sc[0] = G.sc[1] = 0.f;
#pragma unroll
                for (int i = 0; i < 4; i++) G.rot[i] = 0.f;
#pragma unroll
                for (int i = 0; i < 9; i++) G.tm[i] = 0.f;
                if (has_sh && !sum_sh) for (int i = 0; i < M3; i++) shg[i] = 0.f;
            }
            // ---- per-frame outputs are written now, shared ones accumulate
            float* o2d = fr(dL_dmeans2D, fs.g_m2d, f) + 3 * (size_t)idx;
            o2d[0] = G.m2d[0]; o2d[1] = G.m2d[1]; o2d[2] = G.m2d[2];
            if (dL_dtransMat != nullptr) {
                float* otm = fr(dL_dtransMat, fs.g_tm, f) + 9 * (size_t)idx;
#pragma unroll
                for (int i = 0; i < 9; i++) otm[i] = G.tm[i];
            }
            if (sum_m3d) { a_m3d[0] += G.m3d[0]; a_m3d[1] += G.m3d[1]; a_m3d[2] += G.m3d[2]; }
            else { float* o = fr(dL_dmeans3D, fs.g_m3d, f) + 3 * (size_t)idx; o[0] = G.m3d[0]; o[1] = G.m3d[1]; o[2] = G.m3d[2]; }
            if (sum_col) { a_col[0] += G.col[0]; a_col[1] += G.col[1]; a_col[2] += G.col[2]; }
            else { float* o = fr(dL_dcolors, fs.g_col, f) + 3 * (size_t)idx; o[0] = G.col[0]; o[1] = G.col[1]; o[2] = G.col[2]; }
            if (sum_op) a_op += G.op; else fr(dL_dopacity, fs.g_opac, f)[idx] = G.op;
            if (sum_sc) { a_sc[0] += G.sc[0]; a_sc[1] += G.sc[1]; } else fr(dL_dscales, fs.g_scales, f)[idx] = make_float2(G.sc[0], G.sc[1]);
            if (sum_rot) { a_rot[0] += G.rot[0]; a_rot[1] += G.rot[1]; a_rot[2] += G.rot[2]; a_rot[3] += G.rot[3]; }
            else fr(dL_drotations, fs.g_rots, f)[idx] = make_float4(G.rot[0], G.rot[1], G.rot[2], G.rot[3]);
        }
        if (has_sh && !sum_sh) {
            __syncthreads();
            stage_rows_out(fr(dL_dsh, fs.g_sh, f) + (size_t)base * M3, shg_all, nrows, M3, stride);
        }
    }
    if (idx < c_.P) {
        if (sum_m3d) { float* o = dL_dmeans3D + 3 * (size_t)idx; o[0] = a_m3d[0]; o[1] = a_m3d[1]; o[2] = a_m3d[2]; }
        if (sum_col) { float* o = dL_dcolors + 3 * (size_t)idx; o[0] = a_col[0]; o[1] = a_col[1]; o[2] = a_col[2]; }
        if (sum_op) dL_dopacity[idx] = a_op;
        if (sum_sc) dL_dscales[idx] = make_float2(a_sc[0], a_sc[1]);
        if (sum_rot) dL_drotations[idx] = make_float4(a_rot[0], a_rot[1], a_rot[2], a_rot[3]);
    }
    if (has_sh && sum_sh) {
        __syncthreads();
        stage_rows_out(dL_dsh + (size_t)base * M3, shg_all, nrows, M3, stride);
    }
}

template <bool ACC>
__device__ __forceinline__ void
surfel_bwd_body(const CamParams& c, const int idx, const int M, const float* shv, float* shg, const float* __restrict__ means3D,
                const bool has_sh, const float2* __restrict__ scales, const float4* __restrict__ rotations,
                const float4* __restrict__ srec, const uint8_t* __restrict__ clamped, const float4* __restrict__ sgrad,
                SurfelGrad& G) {
    float vm[16];
#pragma unroll
    for (int i = 0; i < 16; i++) vm[i] = __ldg(c.vm + i);
    const float4* g4 = sgrad + (size_t)idx * 5;
    const float4 g0 = g4[0], g1 = g4[1], g2 = g4[2], g3 = g4[3], g4v = g4[4];
    float dT[9] = {g0.x, g0.y, g0.z, g0.w, g1.x, g1.y, g1.z, g1.w, g2.x};
    // accumulator layout: common.cuh SR_G_*
    const float dop = g2.y;
    const float dcol[3] = {g2.z, g2.w, g3.x};
    const float dnr[3] = {g3.y, g3.z, g3.w};
    const float dmx = g4v.x, dmy = g4v.y;
    const float4* r4 = srec + (size_t)idx * 5;
    const float4 r0 = __ldg(r4), r1 = __ldg(r4 + 1), r2 = __ldg(r4 + 2);
    const float T[9] = {r0.x, r0.y, r0.z, r0.w, r1.x, r1.y, r1.z, r1.w, r2.x};

    // ---- computeAABB vjp (backward.cu:599-649): dL/dcentre -> dL/dT ----
    {
        const float d = T[6] * T[6] + T[7] * T[7] - T[8] * T[8];
        const float inv = 1.0f / d;
        const float f[3] = {inv, inv, -inv};
        float dL_dT3[3], dL_df[3];
#pragma unroll
        for (int i = 0; i < 3; i++) {
            dT[i] += dmx * f[i] * T[6 + i];
            dT[3 + i] += dmy * f[i] * T[6 + i];
            dL_dT3[i] = dmx * f[i] * T[i] + dmy * f[i] * T[3 + i];
            dL_df[i] = dmx * T[i] * T[6 + i] + dmy * T[3 + i] * T[6 + i];
        }
        const float dL_dd = (dL_df[0] * f[0] + dL_df[1] * f[1] + dL_df[2] * f[2]) * (-1.0f / d);
        dT[6] += dL_dT3[0] + dL_dd * (2.0f * T[6]);
        dT[7] += dL_dT3[1] + dL_dd * (2.0f * T[7]);
        dT[8] += dL_dT3[2] + dL_dd * (-2.0f * T[8]);
    }
#pragma unroll
    for (int i = 0; i < 9; i++) G.tm[i] = dT[i];
    // densification proxy that the reference stores into dL_dmean2D (backward.cu:645-648)
    G.m2d[0] = dT[2] * T[8] * c.bcx;
    G.m2d[1] = dT[5] * T[8] * c.bcy;
    G.m2d[2] = 0.f;
    G.op = dop;
#pragma unroll
    for (int i = 0; i < 3; i++) G.col[i] = dcol[i];

    // ---- computeTransMat vjp (backward.cu:451-529) ----
    const float4 q = __ldg(rotations + idx);
    const float2 sc = __ldg(scales + idx);
    const float sN = rsqrtf(q.w * q.w + q.x * q.x + q.y * q.y + q.z * q.z);
    const float w = q.x * sN, x = q.y * sN, y = q.z * sN, z = q.w * sN;
    // column-major R of the normalised quaternion
    const float R[9] = {1.f - 2.f * (y * y + z * z), 2.f * (x * y + w * z), 2.f * (x * z - w * y),
                        2.f * (x * y - w * z), 1.f - 2.f * (x * x + z * z), 2.f * (y * z + w * x),
                        2.f * (x * z + w * y), 2.f * (y * z - w * x), 1.f - 2.f * (x * x + y * y)};
    const V3 p = {__ldg(means3D + 3 * (size_t)idx), __ldg(means3D + 3 * (size_t)idx + 1), __ldg(means3D + 3 * (size_t)idx + 2)};
    V3 pv = wmul(vm, p);
    pv.x += vm[12]; pv.y += vm[13]; pv.z += vm[14];
    // dL_dM column j = K^T (dTu[j], dTv[j], dTw[j]) with the BACKWARD intrinsics (cx = focal*tanfov + cx_off)
    V3 dM[3];
#pragma unroll
    for (int j = 0; j < 3; j++) {
        dM[j].x = c.focal_x * dT[j];
        dM[j].y = c.focal_y * dT[3 + j];
        dM[j].z = c.kcx * dT[j] + c.kcy * dT[3 + j] + dT[6 + j];
    }
    const V3 dRS0 = wtmul(vm, dM[0]), dRS1 = wtmul(vm, dM[1]), dpw = wtmul(vm, dM[2]);
    V3 dtn = wtmul(vm, V3{dnr[0], dnr[1], dnr[2]});
    const V3 tn = wmul(vm, V3{R[6], R[7], R[8]});
    const float cosv = -tn.x * pv.x - tn.y * pv.y - tn.z * pv.z;
    const float mult = cosv > 0.f ? 1.f : -1.f;
    dtn.x *= mult; dtn.y *= mult; dtn.z *= mult;
    // v_R[col][row]
    const float vR[3][3] = {{dRS0.x * sc.x, dRS0.y * sc.x, dRS0.z * sc.x},
                            {dRS1.x * sc.y, dRS1.y * sc.y, dRS1.z * sc.y},
                            {dtn.x, dtn.y, dtn.z}};
    float4 dq;
    dq.x = 2.f * (x * (vR[1][2] - vR[2][1]) + y * (vR[2][0] - vR[0][2]) + z * (vR[0][1] - vR[1][0]));
    dq.y = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[0][1] + vR[1][0]) + z * (vR[0][2] + vR[2][0]) + w * (vR[1][2] - vR[2][1]));
    dq.z = 2.f * (x * (vR[0][1] + vR[1][0]) - 2.f * y * (vR[0][0] + vR[2][2]) + z * (vR[1][2] + vR[2][1]) + w * (vR[2][0] - vR[0][2]));
    dq.w = 2.f * (x * (vR[0][2] + vR[2][0]) + y * (vR[1][2] + vR[2][1]) - 2.f * z * (vR[0][0] + vR[1][1]) + w * (vR[0][1] - vR[1][0]));
    G.rot[0] = dq.x; G.rot[1] = dq.y; G.rot[2] = dq.z; G.rot[3] = dq.w;
    G.sc[0] = dRS0.x * R[0] + dRS0.y * R[1] + dRS0.z * R[2];
    G.sc[1] = dRS1.x * R[3] + dRS1.y * R[4] + dRS1.z * R[5];
    float dmean[3] = {dpw.x, dpw.y, dpw.z};

    // ---- SH vjp (backward.cu:20-139) ----
    if (has_sh) {
        const int deg = c.D;
        const float dox = p.x - __ldg(c.campos), doy = p.y - __ldg(c.campos + 1), doz = p.z - __ldg(c.campos + 2);
        const float len = sqrtf(dox * dox + doy * doy + doz * doz);
        const float dx = dox / len, dy = doy / len, dz = doz / len;
        const uint32_t cl = clamped[idx];
        float dRGB[3];
#pragma unroll
        for (int ch = 0; ch < 3; ch++) dRGB[ch] = (cl >> ch) & 1u ? 0.f : dcol[ch];
        float ddx = 0.f, ddy = 0.f, ddz = 0.f;   // dL/ddir accumulated over channels
#define SH(k, ch) shv[3 * (k) + (ch)]
#define SETSH(k, wgt) { const float w_ = (wgt); \
        if (ACC) { shg[3 * (k)] += w_ * dRGB[0]; shg[3 * (k) + 1] += w_ * dRGB[1]; shg[3 * (k) + 2] += w_ * dRGB[2]; } \
        else { shg[3 * (k)] = w_ * dRGB[0]; shg[3 * (k) + 1] = w_ * dRGB[1]; shg[3 * (k) + 2] = w_ * dRGB[2]; } }
        const float xx = dx * dx, yy = dy * dy, zz = dz * dz, xy = dx * dy, yz = dy * dz, xz = dx * dz;
        // (1) gradient w.r.t. the view direction (reads the SH row)
        if (deg > 0) {
#pragma unroll
            for (int ch = 0; ch < 3; ch++) {
                float gx = -kSH_C1 * SH(3, ch), gy = -kSH_C1 * SH(1, ch), gz = kSH_C1 * SH(2, ch);
                if (deg > 1) {
                    gx += kSH_C2[0] * dy * SH(4, ch) + kSH_C2[2] * 2.f * -dx * SH(6, ch) + kSH_C2[3] * dz * SH(7, ch) + kSH_C2[4] * 2.f * dx * SH(8, ch);
                    gy += kSH_C2[0] * dx * SH(4, ch) + kSH_C2[1] * dz * SH(5, ch) + kSH_C2[2] * 2.f * -dy * SH(6, ch) + kSH_C2[4] * 2.f * -dy * SH(8, ch);
                    gz += kSH_C2[1] * dy * SH(5, ch) + kSH_C2[2] * 2.f * 2.f * dz * SH(6, ch) + kSH_C2[3] * dx * SH(7, ch);
                    if (deg > 2) {
                        gx += kSH_C3[0] * SH(9, ch) * 3.f * 2.f * xy + kSH_C3[1] * SH(10, ch) * yz + kSH_C3[2] * SH(11, ch) * -2.f * xy +
                              kSH_C3[3] * SH(12, ch) * -3.f * 2.f * xz + kSH_C3[4] * SH(13, ch) * (-3.f * xx + 4.f * zz - yy) +
                              kSH_C3[5] * SH(14, ch) * 2.f * xz + kSH_C3[6] * SH(15, ch) * 3.f * (xx - yy);
                        gy += kSH_C3[0] * SH(9, ch) * 3.f * (xx - yy) + kSH_C3[1] * SH(10, ch) * xz +
                              kSH_C3[2] * SH(11, ch) * (-3.f * yy + 4.f * zz - xx) + kSH_C3[3] * SH(12, ch) * -3.f * 2.f * yz +
                              kSH_C3[4] * SH(13, ch) * -2.f * xy + kSH_C3[5] * SH(14, ch) * -2.f * yz + kSH_C3[6] * SH(15, ch) * -3.f * 2.f * xy;
                        gz += kSH_C3[1] * SH(10, ch) * xy + kSH_C3[2] * SH(11, ch) * 4.f * 2.f * yz +
                              kSH_C3[3] * SH(12, ch) * 3.f * (2.f * zz - xx - yy) + kSH_C3[4] * SH(13, ch) * 4.f * 2.f * xz +
                              kSH_C3[5] * SH(14, ch) * (xx - yy);
                    }
                }
                ddx += gx * dRGB[ch]; ddy += gy * dRGB[ch]; ddz += gz * dRGB[ch];
            }
        }
        // (2) dL/dSH into the gradient row (summed over frames when the SH tensor is shared by the batch)
        SETSH(0, kSH_C0);
        if (deg > 0) {
            SETSH(1, -kSH_C1 * dy); SETSH(2, kSH_C1 * dz); SETSH(3, -kSH_C1 * dx);
            if (deg > 1) {
                SETSH(4, kSH_C2[0] * xy); SETSH(5, kSH_C2[1] * yz); SETSH(6, kSH_C2[2] * (2.f * zz - xx - yy));
                SETSH(7, kSH_C2[3] * xz); SETSH(8, kSH_C2[4] * (xx - yy));
                if (deg > 2) {
                    SETSH(9, kSH_C3[0] * dy * (3.f * xx - yy)); SETSH(10, kSH_C3[1] * xy * dz);
                    SETSH(11, kSH_C3[2] * dy * (4.f * zz - xx - yy)); SETSH(12, kSH_C3[3] * dz * (2.f * zz - 3.f * xx - 3.f * yy));
                    SETSH(13, kSH_C3[4] * dx * (4.f * zz - xx - yy)); SETSH(14, kSH_C3[5] * dz * (xx - yy));
                    SETSH(15, kSH_C3[6] * dx * (xx - 3.f * yy));
                }
            }
        }
        // coefficients above the active degree receive no gradient
        const int used = (deg + 1) * (deg + 1);
        if (!ACC) for (int k = used; k < M; k++) { shg[3 * k] = 0.f; shg[3 * k + 1] = 0.f; shg[3 * k + 2] = 0.f; }
#undef SH
#undef SETSH
        // through the normalisation of the view direction (auxiliary.h:125-135)
        const float sum2 = dox * dox + doy * doy + doz * doz;
        const float inv32 = 1.0f / sqrtf(sum2 * sum2 * sum2);
        dmean[0] += ((sum2 - dox * dox) * ddx - doy * dox * ddy - doz * dox * ddz) * inv32;
        dmean[1] += (-dox * doy * ddx + (sum2 - doy * doy) * ddy - doz * doy * ddz) * inv32;
        dmean[2] += (-dox * doz * ddx - doy * doz * ddy + (sum2 - doz * doz) * ddz) * inv32;
    }
    G.m3d[0] = dmean[0]; G.m3d[1] = dmean[1]; G.m3d[2] = dmean[2];
}

}  // namespace

cudaError_t launch_surfel_bwd(const BwdArgs& a) {
    const int nb = (a.cam.P + SB - 1) / SB;
    const size_t smem = (size_t)2 * SB * (3 * a.cam.M + 1) * sizeof(float);
    if (cudaError_t e = sr_opt_in_smem(surfel_bwd_kernel, smem)) return e;
    ProfileScope ps("surfel_bwd", a.stream);
    surfel_bwd_kernel<<<nb, SB, smem, a.stream>>>(
        a.cam, a.fs, a.means3D, a.shs, (const float2*)a.scales, (const float4*)a.rotations, a.radii,
        (const float4*)(a.geom + a.gl.surfel_rec), (const uint8_t*)(a.geom + a.gl.clamped),
        (const float4*)(a.geom + a.gl.sgrad), a.dL_dmeans2D, a.dL_dcolors, a.dL_dopacity, a.dL_dmeans3D,
        a.dL_dtransMat, a.dL_dsh, (float2*)a.dL_dscales, (float4*)a.dL_drotations);
    sr_count_launch();
    return cudaGetLastError();
}
