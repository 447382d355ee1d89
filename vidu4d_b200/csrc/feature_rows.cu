// feature_rows.cu -- Stage 3's per-surfel feature rows, forward and backward (DESIGN.md section 3.5d): for every frame m
// and surfel p the (Cf + 6)-wide row [regist (Cf) | flow / s (2) | normal (3) | Gaussian-bone density (1)] that the
// rasterizer composites next to the colour, with the flow scale s and the density as outputs of their own.
//
// Replaces (behaviour, not code) the reference's PyTorch statements
//   lab4d/nnutils/deformable_gaussian.py:1106-1182   query_field: the rows, the normal, the flow and its scale
//   lab4d/nnutils/deformable_gaussian.py:817-883     compute_flow: pi(K_m', x_m') - pi(K_m, x_m), m' = m xor 1
//   lab4d/nnutils/deformable_gaussian.py:789-805     flip_pair (a single frame is its own pair: flow 0)
//   lab4d/nnutils/deformable_gaussian.py:1742-1769   compute_gauss_density: exp(logibeta) * density
//   lab4d/nnutils/warping.py:463-495                 get_gauss_density: max_b exp(-0.5 |x - c_b|^2 / 0.01^2)
//   lab4d/utils/transforms.py:28-40                  get_xyz_bone_distance, c_b = translation of the rest bone
//   lab4d/utils/quat_transform.py:259-276            quaternion_apply (no normalisation: |q|^2 scales the result)
// which builds (P,B,3) differences for the density, repeats the camera quaternions over (M,P,4), and runs two batched
// 3x3 matmuls, four flip_pairs, a global max / min and a cat per frame, plus the autograd of all of them.
//
// Three quirks of the reference are reproduced, not fixed:
//   1. the normal's axis is the arg-min of the surfel's TWO tangent scales (first on ties): e_x or e_y, never e_z;
//   2. rot_cam already holds the camera rotation and the camera quaternion is applied again;
//   3. s = max(max(flow), |min(flow)|) + 1e-6 is not detached: its gradient reaches the flow, split over tied extreme
//      elements the way torch's autograd splits it.
//
// frows_absmax  one thread per surfel: max |flow| over all frames as an atomicMax on the bit pattern of a non-negative
//               float (deterministic; a NaN's pattern exceeds +inf's, so NaN wins as it does in torch.max).
// frows_fwd     one thread per surfel, loops over the frames: the regist row, xyz and the two scales are read once, the
//               B bone centres sit in shared memory.  Writes rows (M,P,Cf+6), density (P,), s, and counts the flow
//               values equal to +max|flow| and -max|flow| (the tied extremes the backward routes s's gradient to).
// frows_bwd_sum one thread per surfel: sum of g_row_flow * flow, the part of dL/ds that comes through the rows.
// frows_bwd     one thread per surfel, loops over the frames: dL/dxyz_cam of frame m and of its partner m xor 1 are both
//               computed by the thread, so everything per surfel is written directly, without atomics; the gradients of
//               the camera quaternions, the bone centres and exp(logibeta) are reduced warp -> shared memory -> one
//               global atomic per value and CTA.
//
// Every arithmetic step that decides a tie (the projection, the flow, the density scores) uses explicit-rounding
// intrinsics, so the three kernels that recompute the flow agree bit for bit whatever FMA contraction would do.
#include "warp_common.cuh"

namespace {

constexpr int FR_THREADS = 256;
constexpr int FR_M_MAX = 1024;            // g_cam_q of every frame is accumulated in shared memory
constexpr float FR_R2 = 1e-4f;            // 0.01^2, the Gaussian bones' radius squared (warping.py:480), as fp32
constexpr float FR_EPS = 1e-6f;           // added to the flow scale (deformable_gaussian.py:1178)

struct FrDims {
    int P, M, B, Cf;
    int vec;                               // Cf even and every row pointer 8-byte aligned: float2 row accesses
};

// pi(K, x) = (K x)[0:2] / (K x)[2], all three rows of K, no epsilon (deformable_gaussian.py:841-843)
struct Proj { float u0, u1, v0, v1, v2; };
__device__ __forceinline__ Proj project(const float* __restrict__ K, const float* __restrict__ x) {
    const float x0 = __ldg(x), x1 = __ldg(x + 1), x2 = __ldg(x + 2);
    auto row = [&](int i) {
        return __fadd_rn(__fadd_rn(__fmul_rn(__ldg(K + 3 * i), x0), __fmul_rn(__ldg(K + 3 * i + 1), x1)), __fmul_rn(__ldg(K + 3 * i + 2), x2));
    };
    Proj r;
    r.v0 = row(0); r.v1 = row(1); r.v2 = row(2);
    r.u0 = __fdiv_rn(r.v0, r.v2); r.u1 = __fdiv_rn(r.v1, r.v2);
    return r;
}

// vjp of pi: g_x = K^T g_v, g_v = (g0 / v2, g1 / v2, -(g0 u0 + g1 u1) / v2)
__device__ __forceinline__ void project_vjp(const float* __restrict__ K, const Proj& p, float g0, float g1, float* __restrict__ gx) {
    const float gv0 = g0 / p.v2, gv1 = g1 / p.v2, gv2 = -(g0 * p.u0 + g1 * p.u1) / p.v2;
#pragma unroll
    for (int j = 0; j < 3; j++) gx[j] = __ldg(K + j) * gv0 + __ldg(K + 3 + j) * gv1 + __ldg(K + 6 + j) * gv2;
}

// the partner frame of the pair that starts at m (a single frame pairs with itself)
__device__ __forceinline__ int partner(int m, int M) { return M == 1 ? m : m + 1; }

// max_b exp(-0.5 |x - c_b|^2 / 0.01^2) and its first arg-max (torch's max(-1)); a NaN score wins, as in torch
__device__ __forceinline__ float gauss_score(const float* __restrict__ c, int B, float x0, float x1, float x2, int& arg) {
    float best = 0.f;
    arg = 0;
    for (int b = 0; b < B; b++) {
        const float d0 = __fsub_rn(x0, c[3 * b]), d1 = __fsub_rn(x1, c[3 * b + 1]), d2 = __fsub_rn(x2, c[3 * b + 2]);
        const float r2 = __fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
        const float v = expf(__fmul_rn(-0.5f, __fdiv_rn(r2, FR_R2)));
        if (b == 0 || v > best || (v != v && best == best)) { best = v; arg = b; }
    }
    return best;
}

// reference quirk 1: e_x or e_y, whichever tangent scale is smaller (e_x on ties; a NaN scale is the minimum, as in torch)
__device__ __forceinline__ int short_axis(const float* __restrict__ scaling, size_t p) {
    const float s0 = __ldg(scaling + 2 * p), s1 = __ldg(scaling + 2 * p + 1);
    return (s1 < s0 || (s1 != s1 && s0 == s0)) ? 1 : 0;
}

__device__ __forceinline__ Q4 ld4(const float* __restrict__ q) { return {__ldg(q), __ldg(q + 1), __ldg(q + 2), __ldg(q + 3)}; }

__global__ void __launch_bounds__(FR_THREADS)
frows_absmax_kernel(const FrDims d, const float* __restrict__ xyz_cam, const float* __restrict__ Kmat, uint32_t* __restrict__ aux) {
    __shared__ uint32_t smax;
    if (threadIdx.x == 0) smax = 0u;
    __syncthreads();
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t mx = 0u;
    if (p < d.P) {
        for (int m = 0; m < d.M; m += 2) {            // flow of frame m + 1 is exactly minus that of frame m
            const int m1 = partner(m, d.M);
            const Proj a = project(Kmat + 9 * m, xyz_cam + 3 * ((size_t)m * d.P + p));
            const Proj b = project(Kmat + 9 * m1, xyz_cam + 3 * ((size_t)m1 * d.P + p));
            mx = max(mx, __float_as_uint(fabsf(__fsub_rn(b.u0, a.u0))));
            mx = max(mx, __float_as_uint(fabsf(__fsub_rn(b.u1, a.u1))));
        }
    }
    mx = __reduce_max_sync(0xffffffffu, mx);
    if ((threadIdx.x & 31) == 0) atomicMax(&smax, mx);
    __syncthreads();
    if (threadIdx.x == 0 && smax) atomicMax(aux, smax);
}

__global__ void __launch_bounds__(FR_THREADS)
frows_fwd_kernel(const FrDims d, const float* __restrict__ regist, const float* __restrict__ xyz, const float* __restrict__ scaling,
                 const float* __restrict__ xyz_cam, const float* __restrict__ rot_cam, const float* __restrict__ Kmat,
                 const float* __restrict__ cam_q, const float* __restrict__ centres, const float* __restrict__ beta,
                 float* __restrict__ rows, float* __restrict__ density, float* __restrict__ flow_scale, uint32_t* __restrict__ aux) {
    extern __shared__ float sc[];                     // centres [B*3]
    for (int i = threadIdx.x; i < d.B * 3; i += blockDim.x) sc[i] = __ldg(centres + i);
    __syncthreads();
    const float sm = __uint_as_float(aux[0]);         // max |flow|, frows_absmax
    const float s = __fadd_rn(sm, FR_EPS);
    if (blockIdx.x == 0 && threadIdx.x == 0) *flow_scale = s;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t hi = 0u, lo = 0u;
    if (p < d.P) {
        const int P = d.P, M = d.M, Cf = d.Cf, W = Cf + 6;
        const size_t ps = p;
        int arg;
        const float dens = __fmul_rn(gauss_score(sc, d.B, __ldg(xyz + 3 * ps), __ldg(xyz + 3 * ps + 1), __ldg(xyz + 3 * ps + 2), arg),
                                     __ldg(beta));
        density[ps] = dens;
        const int ax = short_axis(scaling, ps);
        // the regist row, read once, into every frame's row
        if (d.vec) {
            for (int j = 0; j < Cf; j += 2) {
                const float2 v = *reinterpret_cast<const float2*>(regist + ps * Cf + j);
                for (int m = 0; m < M; m++) *reinterpret_cast<float2*>(rows + ((size_t)m * P + ps) * W + j) = v;
            }
        } else {
            for (int j = 0; j < Cf; j++) {
                const float v = __ldg(regist + ps * Cf + j);
                for (int m = 0; m < M; m++) rows[((size_t)m * P + ps) * W + j] = v;
            }
        }
        auto emit = [&](int m, float f0, float f1) {
            hi += (f0 == sm) + (f1 == sm);
            lo += (f0 == -sm) + (f1 == -sm);
            const size_t n = (size_t)m * P + ps;
            float v0, v1, v2, n0, n1, n2;
            qrot(ld4(rot_cam + 4 * n), ax == 0 ? 1.f : 0.f, ax == 1 ? 1.f : 0.f, 0.f, v0, v1, v2);
            qrot(ld4(cam_q + 4 * m), v0, v1, v2, n0, n1, n2);                  // reference quirk 2
            float* r = rows + n * W + Cf;
            const float t[6] = {__fdiv_rn(f0, s), __fdiv_rn(f1, s), n0, n1, n2, dens};
            if (d.vec) {
#pragma unroll
                for (int k = 0; k < 3; k++) reinterpret_cast<float2*>(r)[k] = make_float2(t[2 * k], t[2 * k + 1]);
            } else {
#pragma unroll
                for (int k = 0; k < 6; k++) r[k] = t[k];
            }
        };
        for (int m = 0; m < M; m += 2) {
            const int m1 = partner(m, M);
            const Proj a = project(Kmat + 9 * m, xyz_cam + 3 * ((size_t)m * P + ps));
            const Proj b = project(Kmat + 9 * m1, xyz_cam + 3 * ((size_t)m1 * P + ps));
            const float f0 = __fsub_rn(b.u0, a.u0), f1 = __fsub_rn(b.u1, a.u1);
            emit(m, f0, f1);
            if (m1 != m) emit(m1, -f0, -f1);                                   // a - b == -(b - a) exactly
        }
    }
    hi = __reduce_add_sync(0xffffffffu, hi);
    lo = __reduce_add_sync(0xffffffffu, lo);
    if ((threadIdx.x & 31) == 0 && (hi | lo)) { atomicAdd(aux + 1, hi); atomicAdd(aux + 2, lo); }
}

// sum over the batch of g_row_flow * flow into *acc (dL/ds through the rows is -acc / s^2)
__global__ void __launch_bounds__(FR_THREADS)
frows_bwd_sum_kernel(const FrDims d, const float* __restrict__ xyz_cam, const float* __restrict__ Kmat, const float* __restrict__ g_rows,
                     float* __restrict__ acc) {
    __shared__ float wsum[FR_THREADS / 32];
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    float sum = 0.f;
    if (p < d.P) {
        const int P = d.P, M = d.M, W = d.Cf + 6;
        for (int m = 0; m < M; m += 2) {
            const int m1 = partner(m, M);
            const Proj a = project(Kmat + 9 * m, xyz_cam + 3 * ((size_t)m * P + p));
            const Proj b = project(Kmat + 9 * m1, xyz_cam + 3 * ((size_t)m1 * P + p));
            const float f0 = __fsub_rn(b.u0, a.u0), f1 = __fsub_rn(b.u1, a.u1);
            const float* g = g_rows + ((size_t)m * P + p) * W + d.Cf;
            sum += __ldg(g) * f0 + __ldg(g + 1) * f1;
            if (m1 != m) {
                const float* h = g_rows + ((size_t)m1 * P + p) * W + d.Cf;
                sum -= __ldg(h) * f0 + __ldg(h + 1) * f1;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < FR_THREADS / 32; w++) t += wsum[w];
        if (t != 0.f) atomicAdd(acc, t);
    }
}

// g_tables: g_cam_q [M*4] | g_centres [B*3] | g_beta [1] | sum of g_row_flow * flow [1] (frows_bwd_sum)
__global__ void __launch_bounds__(FR_THREADS)
frows_bwd_kernel(const FrDims d, const float* __restrict__ xyz, const float* __restrict__ scaling, const float* __restrict__ xyz_cam,
                 const float* __restrict__ rot_cam, const float* __restrict__ Kmat, const float* __restrict__ cam_q,
                 const float* __restrict__ centres, const float* __restrict__ beta, const float* __restrict__ flow_scale,
                 const uint32_t* __restrict__ aux, const float* __restrict__ g_rows, const float* __restrict__ g_density,
                 const float* __restrict__ g_flow_scale, float* __restrict__ g_regist, float* __restrict__ g_xyz,
                 float* __restrict__ g_xyz_cam, float* __restrict__ g_rot_cam, float* __restrict__ g_tables) {
    extern __shared__ float sh[];
    const int P = d.P, M = d.M, B = d.B, Cf = d.Cf, W = Cf + 6;
    const int ntab = M * 4 + B * 3 + 1;
    float* sc = sh;                                    // centres [B*3]
    float* gt = sh + B * 3;                            // g_cam_q [M*4] | g_centres [B*3] | g_beta
    for (int i = threadIdx.x; i < B * 3; i += blockDim.x) sc[i] = __ldg(centres + i);
    for (int i = threadIdx.x; i < ntab; i += blockDim.x) gt[i] = 0.f;
    __syncthreads();
    float* gcq = gt;
    float* gcen = gt + M * 4;
    float* gbeta = gcen + B * 3;

    // dL/ds = the caller's g_s + the rows' -sum(g * flow) / s^2, routed as torch's autograd routes
    // s = maximum(max(flow), abs(min(flow))) + eps: maximum halves on a tie, max / min spread evenly over tied elements,
    // abs multiplies by sign(min).  max(flow) = sm iff some element equals +sm, |min(flow)| = sm iff some equals -sm.
    const float s = __ldg(flow_scale), sm = __uint_as_float(__ldg(aux));
    const uint32_t hi = __ldg(aux + 1), lo = __ldg(aux + 2);
    const float G = (g_flow_scale ? __ldg(g_flow_scale) : 0.f) + -__ldg(g_tables + ntab) / __fmul_rn(s, s);
    const float g_hi = hi ? (lo ? G * 0.5f : G) / (float)hi : 0.f;
    const float sgn_min = sm > 0.f ? -1.f : 0.f;                               // sign(min(flow)) = sign(-sm)
    const float g_lo = lo ? ((hi ? G * 0.5f : G) * sgn_min) / (float)lo : 0.f;

    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < P;                           // dead lanes take part in the warp sums with zeros
    const size_t ps = live ? (size_t)p : 0;
    const int ax = short_axis(scaling, ps);
    auto gflow = [&](size_t n, float f, int c) {
        return __fdiv_rn(__ldg(g_rows + n * W + Cf + c), s) + (f == sm ? g_hi : 0.f) + (f == -sm ? g_lo : 0.f);
    };
    float g_dens = (live && g_density) ? __ldg(g_density + ps) : 0.f;
    auto normal_vjp = [&](int m, size_t n) {
        const float* g = g_rows + n * W + Cf + 2;
        const Q4 r = ld4(rot_cam + 4 * n), cq = ld4(cam_q + 4 * m);
        const float a0 = ax == 0 ? 1.f : 0.f, a1 = ax == 1 ? 1.f : 0.f;
        float v0, v1, v2, gv0, gv1, gv2, ga0, ga1, ga2;
        qrot(r, a0, a1, 0.f, v0, v1, v2);
        Q4 gcq_m, gr;
        qrot_vjp(cq, v0, v1, v2, __ldg(g), __ldg(g + 1), __ldg(g + 2), gcq_m, gv0, gv1, gv2);
        qrot_vjp(r, a0, a1, 0.f, gv0, gv1, gv2, gr, ga0, ga1, ga2);
        if (live) {
            float* o = g_rot_cam + 4 * n;
            o[0] = gr.w; o[1] = gr.x; o[2] = gr.y; o[3] = gr.z;
            g_dens += __ldg(g_rows + n * W + Cf + 5);
        }
        acc_q(gcq + 4 * m, live ? gcq_m : Q4{0.f, 0.f, 0.f, 0.f});
    };
    for (int m = 0; m < M; m += 2) {
        const int m1 = partner(m, M);
        const size_t n0 = (size_t)m * P + ps, n1 = (size_t)m1 * P + ps;
        const Proj a = project(Kmat + 9 * m, xyz_cam + 3 * n0);
        const Proj b = project(Kmat + 9 * m1, xyz_cam + 3 * n1);
        const float f0 = __fsub_rn(b.u0, a.u0), f1 = __fsub_rn(b.u1, a.u1);
        // flow[m] = pi_m1 - pi_m, flow[m1] = pi_m - pi_m1:  dL/dpi_m = g_flow[m1] - g_flow[m], dL/dpi_m1 = its negative
        const float h0 = gflow(n0, f0, 0), h1 = gflow(n0, f1, 1);
        const float k0 = m1 != m ? gflow(n1, -f0, 0) : h0, k1 = m1 != m ? gflow(n1, -f1, 1) : h1;
        float gx[3];
        if (live) {
            project_vjp(Kmat + 9 * m, a, k0 - h0, k1 - h1, gx);
            g_xyz_cam[3 * n0] = gx[0]; g_xyz_cam[3 * n0 + 1] = gx[1]; g_xyz_cam[3 * n0 + 2] = gx[2];
            if (m1 != m) {
                project_vjp(Kmat + 9 * m1, b, h0 - k0, h1 - k1, gx);
                g_xyz_cam[3 * n1] = gx[0]; g_xyz_cam[3 * n1 + 1] = gx[1]; g_xyz_cam[3 * n1 + 2] = gx[2];
            }
        }
        normal_vjp(m, n0);
        if (m1 != m) normal_vjp(m1, n1);
    }
    // regist: the sum over the frames' rows
    if (live) {
        if (d.vec) {
            for (int j = 0; j < Cf; j += 2) {
                float2 t = make_float2(0.f, 0.f);
                for (int m = 0; m < M; m++) {
                    const float2 v = *reinterpret_cast<const float2*>(g_rows + ((size_t)m * P + ps) * W + j);
                    t.x += v.x; t.y += v.y;
                }
                *reinterpret_cast<float2*>(g_regist + ps * Cf + j) = t;
            }
        } else {
            for (int j = 0; j < Cf; j++) {
                float t = 0.f;
                for (int m = 0; m < M; m++) t += __ldg(g_rows + ((size_t)m * P + ps) * W + j);
                g_regist[ps * Cf + j] = t;
            }
        }
    }
    // density = beta * exp(u), u = -0.5 * (|x - c|^2 / r^2), at the first arg-max bone (no gradient once it underflows)
    const float x0 = __ldg(xyz + 3 * ps), x1 = __ldg(xyz + 3 * ps + 1), x2 = __ldg(xyz + 3 * ps + 2);
    int arg;
    const float score = gauss_score(sc, B, x0, x1, x2, arg);
    acc_table(gbeta, live ? g_dens * score : 0.f);
    const float g_r2 = ((-0.5f * ((g_dens * __ldg(beta)) * score)) / FR_R2) * 2.f;
    const float gd[3] = {(x0 - sc[3 * arg]) * g_r2, (x1 - sc[3 * arg + 1]) * g_r2, (x2 - sc[3 * arg + 2]) * g_r2};
    if (live) {
        g_xyz[3 * ps] = gd[0]; g_xyz[3 * ps + 1] = gd[1]; g_xyz[3 * ps + 2] = gd[2];
#pragma unroll
        for (int k = 0; k < 3; k++)
            if (gd[k] != 0.f) atomicAdd(gcen + 3 * arg + k, -gd[k]);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < ntab; i += blockDim.x)
        if (gt[i] != 0.f) atomicAdd(g_tables + i, gt[i]);
}

int check_rows(int32_t P, int32_t M, int32_t B, int32_t Cf) {
    if (P < 0) return sr_fail(SR_EINVAL, "P must be >= 0, got %d", P);
    if (M < 1 || (M > 1 && M % 2) || M > FR_M_MAX)
        return sr_fail(SR_EINVAL, "M must be 1 or even (frames are flow pairs 2k, 2k+1) and at most %d, got %d", FR_M_MAX, M);
    if (B < 1 || B > 64) return sr_fail(SR_EINVAL, "B must be in [1, 64], got %d", B);
    if (Cf < 0 || Cf + 6 > 32) return sr_fail(SR_EINVAL, "Cf must be in [0, 26] (rows of Cf + 6 <= 32 channels), got %d", Cf);
    return 0;
}

int row_vec(int Cf, const void* a, const void* b) {
    return Cf % 2 == 0 && ((uintptr_t)a & 7) == 0 && ((uintptr_t)b & 7) == 0;
}

}  // namespace

extern "C" {

SR_API int sr_feature_rows_forward(int32_t P, int32_t M, int32_t B, int32_t Cf, const float* regist, const float* xyz,
                                   const float* scaling, const float* xyz_cam, const float* rot_cam, const float* Kmat,
                                   const float* cam_q, const float* centres, const float* beta, float* rows, float* density,
                                   float* flow_scale, uint32_t* aux, void* stream_) {
    if (int rc = check_rows(P, M, B, Cf)) return rc;
    const bool per_surfel = P > 0;                    // an empty surfel set may come with NULL per-surfel arrays
    if ((per_surfel && ((Cf > 0 && !regist) || !xyz || !scaling || !xyz_cam || !rot_cam || !rows || !density)) || !Kmat || !cam_q ||
        !centres || !beta || !flow_scale || !aux)
        return sr_fail(SR_EINVAL, "sr_feature_rows_forward: a required pointer is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    if (cudaMemsetAsync(aux, 0, 3 * sizeof(uint32_t), s) != cudaSuccess) return SR_ECUDA;
    const FrDims d{P, M, B, Cf, row_vec(Cf, regist, rows)};
    const int blocks = (P + FR_THREADS - 1) / FR_THREADS;
    int launches = 1;
    if (P > 0) {
        ProfileScope ps("frows_absmax", s);
        frows_absmax_kernel<<<blocks, FR_THREADS, 0, s>>>(d, xyz_cam, Kmat, aux);
        launches++;
    }
    {
        ProfileScope ps("frows_fwd", s);                // at least one block: it also writes the flow scale
        frows_fwd_kernel<<<blocks > 0 ? blocks : 1, FR_THREADS, B * 3 * sizeof(float), s>>>(d, regist, xyz, scaling, xyz_cam, rot_cam,
                                                                                          Kmat, cam_q, centres, beta, rows, density,
                                                                                          flow_scale, aux);
    }
    sr_count_launch(launches);
    return cudaGetLastError() == cudaSuccess ? 0 : SR_ECUDA;
}

SR_API int sr_feature_rows_backward(int32_t P, int32_t M, int32_t B, int32_t Cf, const float* xyz, const float* scaling,
                                    const float* xyz_cam, const float* rot_cam, const float* Kmat, const float* cam_q,
                                    const float* centres, const float* beta, const float* flow_scale, const uint32_t* aux,
                                    const float* g_rows, const float* g_density, const float* g_flow_scale, float* g_regist,
                                    float* g_xyz, float* g_xyz_cam, float* g_rot_cam, float* g_tables, void* stream_) {
    if (int rc = check_rows(P, M, B, Cf)) return rc;
    const bool per_surfel = P > 0;
    if ((per_surfel && (!xyz || !scaling || !xyz_cam || !rot_cam || !g_rows || (Cf > 0 && !g_regist) || !g_xyz || !g_xyz_cam ||
                        !g_rot_cam)) || !Kmat || !cam_q || !centres || !beta || !flow_scale || !aux || !g_tables)
        return sr_fail(SR_EINVAL, "sr_feature_rows_backward: a required pointer is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    const int ntab = M * 4 + B * 3 + 1;
    if (cudaMemsetAsync(g_tables, 0, (ntab + 1) * sizeof(float), s) != cudaSuccess) return SR_ECUDA;
    if (P == 0) return 0;
    const FrDims d{P, M, B, Cf, row_vec(Cf, g_rows, g_regist)};
    const int blocks = (P + FR_THREADS - 1) / FR_THREADS;
    {
        ProfileScope ps("frows_bwd_sum", s);
        frows_bwd_sum_kernel<<<blocks, FR_THREADS, 0, s>>>(d, xyz_cam, Kmat, g_rows, g_tables + ntab);
    }
    {
        ProfileScope ps("frows_bwd", s);
        const size_t smem = (size_t)(B * 3 + ntab) * sizeof(float);
        frows_bwd_kernel<<<blocks, FR_THREADS, smem, s>>>(d, xyz, scaling, xyz_cam, rot_cam, Kmat, cam_q, centres, beta, flow_scale,
                                                          aux, g_rows, g_density, g_flow_scale, g_regist, g_xyz, g_xyz_cam,
                                                          g_rot_cam, g_tables);
    }
    sr_count_launch(2);
    return cudaGetLastError() == cudaSuccess ? 0 : SR_ECUDA;
}

}  // extern "C"
