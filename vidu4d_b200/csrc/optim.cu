// optim.cu -- optimizer-side kernels over the FLAT surfel parameter buffer (SURVEY.md section 8(f) row N4).
//
// The Stage-3 surfel parameters (xyz 3, f_dc 3, f_rest 45, opacity 1, scaling 2, rotation 4 floats per surfel;
// lab4d/engine/trainer.py:243-251) live back to back in ONE fp32 buffer -- the same layout the gradient all-reduce runs
// over (vidu4d_b200/distributed.py FlatGrads) -- so that
//   * the Adam update of all six parameter groups is ONE kernel over that buffer (the reference steps a
//     torch.optim.Adam with seven param groups, trainer.py:253, eps = 1e-15), with the 1/(frames x ranks) gradient
//     averaging folded in, and
//   * densify / prune (gs/scene/gaussian_model.py:291-446: _prune_optimizer, cat_tensors_to_optimizer,
//     densification_postfix, densify_and_split, densify_and_clone, prune_points) becomes ONE gather kernel that writes the
//     new parameter, exp_avg and exp_avg_sq buffers from a source-index list, instead of ~60 torch cat / index /
//     nn.Parameter re-creations per call.
// Semantics are torch.optim.Adam's (amsgrad off, no weight decay; its default foreach path on CUDA) and the reference's
// row-wise copy rules.  The Adam constants are formed as torch forms them from its double betas and rates: 1 - beta in
// double rounded once, beta^t and lr / (1 - beta1^t) in double; every element operation is torch's, rounded where torch
// rounds.  Both moments equal torch's bit for bit; so do the parameters when the rates are fp32 values.  Both entry
// points take the rates as fp32, so a rate that is not one is rounded first (a step size within 3 u of torch's).
//
// The per-step optimizer state can also live on the device (include/surfel_optim.h): a group-wise float64 sum of squares
// of the gradient buffer gives torch.nn.utils.clip_grad_norm_'s coefficient in a one-CTA finish, and the Adam pass reads
// its step count, learning rates and that coefficient from device memory, so a replayed CUDA graph steps as the
// reference does (lab4d/engine/trainer.py:547, 589-591) without a re-capture.
//
// The densification statistics of a batch of M frames (trainer.py:553-560, gaussian_model.py:450-452) are one kernel
// too: sr_densify_stats reads the batched backward's (M,P,3) screen-space proxy gradient and (M,P) radii once.
#include "common.cuh"
#include "../../include/surfel_optim.h"

namespace {

constexpr int MAXG = 8;
struct AdamGroups {
    int n;
    long long begin[MAXG + 1];     // element offsets of the groups inside the flat buffer; begin[n] = total
    float step_size[MAXG];         // sr_adam_flat: (float)(lr / (1 - beta1^t)), formed in double on the host
};

// sr_adam_flat_state's device state; unused (all NULL) in sr_adam_flat's instantiation
struct AdamDeviceState {
    const float* lr;               // [n_groups]
    const long long* step;         // already incremented: the 1-based number of this step
    const float* coef;             // clip coefficient, or NULL for 1
};

// torch/optim/adam.py _multi_tensor_adam's scalars, all in double: bias_correction1 = 1 - beta1 ** t,
// step_size = lr / bias_correction1, bias_correction2_sqrt = (1 - beta2 ** t) ** 0.5; the kernels get them rounded to fp32
// as torch's foreach ops do.  beta^1 is beta exactly, without a pow that the device library may round differently from
// the host's: at t = 1 two of the Stage-3 rates sit within an ulp of a rounding boundary of lr / (1 - beta1)
__host__ __device__ __forceinline__ double adam_pow(double beta, long long step) { return step == 1 ? beta : pow(beta, (double)step); }
__host__ __device__ __forceinline__ double adam_bc1(double beta1, long long step) { return 1.0 - adam_pow(beta1, step); }
__host__ __device__ __forceinline__ float adam_sqrt_bc2(double beta2, long long step) {
    return (float)sqrt(1.0 - adam_pow(beta2, step));
}

// DEVICE_STATE = false: sr_adam_flat, every scalar a launch argument.  DEVICE_STATE = true: sr_adam_flat_state, the step,
// rates and clip coefficient read from S (sqrt_bc2 / G.step_size are then ignored).
template <bool DEVICE_STATE>
__global__ void __launch_bounds__(256)
adam_flat_kernel(const AdamGroups G, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                 float* __restrict__ v, double beta1, double beta2, float eps, float sqrt_bc2, float grad_scale,
                 const AdamDeviceState S) {
    float steps[MAXG], coef = 1.0f;
    if constexpr (DEVICE_STATE) {
        // thread q < MAXG forms group q's step size, thread MAXG the second bias correction (float64 pow each); the rest
        // read them from shared memory
        __shared__ float sc[MAXG + 2];
        const long long t = *S.step;
        if (threadIdx.x < MAXG) sc[threadIdx.x] = threadIdx.x < G.n ? (float)((double)S.lr[threadIdx.x] / adam_bc1(beta1, t)) : 0.0f;
        if (threadIdx.x == MAXG) sc[MAXG] = adam_sqrt_bc2(beta2, t);
        if (threadIdx.x == MAXG + 1) sc[MAXG + 1] = S.coef ? *S.coef : 1.0f;
        __syncthreads();
        sqrt_bc2 = sc[MAXG]; coef = sc[MAXG + 1];
#pragma unroll
        for (int q = 0; q < MAXG; q++) steps[q] = sc[q];
    }
    // torch's foreach scalars are fp32 (opmath) values: 1 - beta rounded once from double, beta2 rounded
    const float c1 = (float)(1.0 - beta1), b2 = (float)beta2, c2 = (float)(1.0 - beta2);
    const long long total = G.begin[G.n];
    for (long long i = (long long)blockIdx.x * 1024 + threadIdx.x * 4; i < total; i += (long long)gridDim.x * 1024) {
        // four consecutive elements; a group boundary can fall inside them, so the rate is looked up per element
        const bool vec = i + 3 < total;
        float4 pp, gg, mm, vv;
        if (vec) {
            pp = *reinterpret_cast<const float4*>(p + i); gg = *reinterpret_cast<const float4*>(g + i);
            mm = *reinterpret_cast<const float4*>(m + i); vv = *reinterpret_cast<const float4*>(v + i);
        } else {
            float t[4][4] = {};
            for (int k = 0; k < 4 && i + k < total; k++) { t[0][k] = p[i + k]; t[1][k] = g[i + k]; t[2][k] = m[i + k]; t[3][k] = v[i + k]; }
            pp = make_float4(t[0][0], t[0][1], t[0][2], t[0][3]); gg = make_float4(t[1][0], t[1][1], t[1][2], t[1][3]);
            mm = make_float4(t[2][0], t[2][1], t[2][2], t[2][3]); vv = make_float4(t[3][0], t[3][1], t[3][2], t[3][3]);
        }
        float* P4 = &pp.x; float* G4 = &gg.x; float* M4 = &mm.x; float* V4 = &vv.x;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const long long e = i + k;
            float step = DEVICE_STATE ? steps[0] : G.step_size[0];
#pragma unroll
            for (int q = 1; q < MAXG; q++) if (q < G.n && e >= G.begin[q]) step = DEVICE_STATE ? steps[q] : G.step_size[q];
            // (g * grad_scale) * coef, each product rounded: the averaging, then clip_grad_norm_'s in-place multiply
            const float gr = __fmul_rn(__fmul_rn(G4[k], grad_scale), coef);
            // torch's _multi_tensor_adam, one foreach op after another, each rounded to fp32:
            //   exp_avg.lerp_(grad, 1 - beta1)              ATen lerp: self + w (end - self) for |w| < 0.5, else
            //                                               end - (end - self)(1 - w), each one FMA
            //   exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)        addcmul: fma(value, grad * grad, self)
            //   denom = exp_avg_sq.sqrt() / bias_correction2_sqrt + eps
            //   param.addcdiv_(exp_avg, denom, -step_size)                    addcdiv: fma(value, exp_avg / denom, param)
            const float d = __fsub_rn(gr, M4[k]);
            M4[k] = c1 < 0.5f ? __fmaf_rn(c1, d, M4[k]) : __fmaf_rn(-d, __fsub_rn(1.0f, c1), gr);
            V4[k] = __fmaf_rn(c2, __fmul_rn(gr, gr), __fmul_rn(V4[k], b2));
            const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(V4[k]), sqrt_bc2), eps);
            P4[k] = __fmaf_rn(-step, __fdiv_rn(M4[k], denom), P4[k]);
        }
        if (vec) {
            *reinterpret_cast<float4*>(p + i) = pp; *reinterpret_cast<float4*>(m + i) = mm; *reinterpret_cast<float4*>(v + i) = vv;
        } else {
            for (int k = 0; k < 4 && i + k < total; k++) { p[i + k] = P4[k]; m[i + k] = M4[k]; v[i + k] = V4[k]; }
        }
    }
}

// new[s] <- old[src[s]] for every parameter group and both Adam moments.  kind[s]: 0 = the surfel survives (state kept),
// 1 = clone (fresh state), 2 = split child (fresh state; xyz and scaling come from the override arrays).
struct CompactGroups {
    int n;
    int width[MAXG];               // floats per surfel of each group
    long long old_begin[MAXG], new_begin[MAXG];
    int xyz_group, scaling_group;  // which groups the split overrides replace (-1: none)
};

__global__ void __launch_bounds__(256)
compact_kernel(const CompactGroups G, int P_new, const int* __restrict__ src, const uint8_t* __restrict__ kind,
               const int* __restrict__ child_slot, const float* __restrict__ child_xyz, const float* __restrict__ child_scaling,
               const float* __restrict__ p_old, const float* __restrict__ m_old, const float* __restrict__ v_old,
               float* __restrict__ p_new, float* __restrict__ m_new, float* __restrict__ v_new) {
    // one warp per destination surfel and group element range: lanes stride over the (up to 45) floats of a group row
    const int s = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (s >= P_new) return;
    const int lane = threadIdx.x & 31;
    const int from = src[s];
    const int k = kind[s];
    for (int q = 0; q < G.n; q++) {
        const int w = G.width[q];
        const float* po = p_old + G.old_begin[q] + (long long)from * w;
        const float* mo = m_old + G.old_begin[q] + (long long)from * w;
        const float* vo = v_old + G.old_begin[q] + (long long)from * w;
        float* pn = p_new + G.new_begin[q] + (long long)s * w;
        float* mn = m_new + G.new_begin[q] + (long long)s * w;
        float* vn = v_new + G.new_begin[q] + (long long)s * w;
        for (int e = lane; e < w; e += 32) {
            float val = po[e];
            if (k == 2 && q == G.xyz_group) val = child_xyz[(long long)child_slot[s] * 3 + e];
            if (k == 2 && q == G.scaling_group) val = child_scaling[(long long)child_slot[s] * w + e];
            pn[e] = val;
            mn[e] = k == 0 ? mo[e] : 0.f;
            vn[e] = k == 0 ? vo[e] : 0.f;
        }
    }
}

// ---- gradient norm (clip_grad_norm_) ----------------------------------------------------------------------------------
// The grid is a function of the buffer size alone (never of the device), so every rank of a multi-GPU run, holding the
// same all-reduced bytes, gets the same partials, the same sums and the same coefficient.
constexpr int NORM_THREADS = 256, NORM_MAX_CTAS = 1024;
struct GroupBounds {
    int n;
    long long begin[MAXG + 1];
};

int norm_ctas(long long total) {
    const long long c = (total + NORM_THREADS * 4 - 1) / (NORM_THREADS * 4);
    return (int)(c < NORM_MAX_CTAS ? c : NORM_MAX_CTAS);
}

// partials[q * gridDim.x + cta] = this CTA's float64 sum over group q of (g * grad_scale)^2.  The square of an fp32 value
// is exact in float64, so the only roundings are the float64 additions, each in an order fixed by the launch shape.
__global__ void __launch_bounds__(NORM_THREADS)
grad_sumsq_kernel(const GroupBounds G, const float* __restrict__ g, float grad_scale, double* __restrict__ partials) {
    const long long total = G.begin[G.n];
    double acc[MAXG];
#pragma unroll
    for (int q = 0; q < MAXG; q++) acc[q] = 0.0;
    // a thread's elements only move forward, so it runs one sum for the current group and banks it when a group ends
    int cq = 0;
    long long cend = G.begin[1];
    double run = 0.0;
    for (long long i = (long long)blockIdx.x * (NORM_THREADS * 4) + threadIdx.x * 4; i < total;
         i += (long long)gridDim.x * (NORM_THREADS * 4)) {
        float4 x4;
        if (i + 3 < total) {
            x4 = *reinterpret_cast<const float4*>(g + i);
        } else {
            float t[4] = {};
            for (int k = 0; k < 4 && i + k < total; k++) t[k] = g[i + k];
            x4 = make_float4(t[0], t[1], t[2], t[3]);
        }
        const float* X = &x4.x;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const long long e = i + k;
            if (e >= total) break;
            while (e >= cend) {           // groups may be empty and may start inside a float4
#pragma unroll
                for (int q = 0; q < MAXG; q++) if (q == cq) acc[q] += run;
                run = 0.0; cq++; cend = G.begin[cq + 1];
            }
            const double y = (double)(X[k] * grad_scale);
            run += y * y;
        }
    }
#pragma unroll
    for (int q = 0; q < MAXG; q++) if (q == cq) acc[q] += run;

    __shared__ double red[MAXG][NORM_THREADS / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int q = 0; q < MAXG; q++) {
        if (q >= G.n) break;
        double a = acc[q];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) red[q][warp] = a;
    }
    __syncthreads();
    if (threadIdx.x < G.n) {
        double t = 0.0;
#pragma unroll
        for (int w = 0; w < NORM_THREADS / 32; w++) t += red[threadIdx.x][w];
        partials[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = t;
    }
}

// One CTA: each group's partials summed in a fixed order, then the norm and torch's clip coefficient.
__global__ void __launch_bounds__(NORM_THREADS)
grad_norm_finish_kernel(int n, int parts, const double* __restrict__ partials, const float* __restrict__ extra_norms, int n_extra,
                        float max_norm, float* __restrict__ total_norm, float* __restrict__ clip_coef,
                        double* __restrict__ group_sumsq) {
    __shared__ double S[MAXG];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int q = warp; q < n; q += NORM_THREADS / 32) {
        double a = 0.0;
        for (int i = lane; i < parts; i += 32) a += partials[(size_t)q * parts + i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) S[q] = a;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        double t = 0.0;
        for (int q = 0; q < n; q++) {
            t += S[q];
            if (group_sumsq) group_sumsq[q] = S[q];
        }
        for (int e = 0; e < n_extra; e++) {
            const double x = extra_norms[e];
            t += x * x;
        }
        const float tot = (float)sqrt(t);
        // torch: max_norm / (total + 1e-6) is (total + 1e-6).reciprocal() * max_norm (Tensor.__rdiv__), all in fp32;
        // clamp(max=1) passes a NaN through
        const float c = (1.0f / (tot + 1e-6f)) * max_norm;
        *total_norm = tot;
        *clip_coef = c > 1.0f ? 1.0f : c;
    }
}

__global__ void adam_step_count_kernel(long long* step) { *step += 1; }

// ---- densification statistics (sr_densify_stats) ----------------------------------------------------------------------
// One thread per surfel walks the M frames in order, so each statistic is updated frame after frame exactly as M
// successive calls of the per-frame torch update would (no atomics: the bits depend on the inputs alone).
__global__ void __launch_bounds__(256)
densify_stats_kernel(int M, int P, const float* __restrict__ g, const int* __restrict__ radii, float grad_scale,
                     float* __restrict__ accum, float* __restrict__ denom, float* __restrict__ max_radii) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    float a = accum[i], d = denom[i], r = max_radii[i];
    for (int m = 0; m < M; m++) {
        const long long e = (long long)m * P + i;
        const int rad = radii[e];
        if (rad <= 0) continue;
        const float x = __fmul_rn(g[e * 3 + 0], grad_scale), y = __fmul_rn(g[e * 3 + 1], grad_scale),
                    z = __fmul_rn(g[e * 3 + 2], grad_scale);
        // torch.norm(dim=-1) over a row of 3 (ATen's NormTwoOps through gpu_reduce_kernel): two lanes share the row,
        // lane 0 sums elements 0 and 2, lane 1 holds element 1, then the lanes combine -- every square and sum rounded
        const float sq = __fadd_rn(__fadd_rn(__fmul_rn(x, x), __fmul_rn(z, z)), __fmul_rn(y, y));
        a = __fadd_rn(a, sqrtf(sq));
        d = __fadd_rn(d, 1.0f);
        r = fmaxf(r, (float)rad);
    }
    accum[i] = a; denom[i] = d; max_radii[i] = r;
}

// the group table both device-state entry points take: n_groups in [1, MAXG], begin[0] = 0, begin non-decreasing
int check_groups(const char* fn, int32_t n_groups, const int64_t* begin) {
    if (n_groups < 1 || n_groups > MAXG) return sr_fail(SR_EINVAL, "%s: n_groups must be in [1, %d], got %d", fn, MAXG, n_groups);
    if (!begin) return sr_fail(SR_EINVAL, "%s: begin is NULL", fn);
    if (begin[0] != 0) return sr_fail(SR_EINVAL, "%s: begin[0] must be 0, got %lld", fn, (long long)begin[0]);
    for (int i = 0; i < n_groups; i++)
        if (begin[i + 1] < begin[i])
            return sr_fail(SR_EINVAL, "%s: begin must be non-decreasing (begin[%d] = %lld > begin[%d] = %lld)", fn, i,
                           (long long)begin[i], i + 1, (long long)begin[i + 1]);
    return 0;
}

}  // namespace

extern "C" {

/* One Adam step over a flat buffer of `n_groups` back-to-back parameter groups (group g = elements [begin[g], begin[g+1])),
 * each with its own learning rate; torch.optim.Adam semantics (amsgrad off, weight_decay 0).  `step` is the 1-based step
 * count (bias correction); the betas are torch's double values; grad_scale multiplies every gradient first (1 / (frames x ranks) averaging).  All device
 * pointers, 16-byte aligned. */
SR_API int sr_adam_flat(int32_t n_groups, const int64_t* begin /* host, n_groups + 1 */, const float* lr /* host, n_groups */,
                        double beta1, double beta2, float eps, int64_t step, float grad_scale, float* params, const float* grads,
                        float* exp_avg, float* exp_avg_sq, void* stream_) {
    if (n_groups < 1 || n_groups > MAXG) return sr_fail(SR_EINVAL, "sr_adam_flat: n_groups must be in [1, %d], got %d", MAXG, n_groups);
    if (!begin || !lr || !params || !grads || !exp_avg || !exp_avg_sq) return sr_fail(SR_EINVAL, "sr_adam_flat: a required pointer is NULL");
    if (step < 1) return sr_fail(SR_EINVAL, "sr_adam_flat: step must be >= 1, got %lld", (long long)step);
    if (((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15)
        return sr_fail(SR_EINVAL, "sr_adam_flat: params, grads, exp_avg and exp_avg_sq must be 16-byte aligned");
    AdamGroups G{};
    G.n = n_groups;
    for (int i = 0; i <= n_groups; i++) G.begin[i] = begin[i];
    const double bc1 = adam_bc1(beta1, step);
    for (int i = 0; i < n_groups; i++) G.step_size[i] = (float)((double)lr[i] / bc1);
    const long long total = begin[n_groups];
    if (total <= 0) return 0;
    cudaStream_t s = (cudaStream_t)stream_;
    const long long blocks = (total + 1023) / 1024;
    ProfileScope ps("adam_flat", s);
    // grid-stride: at most 16 CTAs per SM of an H100 SXM (132 SMs)
    adam_flat_kernel<false><<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, s>>>(
        G, params, grads, exp_avg, exp_avg_sq, beta1, beta2, eps, adam_sqrt_bc2(beta2, step), grad_scale, AdamDeviceState{});
    return sr_launched(1, "sr_adam_flat");
}

SR_API int64_t sr_grad_norm_scratch_bytes(int32_t n_groups) {
    if (n_groups < 1 || n_groups > MAXG) return -1;
    return (int64_t)NORM_MAX_CTAS * n_groups * (int64_t)sizeof(double);
}

SR_API int sr_grad_norm_flat(int32_t n_groups, const int64_t* begin, const float* grads, float grad_scale, const float* extra_norms,
                             int32_t n_extra, float max_norm, float* total_norm, float* clip_coef, double* group_sumsq,
                             void* scratch, int64_t scratch_bytes, void* stream_) {
    int rc = check_groups("sr_grad_norm_flat", n_groups, begin);
    if (rc) return rc;
    if (!grads || !total_norm || !clip_coef || !scratch)
        return sr_fail(SR_EINVAL, "sr_grad_norm_flat: grads, total_norm, clip_coef and scratch must not be NULL");
    if ((uintptr_t)grads & 15) return sr_fail(SR_EINVAL, "sr_grad_norm_flat: grads must be 16-byte aligned");
    if ((uintptr_t)scratch & 7) return sr_fail(SR_EINVAL, "sr_grad_norm_flat: scratch must be 8-byte aligned");
    if (n_extra < 0) return sr_fail(SR_EINVAL, "sr_grad_norm_flat: n_extra must be >= 0, got %d", n_extra);
    if (n_extra > 0 && !extra_norms) return sr_fail(SR_EINVAL, "sr_grad_norm_flat: extra_norms is NULL but n_extra = %d", n_extra);
    if (scratch_bytes < sr_grad_norm_scratch_bytes(n_groups))
        return sr_fail(SR_EINVAL, "sr_grad_norm_flat: scratch holds fewer bytes than sr_grad_norm_scratch_bytes(%d)", n_groups);
    GroupBounds G{};
    G.n = n_groups;
    for (int i = 0; i <= n_groups; i++) G.begin[i] = begin[i];
    const int parts = norm_ctas(begin[n_groups]);
    double* partials = (double*)scratch;
    cudaStream_t s = (cudaStream_t)stream_;
    if (parts > 0) {
        ProfileScope ps("grad_sumsq", s);
        grad_sumsq_kernel<<<parts, NORM_THREADS, 0, s>>>(G, grads, grad_scale, partials);
    }
    {
        ProfileScope ps("grad_norm_finish", s);
        grad_norm_finish_kernel<<<1, NORM_THREADS, 0, s>>>(n_groups, parts, partials, extra_norms, n_extra, max_norm, total_norm,
                                                          clip_coef, group_sumsq);
    }
    return sr_launched(parts > 0 ? 2 : 1, "sr_grad_norm_flat");
}

SR_API int sr_adam_flat_state(int32_t n_groups, const int64_t* begin, const float* lr, double beta1, double beta2, float eps,
                              int64_t* step, float grad_scale, const float* clip_coef, float* params, const float* grads,
                              float* exp_avg, float* exp_avg_sq, void* stream_) {
    int rc = check_groups("sr_adam_flat_state", n_groups, begin);
    if (rc) return rc;
    if (!lr || !step || !params || !grads || !exp_avg || !exp_avg_sq)
        return sr_fail(SR_EINVAL, "sr_adam_flat_state: a required pointer is NULL");
    if (((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15)
        return sr_fail(SR_EINVAL, "sr_adam_flat_state: params, grads, exp_avg and exp_avg_sq must be 16-byte aligned");
    if ((uintptr_t)step & 7) return sr_fail(SR_EINVAL, "sr_adam_flat_state: step must be 8-byte aligned");
    AdamGroups G{};
    G.n = n_groups;
    for (int i = 0; i <= n_groups; i++) G.begin[i] = begin[i];
    const long long total = begin[n_groups];
    cudaStream_t s = (cudaStream_t)stream_;
    {
        ProfileScope ps("adam_step_count", s);
        adam_step_count_kernel<<<1, 1, 0, s>>>(reinterpret_cast<long long*>(step));
    }
    if (total == 0) return sr_launched(1, "sr_adam_flat_state");
    const long long blocks = (total + 1023) / 1024;
    ProfileScope ps("adam_flat_state", s);
    adam_flat_kernel<true><<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, s>>>(
        G, params, grads, exp_avg, exp_avg_sq, beta1, beta2, eps, 1.0f, grad_scale,
        AdamDeviceState{lr, reinterpret_cast<const long long*>(step), clip_coef});
    return sr_launched(2, "sr_adam_flat_state");
}

SR_API int sr_densify_stats(int32_t M, int32_t P, const float* viewspace_grad, const int32_t* radii, float grad_scale,
                            float* accum, float* denom, float* max_radii, void* stream_) {
    if (M < 0 || P < 0) return sr_fail(SR_EINVAL, "sr_densify_stats: M and P must be >= 0, got M = %d, P = %d", M, P);
    if (M == 0 || P == 0) return 0;
    if (!viewspace_grad || !radii || !accum || !denom || !max_radii)
        return sr_fail(SR_EINVAL, "sr_densify_stats: viewspace_grad, radii, accum, denom and max_radii must not be NULL");
    if (((uintptr_t)viewspace_grad | (uintptr_t)radii | (uintptr_t)accum | (uintptr_t)denom | (uintptr_t)max_radii) & 3)
        return sr_fail(SR_EINVAL, "sr_densify_stats: every array must be 4-byte aligned");
    cudaStream_t s = (cudaStream_t)stream_;
    ProfileScope ps("densify_stats", s);
    densify_stats_kernel<<<(P + 255) / 256, 256, 0, s>>>(M, P, viewspace_grad, radii, grad_scale, accum, denom, max_radii);
    return sr_launched(1, "sr_densify_stats");
}

/* Gather the surfel rows of every parameter group (and both Adam moments) into new flat buffers: new row s = old row
 * src[s]; kind[s] 0 keeps the optimizer state, 1 (clone) and 2 (split child) start from zero state; for kind 2 the xyz /
 * scaling rows come from child_xyz / child_scaling[child_slot[s]].  widths, old_begin, new_begin: host arrays. */
SR_API int sr_surfel_compact(int32_t n_groups, const int32_t* width, const int64_t* old_begin, const int64_t* new_begin,
                             int32_t xyz_group, int32_t scaling_group, int32_t P_new, const int32_t* src, const uint8_t* kind,
                             const int32_t* child_slot, const float* child_xyz, const float* child_scaling, const float* p_old,
                             const float* m_old, const float* v_old, float* p_new, float* m_new, float* v_new, void* stream_) {
    if (n_groups < 1 || n_groups > MAXG)
        return sr_fail(SR_EINVAL, "sr_surfel_compact: n_groups must be in [1, %d], got %d", MAXG, n_groups);
    if (!width || !old_begin || !new_begin) return sr_fail(SR_EINVAL, "sr_surfel_compact: width / old_begin / new_begin is NULL");
    if (P_new < 0) return sr_fail(SR_EINVAL, "sr_surfel_compact: P_new must be >= 0, got %d", P_new);
    if (P_new == 0) return 0;
    if (!src || !kind || !p_old || !m_old || !v_old || !p_new || !m_new || !v_new)
        return sr_fail(SR_EINVAL, "sr_surfel_compact: a required pointer is NULL");
    CompactGroups G{};
    G.n = n_groups; G.xyz_group = xyz_group; G.scaling_group = scaling_group;
    for (int i = 0; i < n_groups; i++) { G.width[i] = width[i]; G.old_begin[i] = old_begin[i]; G.new_begin[i] = new_begin[i]; }
    cudaStream_t s = (cudaStream_t)stream_;
    ProfileScope ps("surfel_compact", s);
    compact_kernel<<<(P_new + 7) / 8, 256, 0, s>>>(G, P_new, src, kind, child_slot, child_xyz, child_scaling, p_old, m_old, v_old,
                                                   p_new, m_new, v_new);
    return sr_launched(1, "sr_surfel_compact");
}

}  // extern "C"
