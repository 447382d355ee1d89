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
// Semantics are torch.optim.Adam's (amsgrad off, no weight decay) and the reference's row-wise copy rules, bit for bit.
#include "common.cuh"

namespace {

constexpr int MAXG = 8;
struct AdamGroups {
    int n;
    long long begin[MAXG + 1];     // element offsets of the groups inside the flat buffer; begin[n] = total
    float lr[MAXG];
};

__global__ void __launch_bounds__(256)
adam_flat_kernel(const AdamGroups G, float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                 float* __restrict__ v, float beta1, float beta2, float eps, float bc1, float sqrt_bc2, float grad_scale) {
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
            float lr = G.lr[0];
#pragma unroll
            for (int q = 1; q < MAXG; q++) if (q < G.n && e >= G.begin[q]) lr = G.lr[q];
            const float gr = G4[k] * grad_scale;
            // torch/optim/adam.py _single_tensor_adam: exp_avg.lerp_(grad, 1 - beta1); exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2);
            // denom = exp_avg_sq.sqrt() / sqrt(bias_correction2) + eps; param.addcdiv_(exp_avg, denom, value=-lr / bias_correction1)
            M4[k] = M4[k] + (gr - M4[k]) * (1.0f - beta1);
            V4[k] = V4[k] * beta2 + gr * gr * (1.0f - beta2);
            const float denom = sqrtf(V4[k]) / sqrt_bc2 + eps;
            P4[k] = P4[k] - (lr / bc1) * (M4[k] / denom);
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

}  // namespace

extern "C" {

/* One Adam step over a flat buffer of `n_groups` back-to-back parameter groups (group g = elements [begin[g], begin[g+1])),
 * each with its own learning rate; torch.optim.Adam semantics (amsgrad off, weight_decay 0).  `step` is the 1-based step
 * count (bias correction); grad_scale multiplies every gradient first (1 / (frames x ranks) averaging).  All device
 * pointers, 16-byte aligned. */
SR_API int sr_adam_flat(int32_t n_groups, const int64_t* begin /* host, n_groups + 1 */, const float* lr /* host, n_groups */,
                        float beta1, float beta2, float eps, int64_t step, float grad_scale, float* params, const float* grads,
                        float* exp_avg, float* exp_avg_sq, void* stream_) {
    if (n_groups < 1 || n_groups > MAXG) return sr_fail(SR_EINVAL, "sr_adam_flat: n_groups must be in [1, %d], got %d", MAXG, n_groups);
    if (!begin || !lr || !params || !grads || !exp_avg || !exp_avg_sq) return sr_fail(SR_EINVAL, "sr_adam_flat: a required pointer is NULL");
    if (step < 1) return sr_fail(SR_EINVAL, "sr_adam_flat: step must be >= 1, got %lld", (long long)step);
    if (((uintptr_t)params | (uintptr_t)grads | (uintptr_t)exp_avg | (uintptr_t)exp_avg_sq) & 15)
        return sr_fail(SR_EINVAL, "sr_adam_flat: params, grads, exp_avg and exp_avg_sq must be 16-byte aligned");
    AdamGroups G{};
    G.n = n_groups;
    for (int i = 0; i <= n_groups; i++) G.begin[i] = begin[i];
    for (int i = 0; i < n_groups; i++) G.lr[i] = lr[i];
    const long long total = begin[n_groups];
    if (total <= 0) return 0;
    const float bc1 = (float)(1.0 - pow((double)beta1, (double)step));
    const float sqrt_bc2 = (float)sqrt(1.0 - pow((double)beta2, (double)step));
    cudaStream_t s = (cudaStream_t)stream_;
    const long long blocks = (total + 1023) / 1024;
    ProfileScope ps("adam_flat", s);
    // grid-stride: at most 16 CTAs per SM of an H100 SXM (132 SMs)
    adam_flat_kernel<<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, s>>>(G, params, grads, exp_avg, exp_avg_sq, beta1,
                                                                                       beta2, eps, bc1, sqrt_bc2, grad_scale);
    return sr_launched(1, "sr_adam_flat");
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
