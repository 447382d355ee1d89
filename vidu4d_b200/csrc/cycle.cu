// cycle.cu -- Stage 3's deformation-cycle regulariser, forward and backward (DESIGN.md section 3.5c): every frame's warped
// surfels are taken back to object space, warped BACKWARD to the canonical space with the frame's own bones, and compared
// with where they started; the backward warp's skinning entropy and delta-skin terms come out of the same pass.
//
// Replaces (behaviour, not code) of the reference's PyTorch chain
//   lab4d/nnutils/deformable_gaussian.py:1272-1275,1517-1574   cycle_loss
//   lab4d/nnutils/deformable_gaussian.py:738-764     cam_to_field       x_t = qc* x_cam qc + qc* (-tc) qc
//   lab4d/utils/quat_transform.py:286-291            quaternion_translation_inverse
//   lab4d/nnutils/warping.py:378-444                 SkinningWarp.forward(backward=True): skinning on the frame's
//                                                    t_articulation bones, per-bone se3 = rest o t_articulation^-1
//   lab4d/nnutils/skinning.py:89-124                 Gaussian skinning logits -(|x_bone / gauss|^2 + delta), delta
//                                                    evaluated by the caller's frame-conditioned MLP
//   lab4d/utils/geom_utils.py:48-92                  dual_quaternion_skinning (sign-aligned blend, return_qt)
//   lab4d/nnutils/deformable_gaussian.py:1033-1046   apply_qt_to_gaussian, then cyc_dist = |x_cycled - x|
//   lab4d/utils/loss_utils.py:21-42                  cross_entropy_skin_loss (skin_entropy), delta_skin = mean_b delta^2
//   lab4d/engine/model.py:850-853,994-1012           reg_deform_cyc / reg_delta_skin / reg_skin_entropy, each reduced as
//                                                    v[v > 0].mean() * its weight
// which materialises (M, P, B, 4) dual-quaternion temporaries (~240 MB each at M = 2, P = 300 K, B = 25), (M, P, B, 3) bone
// coordinates and a sign tensor, and syncs with the host once per term for v[v > 0].  Here one thread owns one surfel
// and loops over the frames; every frame's bone tables sit in shared memory.  The skinning weights depend on the frame
// (the bones are t_articulation[m]), so unlike bob_warp they are recomputed per frame.
//
// cycle_fwd    one thread per surfel: per frame cyc, ent, dsk; per-frame sums and integer counts of the positive values
//              (warp shuffle -> shared memory -> one global atomic per value and CTA).
// cycle_scale  one thread: scale_k = w_k / count_k over the batch (0 when the count is 0), terms scaled, loss written.
// cycle_bwd    one thread per surfel, recomputes everything; a value v > 0 gets dL/dv = g_loss * scale_k, v = 0 none (the
//              autograd of v[v > 0].mean()).  dL/dxyz_cam and dL/ddelta written directly, dL/dxyz summed over the frames
//              in registers, table gradients reduced butterfly -> shared memory -> one global atomic per value and CTA.
//
// Tables, prepared by the caller with differentiable torch ops (vidu4d_b200.warp.cycle_tables):
//   o2b_q (M,B,4), o2b_t (M,B,3)   object -> bone transform of t_articulation[m, b]
//   inv_gauss (B,3)                exp(-log_gauss)
//   se3_r, se3_d (M,B,4)           rest_articulation o t_articulation[m]^-1 as a dual quaternion
//   cam_q (M,4), cam_t (M,3)       field2cam of each frame
#include "warp_common.cuh"

namespace {

constexpr int CYC_FWD_THREADS = 256;
constexpr int CYC_BWD_THREADS = 128;     // w[B] and gw[B] live in registers, as in bob_warp_bwd / reproj_bwd

struct CycleDims { int P, B, M; };

struct CycleIn { const float *oq, *ot, *ig, *sr, *sd, *cq, *ct; };

// shared-memory tables of all frames: oq[M*B*4] ot[M*B*3] ig[B*3] sr[M*B*4] sd[M*B*4] cq[M*4] ct[M*3]
struct CycleTables {
    float *oq, *ot, *ig, *sr, *sd, *cq, *ct;
    __host__ __device__ static size_t floats(int B, int M) { return (size_t)M * B * 15 + (size_t)B * 3 + (size_t)M * 7; }
    __device__ __forceinline__ void bind(float* s, int B, int M) {
        oq = s; ot = oq + M * B * 4; ig = ot + M * B * 3; sr = ig + B * 3; sd = sr + M * B * 4; cq = sd + M * B * 4; ct = cq + M * 4;
    }
    // the warp_common.cuh view of frame m: that frame's object -> bone transforms, the shared inv_gauss, every frame's
    // blend tables (blend / blend_vjp index them by m) and the cameras
    __device__ __forceinline__ Tables frame(int B, int m) const {
        Tables T;
        T.oq = oq + m * B * 4; T.ot = ot + m * B * 3; T.ig = ig; T.sr = sr; T.sd = sd; T.cq = cq; T.ct = ct;
        return T;
    }
};

__device__ __forceinline__ void load_cycle_tables(float* s, int B, int M, const CycleIn in) {
    const float* src[7] = {in.oq, in.ot, in.ig, in.sr, in.sd, in.cq, in.ct};
    const int n[7] = {M * B * 4, M * B * 3, B * 3, M * B * 4, M * B * 4, M * 4, M * 3};
    float* p = s;
#pragma unroll
    for (int k = 0; k < 7; k++) {
        for (int i = threadIdx.x; i < n[k]; i += blockDim.x) p[i] = __ldg(src[k] + i);
        p += n[k];
    }
}

// frame m's backward warp of one camera-space point: x_t in object space at time t, skinning weights on the frame's
// bones, the blended (q, qd) and the cycled point xo = q x_t q* + t
template <int BMAX>
__device__ __forceinline__ void cycle_point(const Tables& T, int B, int m, const float (&xcam)[3], const float* __restrict__ delta_row,
                                            float (&xt)[3], float (&w)[BMAX], int& anchor, float& ent, Q4& q, Q4& qd, float& inv,
                                            float (&xo)[3]) {
    const Q4 qi = qconj(ldq(T.cq + 4 * m));
    float a0, a1, a2, b0, b1, b2;
    qrot(qi, xcam[0], xcam[1], xcam[2], a0, a1, a2);
    qrot(qi, -T.ct[3 * m], -T.ct[3 * m + 1], -T.ct[3 * m + 2], b0, b1, b2);
    xt[0] = a0 + b0; xt[1] = a1 + b1; xt[2] = a2 + b2;
    skin_weights<BMAX>(T, B, xt[0], xt[1], xt[2], delta_row, w, anchor, ent);
    Q4 QR, QD;
    blend<BMAX>(T, B, m, w, anchor, QR, QD);
    inv = rsqrtf(qdot(QR, QR));
    q = qscale(QR, inv); qd = qscale(QD, inv);
    const Q4 t4 = qmul(qd, qconj(q));                               // t = 2 (qd (x) q*)[1:]
    qrot(q, xt[0], xt[1], xt[2], xo[0], xo[1], xo[2]);
    xo[0] += 2.f * t4.x; xo[1] += 2.f * t4.y; xo[2] += 2.f * t4.z;
}

__device__ __forceinline__ float delta_sq_mean(const float* __restrict__ delta_row, int B) {
    float s = 0.f;
    for (int b = 0; b < B; b++) { const float v = __ldg(delta_row + b); s += v * v; }
    return s / (float)B;
}

template <int BMAX>
__global__ void __launch_bounds__(CYC_FWD_THREADS)
cycle_fwd_kernel(const CycleDims d, const float* __restrict__ xyz, const float* __restrict__ xyz_cam, const CycleIn in,
                 const float* __restrict__ delta, float* __restrict__ sums, uint32_t* __restrict__ counts) {
    extern __shared__ float smem[];
    const int B = d.B, M = d.M;
    const size_t nt = CycleTables::floats(B, M);
    load_cycle_tables(smem, B, M, in);
    float* bsum = smem + nt;                                         // per-frame sums [M*3] and counts [M*3] of this CTA
    uint32_t* bcnt = reinterpret_cast<uint32_t*>(bsum + M * 3);
    for (int i = threadIdx.x; i < M * 3; i += blockDim.x) { bsum[i] = 0.f; bcnt[i] = 0u; }
    __syncthreads();
    CycleTables S; S.bind(smem, B, M);
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < d.P;                                       // dead lanes take part in the warp sums with zeros
    float x0 = 0.f, x1 = 0.f, x2 = 0.f;
    if (live) { x0 = xyz[3 * (size_t)p]; x1 = xyz[3 * (size_t)p + 1]; x2 = xyz[3 * (size_t)p + 2]; }
    for (int m = 0; m < M; m++) {
        float v[3] = {0.f, 0.f, 0.f};                               // cyc, dsk, ent
        if (live) {
            const Tables T = S.frame(B, m);
            const size_t n = (size_t)m * d.P + p;
            const float xcam[3] = {xyz_cam[3 * n], xyz_cam[3 * n + 1], xyz_cam[3 * n + 2]};
            const float* drow = delta ? delta + n * B : nullptr;
            float xt[3], w[BMAX], inv, xo[3];
            int anchor; Q4 q, qd;
            cycle_point<BMAX>(T, B, m, xcam, drow, xt, w, anchor, v[2], q, qd, inv, xo);
            const float dx = xo[0] - x0, dy = xo[1] - x1, dz = xo[2] - x2;
            v[0] = sqrtf(dx * dx + dy * dy + dz * dz);
            if (drow) v[1] = delta_sq_mean(drow, B);
        }
#pragma unroll
        for (int k = 0; k < 3; k++) {
            const bool on = v[k] > 0.f;
            float s = on ? v[k] : 0.f;
            uint32_t c = on;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                s += __shfl_xor_sync(0xffffffffu, s, o);
                c += __shfl_xor_sync(0xffffffffu, c, o);
            }
            if ((threadIdx.x & 31) == 0 && c) { atomicAdd(bsum + 3 * m + k, s); atomicAdd(bcnt + 3 * m + k, c); }
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < M * 3; i += blockDim.x)
        if (bcnt[i]) { atomicAdd(sums + i, bsum[i]); atomicAdd(counts + i, bcnt[i]); }
}

// scale_k = w_k / count_k with count_k over the whole batch (the reference's v[v > 0].mean() * wt; 0 when no v > 0)
__global__ void cycle_scale_kernel(int M, const float* __restrict__ weights, const uint32_t* __restrict__ counts,
                                   float* __restrict__ terms, float* __restrict__ scale, float* __restrict__ loss) {
    if (threadIdx.x != 0) return;
    float s[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
        unsigned long long c = 0;
        for (int m = 0; m < M; m++) c += counts[3 * m + k];
        s[k] = c ? __ldg(weights + k) / (float)c : 0.f;
        scale[k] = s[k];
    }
    float l = 0.f;
    for (int m = 0; m < M; m++) {
#pragma unroll
        for (int k = 0; k < 3; k++) { terms[3 * m + k] *= s[k]; l += terms[3 * m + k]; }
    }
    *loss = l;
}

template <int BMAX>
__global__ void __launch_bounds__(CYC_BWD_THREADS)
cycle_bwd_kernel(const CycleDims d, const float* __restrict__ xyz, const float* __restrict__ xyz_cam, const CycleIn in,
                 const float* __restrict__ delta, const float* __restrict__ scale, const float* __restrict__ g_loss,
                 float* __restrict__ g_xyz_cam, float* __restrict__ g_xyz, float* __restrict__ g_delta,
                 float* __restrict__ g_tables) {
    extern __shared__ float smem[];
    const int B = d.B, M = d.M;
    const size_t nt = CycleTables::floats(B, M);
    load_cycle_tables(smem, B, M, in);
    float* gacc = smem + nt;                                        // gradient of every table entry, same layout
    for (int i = threadIdx.x; i < (int)nt; i += blockDim.x) gacc[i] = 0.f;
    __syncthreads();
    CycleTables S, G;
    S.bind(smem, B, M); G.bind(gacc, B, M);
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < d.P;                                       // dead lanes take part in the warp sums with zeros
    const size_t ps = live ? (size_t)p : 0;
    const float lv = live ? 1.f : 0.f;
    const float x0 = xyz[3 * ps], x1 = xyz[3 * ps + 1], x2 = xyz[3 * ps + 2];
    const float gl = __ldg(g_loss);
    const float s_cyc = gl * __ldg(scale), s_dsk = gl * __ldg(scale + 1), s_ent = gl * __ldg(scale + 2);
    float gx0 = 0.f, gx1 = 0.f, gx2 = 0.f;
    for (int m = 0; m < M; m++) {
        const Tables T = S.frame(B, m);
        const size_t n = (size_t)m * d.P + ps;
        const float xcam[3] = {xyz_cam[3 * n], xyz_cam[3 * n + 1], xyz_cam[3 * n + 2]};
        const float* drow = delta ? delta + n * B : nullptr;
        float xt[3], w[BMAX], gw[BMAX], inv, xo[3], ent;
        int anchor; Q4 q, qd;
        cycle_point<BMAX>(T, B, m, xcam, drow, xt, w, anchor, ent, q, qd, inv, xo);
        // ---- the three values: dL/dv = g_loss * scale_k where v > 0, nothing where v = 0
        const float dx = xo[0] - x0, dy = xo[1] - x1, dz = xo[2] - x2;
        const float cyc = sqrtf(dx * dx + dy * dy + dz * dz);
        const float gc = (live && cyc > 0.f) ? s_cyc / cyc : 0.f;
        const float go0 = gc * dx, go1 = gc * dy, go2 = gc * dz;     // dL/dxo;  dL/dxyz = -dL/dxo
        gx0 -= go0; gx1 -= go1; gx2 -= go2;
        const float ge = (live && ent > 0.f) ? s_ent : 0.f;
        const float g_d2 = (live && drow && delta_sq_mean(drow, B) > 0.f) ? s_dsk * 2.f / (float)B : 0.f;
        // ---- xo = q xt q* + t, t = 2 (qd (x) q*)[1:]; normalisation q = QR / |QR|, qd = QD / |QR|
        Q4 gq; float gt0, gt1, gt2;
        qrot_vjp(q, xt[0], xt[1], xt[2], go0, go1, go2, gq, gt0, gt1, gt2);
        const Q4 gct = pure(2.f * go0, 2.f * go1, 2.f * go2);
        const Q4 gqd = qmul(gct, q);
        gq = qadd(gq, qconj(qmul(qconj(qd), gct)));
        const Q4 gQD = qscale(gqd, inv);
        const Q4 gQR = qscale(qadd(gq, qscale(q, -(qdot(q, gq) + qdot(qd, gqd)))), inv);
        // ---- blend, then the skinning weights on frame m's bones (entropy and delta^2 terms included)
#pragma unroll
        for (int b = 0; b < BMAX; b++) gw[b] = 0.f;
        blend_vjp<BMAX>(T, B, m, w, anchor, gQR, gQD, gw, G.sr, G.sd);
        skin_vjp<BMAX>(T, B, xt[0], xt[1], xt[2], w, gw, anchor, ge, n, live, lv, g_delta, drow, g_d2, G.oq + m * B * 4,
                       G.ot + m * B * 3, G.ig, gt0, gt1, gt2);
        // ---- xt = qi xcam qi* + qi (-tc) qi*, qi = qc*
        const Q4 qi = qconj(ldq(T.cq + 4 * m));
        Q4 gqi, gqn; float gc0, gc1, gc2, gn0, gn1, gn2;
        qrot_vjp(qi, xcam[0], xcam[1], xcam[2], gt0, gt1, gt2, gqi, gc0, gc1, gc2);
        qrot_vjp(qi, -T.ct[3 * m], -T.ct[3 * m + 1], -T.ct[3 * m + 2], gt0, gt1, gt2, gqn, gn0, gn1, gn2);
        if (live) { g_xyz_cam[3 * n] = gc0; g_xyz_cam[3 * n + 1] = gc1; g_xyz_cam[3 * n + 2] = gc2; }
        acc_q(G.cq + 4 * m, qconj(qadd(gqi, gqn)));
        acc_table(G.ct + 3 * m, -gn0); acc_table(G.ct + 3 * m + 1, -gn1); acc_table(G.ct + 3 * m + 2, -gn2);
    }
    if (live) { g_xyz[3 * ps] = gx0; g_xyz[3 * ps + 1] = gx1; g_xyz[3 * ps + 2] = gx2; }
    __syncthreads();
    for (int i = threadIdx.x; i < (int)nt; i += blockDim.x)
        if (gacc[i] != 0.f) atomicAdd(g_tables + i, gacc[i]);
}

int check_cycle(int32_t P, int32_t B, int32_t M) {
    if (P < 0) return sr_fail(SR_EINVAL, "P must be >= 0, got %d", P);
    if (M < 1) return sr_fail(SR_EINVAL, "M must be >= 1, got %d", M);
    if (B < 1 || B > 64) return sr_fail(SR_EINVAL, "B must be in [1, 64], got %d", B);
    if (2 * CycleTables::floats(B, M) * sizeof(float) > SR_TABLE_SMEM_MAX)
        return sr_fail(SR_EINVAL, "the bone / frame tables of B = %d, M = %d frames do not fit in shared memory", B, M);
    return 0;
}

}  // namespace

extern "C" {

SR_API size_t sr_cycle_loss_table_floats(int32_t B, int32_t M) { return CycleTables::floats(B, M); }

SR_API int sr_cycle_loss_forward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* xyz_cam, const float* o2b_q,
                                 const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                 const float* se3_d, const float* cam_q, const float* cam_t, const float* weights, float* terms,
                                 uint32_t* counts, float* scale, float* loss, void* stream_) {
    if (int rc = check_cycle(P, B, M)) return rc;
    if (!xyz || !xyz_cam || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !weights || !terms ||
        !counts || !scale || !loss)
        return sr_fail(SR_EINVAL, "sr_cycle_loss_forward: a required pointer is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    CK(cudaMemsetAsync(terms, 0, (size_t)M * 3 * sizeof(float), s), "sr_cycle_loss_forward: memset(terms)");
    CK(cudaMemsetAsync(counts, 0, (size_t)M * 3 * sizeof(uint32_t), s), "sr_cycle_loss_forward: memset(counts)");
    int launches = 1;
    if (P > 0) {
        const CycleDims d{P, B, M};
        const CycleIn in{o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t};
        const size_t smem = CycleTables::floats(B, M) * sizeof(float) + (size_t)M * 3 * 8;
        auto launch = [&](auto kern) -> int {
            CK(sr_opt_in_smem(kern, smem), "sr_cycle_loss_forward: shared-memory opt-in");
            ProfileScope ps("cycle_fwd", s);
            kern<<<(P + CYC_FWD_THREADS - 1) / CYC_FWD_THREADS, CYC_FWD_THREADS, smem, s>>>(d, xyz, xyz_cam, in, delta, terms, counts);
            return 0;
        };
        if (int rc = B <= 32 ? launch(cycle_fwd_kernel<32>) : launch(cycle_fwd_kernel<64>)) return rc;
        launches++;
    }
    {
        ProfileScope ps("cycle_scale", s);
        cycle_scale_kernel<<<1, 32, 0, s>>>(M, weights, counts, terms, scale, loss);
    }
    return sr_launched(launches, "sr_cycle_loss_forward");
}

SR_API int sr_cycle_loss_backward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* xyz_cam, const float* o2b_q,
                                  const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                  const float* se3_d, const float* cam_q, const float* cam_t, const float* scale,
                                  const float* g_loss, float* g_xyz_cam, float* g_xyz, float* g_delta, float* g_tables,
                                  void* stream_) {
    if (int rc = check_cycle(P, B, M)) return rc;
    if (!xyz || !xyz_cam || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !scale || !g_loss ||
        !g_xyz_cam || !g_xyz || !g_tables)
        return sr_fail(SR_EINVAL, "sr_cycle_loss_backward: a required pointer is NULL");
    if (g_delta && !delta) return sr_fail(SR_EINVAL, "sr_cycle_loss_backward: g_delta without delta");
    cudaStream_t s = (cudaStream_t)stream_;
    const size_t nt = CycleTables::floats(B, M);
    CK(cudaMemsetAsync(g_tables, 0, nt * sizeof(float), s), "sr_cycle_loss_backward: memset(g_tables)");
    if (P == 0) return 0;
    const CycleDims d{P, B, M};
    const CycleIn in{o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t};
    const size_t smem = 2 * nt * sizeof(float);
    auto launch = [&](auto kern) -> int {
        CK(sr_opt_in_smem(kern, smem), "sr_cycle_loss_backward: shared-memory opt-in");
        ProfileScope ps("cycle_bwd", s);
        kern<<<(P + CYC_BWD_THREADS - 1) / CYC_BWD_THREADS, CYC_BWD_THREADS, smem, s>>>(d, xyz, xyz_cam, in, delta, scale, g_loss,
                                                                                   g_xyz_cam, g_xyz, g_delta, g_tables);
        return 0;
    };
    if (int rc = B <= 32 ? launch(cycle_bwd_kernel<32>) : launch(cycle_bwd_kernel<64>)) return rc;
    return sr_launched(1, "sr_cycle_loss_backward");
}

}  // extern "C"
