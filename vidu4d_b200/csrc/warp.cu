// warp.cu -- fused "bob" skinning warp of the canonical surfels into every frame's camera space, forward and backward
// (SURVEY.md section 8(f) row N2; the step right BEFORE the rasterizer in a Stage-3 iteration).
//
// Replaces (behaviour, not code) of the reference's PyTorch chain
//   lab4d/nnutils/deformable_gaussian.py:1395-1434   forward_warp
//   lab4d/nnutils/deformable_gaussian.py:1033-1046   apply_qt_to_gaussian           x' = q x q* + t,  r' = q (x) r
//   lab4d/nnutils/warping.py:378-444                 SkinningWarp.forward (forward direction, return_qt)
//   lab4d/nnutils/skinning.py:89-142                 Gaussian skinning logits        -(|x_bone / gauss|^2 + delta)
//   lab4d/utils/geom_utils.py:48-92                  dual_quaternion_skinning        sign-aligned blend, normalise
//   lab4d/utils/quat_transform.py                    quaternion algebra (real part first); the 3-vector products are what
//   lab4d/third_party/quaternion/src/quaternion.cu:27-60   the reference's own helper kernels do (row N3)
//   lab4d/utils/loss_utils.py:21-42                  cross_entropy_skin_loss
// which materialises two (M, P, B, 4) dual-quaternion tensors (~240 MB each at M = 2, P = 300 K, B = 25), a (M, P, B)
// sign tensor and several (M, P, B, 3) temporaries per step, and recomputes the FRAME-INDEPENDENT skinning weights for
// every frame.  Here one thread owns one surfel: its B skinning weights live in registers, are computed once, and are
// reused for all M frames; the per-bone / per-frame transforms sit in shared memory.  HBM traffic is the algorithmic
// minimum: read 28 B (+ 4B of delta) per surfel, write 28 B per surfel and frame.
//
// Inputs that the kernel treats as small tables are prepared by the caller with ordinary (differentiable) torch ops:
//   o2b_q (B,4), o2b_t (B,3)   object -> bone rigid transform of the REST pose (inverse of rest_articulation)
//   inv_gauss (B,3)            exp(-log_gauss)
//   se3_r, se3_d (M,B,4)       per frame and bone: t_articulation o rest_articulation^-1 as a dual quaternion
//   cam_q (M,4), cam_t (M,3)   field2cam of each frame
// The backward recomputes the weights (cheaper than storing (P,B) floats) and returns gradients for every input; table
// gradients are reduced warp -> block (shared memory) -> global (one atomic per value and block).
#include "warp_common.cuh"

namespace {

template <int BMAX>
__global__ void __launch_bounds__(256)
bob_warp_fwd_kernel(const WarpDims d, const float* __restrict__ xyz, const float* __restrict__ rot,
                    const float* __restrict__ o2b_q, const float* __restrict__ o2b_t, const float* __restrict__ inv_gauss,
                    const float* __restrict__ delta, const float* __restrict__ se3_r, const float* __restrict__ se3_d,
                    const float* __restrict__ cam_q, const float* __restrict__ cam_t, float* __restrict__ xyz_cam,
                    float* __restrict__ rot_cam, float* __restrict__ skin_entropy) {
    extern __shared__ float smem[];
    load_tables(smem, d, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t);
    __syncthreads();
    Tables T; T.bind(smem, d.B, d.M);
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= d.P) return;
    const float x = xyz[3 * (size_t)p], y = xyz[3 * (size_t)p + 1], z = xyz[3 * (size_t)p + 2];
    const Q4 r = ldq(rot + 4 * (size_t)p);
    float w[BMAX];
    int anchor; float ent;
    skin_weights<BMAX>(T, d.B, x, y, z, delta ? delta + (size_t)p * d.B : nullptr, w, anchor, ent);
    if (skin_entropy) skin_entropy[p] = ent;
    for (int m = 0; m < d.M; m++) {
        Q4 QR, QD;
        blend<BMAX>(T, d.B, m, w, anchor, QR, QD);
        const float inv = rsqrtf(qdot(QR, QR));
        const Q4 q = qscale(QR, inv), qd = qscale(QD, inv);
        const Q4 t4 = qmul(qd, qconj(q));                           // t = 2 (qd (x) q*)[1:]
        float tx, ty, tz;
        qrot(q, x, y, z, tx, ty, tz);
        tx += 2.f * t4.x; ty += 2.f * t4.y; tz += 2.f * t4.z;
        const Q4 rt = qmul(q, r);
        const Q4 qc = ldq(T.cq + 4 * m);
        float cx, cy, cz;
        qrot(qc, tx, ty, tz, cx, cy, cz);
        float* ox = xyz_cam + ((size_t)m * d.P + p) * 3;
        ox[0] = cx + T.ct[3 * m]; ox[1] = cy + T.ct[3 * m + 1]; ox[2] = cz + T.ct[3 * m + 2];
        const Q4 rc = qmul(qc, rt);
        reinterpret_cast<float4*>(rot_cam)[(size_t)m * d.P + p] = make_float4(rc.w, rc.x, rc.y, rc.z);
    }
}

template <int BMAX>
__global__ void __launch_bounds__(256)
bob_warp_bwd_kernel(const WarpDims d, const float* __restrict__ xyz, const float* __restrict__ rot,
                    const float* __restrict__ o2b_q, const float* __restrict__ o2b_t, const float* __restrict__ inv_gauss,
                    const float* __restrict__ delta, const float* __restrict__ se3_r, const float* __restrict__ se3_d,
                    const float* __restrict__ cam_q, const float* __restrict__ cam_t, const float* __restrict__ g_xyz_cam,
                    const float* __restrict__ g_rot_cam, const float* __restrict__ g_entropy, float* __restrict__ g_xyz,
                    float* __restrict__ g_rot, float* __restrict__ g_delta, float* __restrict__ g_tables) {
    extern __shared__ float smem[];
    const int B = d.B, M = d.M, nt = Tables::floats(B, M);
    load_tables(smem, d, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t);
    float* gacc = smem + nt;                                        // gradient of every table entry, same layout
    for (int i = threadIdx.x; i < nt; i += blockDim.x) gacc[i] = 0.f;
    __syncthreads();
    Tables T; T.bind(smem, B, M);
    float* g_oq = gacc; float* g_ot = g_oq + B * 4; float* g_ig = g_ot + B * 3; float* g_sr = g_ig + B * 3;
    float* g_sd = g_sr + M * B * 4; float* g_cq = g_sd + M * B * 4; float* g_ct = g_cq + M * 4;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = p < d.P;                                       // dead lanes still take part in the warp sums (with zeros)
    const size_t ps = live ? (size_t)p : 0;
    const float x = xyz[3 * ps], y = xyz[3 * ps + 1], z = xyz[3 * ps + 2];
    const Q4 r = ldq(rot + 4 * ps);
    float w[BMAX], gw[BMAX];
    int anchor; float ent;
    skin_weights<BMAX>(T, B, x, y, z, delta ? delta + ps * B : nullptr, w, anchor, ent);
#pragma unroll
    for (int b = 0; b < BMAX; b++) gw[b] = 0.f;
    float gxx = 0.f, gxy = 0.f, gxz = 0.f;
    Q4 grot = {0.f, 0.f, 0.f, 0.f};
    const float lv = live ? 1.f : 0.f;
    for (int m = 0; m < M; m++) {
        Q4 QR, QD;
        blend<BMAX>(T, B, m, w, anchor, QR, QD);
        const float inv = rsqrtf(qdot(QR, QR));
        const Q4 q = qscale(QR, inv), qd = qscale(QD, inv);
        const Q4 t4 = qmul(qd, qconj(q));
        float tx, ty, tz;
        qrot(q, x, y, z, tx, ty, tz);
        tx += 2.f * t4.x; ty += 2.f * t4.y; tz += 2.f * t4.z;
        const Q4 rt = qmul(q, r);
        const Q4 qc = ldq(T.cq + 4 * m);
        const float* gx = g_xyz_cam + ((size_t)m * d.P + ps) * 3;
        const float gcx = gx[0] * lv, gcy = gx[1] * lv, gcz = gx[2] * lv;
        const float4 grc4 = reinterpret_cast<const float4*>(g_rot_cam)[(size_t)m * d.P + ps];
        const Q4 grc = {grc4.x * lv, grc4.y * lv, grc4.z * lv, grc4.w * lv};
        // ---- camera: x_c = qc x_t qc* + tc ; r_c = qc (x) r_t
        Q4 gqc; float gtx, gty, gtz;
        qrot_vjp(qc, tx, ty, tz, gcx, gcy, gcz, gqc, gtx, gty, gtz);
        gqc = qadd(gqc, qmul(grc, qconj(rt)));
        const Q4 grt = qmul(qconj(qc), grc);
        acc_q(g_cq + 4 * m, gqc);
        acc_table(g_ct + 3 * m, gcx); acc_table(g_ct + 3 * m + 1, gcy); acc_table(g_ct + 3 * m + 2, gcz);
        // ---- x_t = q x q* + t ; r_t = q (x) rot
        Q4 gq; float ax, ay, az;
        qrot_vjp(q, x, y, z, gtx, gty, gtz, gq, ax, ay, az);
        gxx += ax; gxy += ay; gxz += az;
        gq = qadd(gq, qmul(grt, qconj(r)));
        grot = qadd(grot, qmul(qconj(q), grt));
        // ---- t = 2 (qd (x) q*)[1:]
        const Q4 gc = pure(2.f * gtx, 2.f * gty, 2.f * gtz);
        const Q4 gqd = qmul(gc, q);
        gq = qadd(gq, qconj(qmul(qconj(qd), gc)));
        // ---- normalisation q = QR / |QR|, qd = QD / |QR|
        const Q4 gQD = qscale(gqd, inv);
        const Q4 gQR = qscale(qadd(gq, qscale(q, -(qdot(q, gq) + qdot(qd, gqd)))), inv);
        // ---- blend
        blend_vjp<BMAX>(T, B, m, w, anchor, gQR, gQD, gw, g_sr, g_sd);
    }
    // ---- softmax (+ entropy) backward, then the Gaussian logits
    float dotwg = 0.f;
#pragma unroll
    for (int b = 0; b < BMAX; b++) dotwg += w[b] * gw[b];
    const float ge = (g_entropy && live) ? g_entropy[ps] : 0.f;
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int c3 = 0; c3 < (BMAX + 2) / 3; c3++) {
        if (3 * c3 < B) {                                            // three bones x (4 + 3 + 3) components per butterfly
            float vals[32];
            vals[30] = 0.f; vals[31] = 0.f;
#pragma unroll
            for (int j = 0; j < 3; j++) {
                const int b = 3 * c3 + j;
#pragma unroll
                for (int i = 0; i < 10; i++) vals[10 * j + i] = 0.f;
                if (b < B && b < BMAX) {
                    const float gl = (w[b] * (gw[b] - dotwg) + ge * (w[b] - (b == anchor ? 1.f : 0.f))) * lv;
                    if (g_delta && live) g_delta[ps * B + b] = -gl;
                    const Q4 qb = ldq(T.oq + 4 * b);
                    float bx, by, bz;
                    qrot(qb, x, y, z, bx, by, bz);
                    bx += T.ot[3 * b]; by += T.ot[3 * b + 1]; bz += T.ot[3 * b + 2];
                    const float i0 = T.ig[3 * b], i1 = T.ig[3 * b + 1], i2 = T.ig[3 * b + 2];
                    // logit = -(|xb * ig|^2 + delta):  g_s = -2 s gl
                    const float gs0 = -2.f * bx * i0 * gl, gs1 = -2.f * by * i1 * gl, gs2 = -2.f * bz * i2 * gl;
                    const float gb0 = gs0 * i0, gb1 = gs1 * i1, gb2 = gs2 * i2;
                    Q4 gqb; float ax, ay, az;
                    qrot_vjp(qb, x, y, z, gb0, gb1, gb2, gqb, ax, ay, az);
                    gxx += ax; gxy += ay; gxz += az;
                    vals[10 * j] = gqb.w; vals[10 * j + 1] = gqb.x; vals[10 * j + 2] = gqb.y; vals[10 * j + 3] = gqb.z;
                    vals[10 * j + 4] = gb0; vals[10 * j + 5] = gb1; vals[10 * j + 6] = gb2;
                    vals[10 * j + 7] = gs0 * bx; vals[10 * j + 8] = gs1 * by; vals[10 * j + 9] = gs2 * bz;
                }
            }
            const float tot = butterfly32(vals, lane);
            const int j = lane / 10, i = lane - 10 * j, b = 3 * c3 + j;
            if (lane < 30 && b < B && tot != 0.f) {
                float* dst = i < 4 ? g_oq + 4 * b + i : (i < 7 ? g_ot + 3 * b + (i - 4) : g_ig + 3 * b + (i - 7));
                atomicAdd(dst, tot);
            }
        }
    }
    if (live) {
        g_xyz[3 * ps] = gxx; g_xyz[3 * ps + 1] = gxy; g_xyz[3 * ps + 2] = gxz;
        reinterpret_cast<float4*>(g_rot)[ps] = make_float4(grot.w, grot.x, grot.y, grot.z);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < nt; i += blockDim.x)
        if (gacc[i] != 0.f) atomicAdd(g_tables + i, gacc[i]);
}

int check_warp(int32_t P, int32_t B, int32_t M) {
    if (P < 0) return sr_fail(SR_EINVAL, "P must be >= 0, got %d", P);
    if (B < 1 || B > 64) return sr_fail(SR_EINVAL, "B must be in [1, 64], got %d", B);
    if (M < 1) return sr_fail(SR_EINVAL, "M must be >= 1, got %d", M);
    return 0;
}

}  // namespace

extern "C" {

SR_API size_t sr_bob_warp_table_floats(int32_t B, int32_t M) { return (size_t)B * 10 + (size_t)M * B * 8 + (size_t)M * 7; }

SR_API int sr_bob_warp_forward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* rot, const float* o2b_q,
                               const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                               const float* se3_d, const float* cam_q, const float* cam_t, float* xyz_cam, float* rot_cam,
                               float* skin_entropy, void* stream_) {
    if (int rc = check_warp(P, B, M)) return rc;
    if (P == 0) return 0;
    if (!xyz || !rot || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !xyz_cam || !rot_cam)
        return sr_fail(SR_EINVAL, "sr_bob_warp_forward: a required pointer is NULL");
    if (((uintptr_t)rot_cam & 15)) return sr_fail(SR_EINVAL, "sr_bob_warp_forward: rot_cam must be 16-byte aligned");
    const WarpDims d{P, B, M};
    const size_t smem = sr_bob_warp_table_floats(B, M) * sizeof(float);
    if (smem > SR_TABLE_SMEM_MAX)                    // split the frames over several calls
        return sr_fail(SR_EINVAL, "sr_bob_warp_forward: the tables of B = %d, M = %d frames do not fit in shared memory", B, M);
    cudaStream_t s = (cudaStream_t)stream_;
    ProfileScope ps("bob_warp_fwd", s);
    auto launch = [&](auto kern) -> int {
        CK(sr_opt_in_smem(kern, smem), "sr_bob_warp_forward: shared-memory opt-in");
        kern<<<(P + 255) / 256, 256, smem, s>>>(d, xyz, rot, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t, xyz_cam,
                                                 rot_cam, skin_entropy);
        return 0;
    };
    if (int rc = B <= 32 ? launch(bob_warp_fwd_kernel<32>) : launch(bob_warp_fwd_kernel<64>)) return rc;
    return sr_launched(1, "sr_bob_warp_forward");
}

/* g_tables: float[sr_bob_warp_table_floats(B, M)], laid out o2b_q[B*4] o2b_t[B*3] inv_gauss[B*3] se3_r[M*B*4] se3_d[M*B*4]
 * cam_q[M*4] cam_t[M*3]; zeroed here. */
SR_API int sr_bob_warp_backward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* rot, const float* o2b_q,
                                const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                const float* se3_d, const float* cam_q, const float* cam_t, const float* g_xyz_cam,
                                const float* g_rot_cam, const float* g_entropy, float* g_xyz, float* g_rot, float* g_delta,
                                float* g_tables, void* stream_) {
    if (int rc = check_warp(P, B, M)) return rc;
    if (!g_tables) return sr_fail(SR_EINVAL, "sr_bob_warp_backward: g_tables is NULL");
    cudaStream_t s = (cudaStream_t)stream_;
    const size_t nt = sr_bob_warp_table_floats(B, M);
    CK(cudaMemsetAsync(g_tables, 0, nt * sizeof(float), s), "sr_bob_warp_backward: memset(g_tables)");
    if (P == 0) return 0;
    if (!xyz || !rot || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !g_xyz_cam || !g_rot_cam ||
        !g_xyz || !g_rot)
        return sr_fail(SR_EINVAL, "sr_bob_warp_backward: a required pointer is NULL");
    if (((uintptr_t)g_rot_cam & 15) || ((uintptr_t)g_rot & 15))
        return sr_fail(SR_EINVAL, "sr_bob_warp_backward: g_rot_cam and g_rot must be 16-byte aligned");
    const WarpDims d{P, B, M};
    const size_t smem = 2 * nt * sizeof(float);
    if (smem > SR_TABLE_SMEM_MAX)
        return sr_fail(SR_EINVAL, "sr_bob_warp_backward: the tables and their gradients of B = %d, M = %d frames do not fit in "
                       "shared memory", B, M);
    ProfileScope ps("bob_warp_bwd", s);
    auto launch = [&](auto kern) -> int {
        CK(sr_opt_in_smem(kern, smem), "sr_bob_warp_backward: shared-memory opt-in");
        // 128-thread blocks: the kernel holds ~200 registers per thread (B weights + B weight gradients)
        kern<<<(P + 127) / 128, 128, smem, s>>>(d, xyz, rot, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t, g_xyz_cam,
                                                 g_rot_cam, g_entropy, g_xyz, g_rot, g_delta, g_tables);
        return 0;
    };
    if (int rc = B <= 32 ? launch(bob_warp_bwd_kernel<32>) : launch(bob_warp_bwd_kernel<64>)) return rc;
    return sr_launched(1, "sr_bob_warp_backward");
}

}  // extern "C"
