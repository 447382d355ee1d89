// warp_common.cuh -- device code shared by the bob-skinning warp of the surfels (warp.cu) and of the feature-matched
// points of Stage 3's reprojection loss (match.cu): quaternion algebra, the shared-memory bone / frame tables, skinning
// weights, the sign-aligned dual-quaternion blend, their vector-Jacobian products and the warp-wide table reductions.
// See warp.cu for the reference lines each piece restates.
#pragma once
#include "common.cuh"

namespace {

struct Q4 { float w, x, y, z; };
__device__ __forceinline__ Q4 qmul(const Q4& a, const Q4& b) {
    return {a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z, a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y,
            a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x, a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w};
}
__device__ __forceinline__ Q4 qconj(const Q4& q) { return {q.w, -q.x, -q.y, -q.z}; }
__device__ __forceinline__ Q4 pure(float x, float y, float z) { return {0.f, x, y, z}; }
__device__ __forceinline__ Q4 qadd(const Q4& a, const Q4& b) { return {a.w + b.w, a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ Q4 qscale(const Q4& a, float s) { return {a.w * s, a.x * s, a.y * s, a.z * s}; }
__device__ __forceinline__ float qdot(const Q4& a, const Q4& b) { return a.w * b.w + a.x * b.x + a.y * b.y + a.z * b.z; }
// v' = q v q*  (general q, as quat_transform.py:259-276)
__device__ __forceinline__ void qrot(const Q4& q, float vx, float vy, float vz, float& ox, float& oy, float& oz) {
    const Q4 t = qmul(qmul(q, pure(vx, vy, vz)), qconj(q));
    ox = t.x; oy = t.y; oz = t.z;
}
// vjp of v' = q v q*:  g_v = (q* g q)[1:],  g_q = -2 g (x) q (x) v
__device__ __forceinline__ void qrot_vjp(const Q4& q, float vx, float vy, float vz, float gx, float gy, float gz, Q4& gq,
                                         float& gvx, float& gvy, float& gvz) {
    const Q4 g = pure(gx, gy, gz);
    const Q4 t = qmul(qmul(qconj(q), g), q);
    gvx = t.x; gvy = t.y; gvz = t.z;
    gq = qscale(qmul(qmul(g, q), pure(vx, vy, vz)), -2.0f);
}
__device__ __forceinline__ Q4 ldq(const float* p) { return {p[0], p[1], p[2], p[3]}; }

struct WarpDims { int P, B, M; };

// shared-memory tables: o2b_q[B*4] o2b_t[B*3] ig[B*3] se3_r[M*B*4] se3_d[M*B*4] cam_q[M*4] cam_t[M*3]
struct Tables {
    const float *oq, *ot, *ig, *sr, *sd, *cq, *ct;
    __device__ __forceinline__ static int floats(int B, int M) { return B * 10 + M * B * 8 + M * 7; }
    __device__ __forceinline__ void bind(float* s, int B, int M) {
        oq = s; ot = oq + B * 4; ig = ot + B * 3; sr = ig + B * 3; sd = sr + M * B * 4; cq = sd + M * B * 4; ct = cq + M * 4;
    }
};

__device__ __forceinline__ void load_tables(float* s, const WarpDims d, const float* __restrict__ o2b_q, const float* __restrict__ o2b_t,
                                            const float* __restrict__ inv_gauss, const float* __restrict__ se3_r,
                                            const float* __restrict__ se3_d, const float* __restrict__ cam_q,
                                            const float* __restrict__ cam_t) {
    const int B = d.B, M = d.M;
    float* p = s;
    for (int i = threadIdx.x; i < B * 4; i += blockDim.x) p[i] = __ldg(o2b_q + i);
    p += B * 4;
    for (int i = threadIdx.x; i < B * 3; i += blockDim.x) p[i] = __ldg(o2b_t + i);
    p += B * 3;
    for (int i = threadIdx.x; i < B * 3; i += blockDim.x) p[i] = __ldg(inv_gauss + i);
    p += B * 3;
    for (int i = threadIdx.x; i < M * B * 4; i += blockDim.x) p[i] = __ldg(se3_r + i);
    p += M * B * 4;
    for (int i = threadIdx.x; i < M * B * 4; i += blockDim.x) p[i] = __ldg(se3_d + i);
    p += M * B * 4;
    for (int i = threadIdx.x; i < M * 4; i += blockDim.x) p[i] = __ldg(cam_q + i);
    p += M * 4;
    for (int i = threadIdx.x; i < M * 3; i += blockDim.x) p[i] = __ldg(cam_t + i);
}

// Skinning weights of one surfel: softmax over bones of -(|x_bone * inv_gauss|^2 + delta); also the arg-max bone and
// log-sum-exp minus max (= the cross entropy against the arg-max one-hot, loss_utils.py:21-42).
template <int BMAX>
__device__ __forceinline__ void skin_weights(const Tables& T, int B, float x, float y, float z, const float* __restrict__ delta_row,
                                             float (&w)[BMAX], int& anchor, float& entropy) {
    float mx = -3.4e38f;
#pragma unroll
    for (int b = 0; b < BMAX; b++) {
        w[b] = -3.4e38f;
        if (b < B) {
            float bx, by, bz;
            qrot(ldq(T.oq + 4 * b), x, y, z, bx, by, bz);
            bx = (bx + T.ot[3 * b]) * T.ig[3 * b]; by = (by + T.ot[3 * b + 1]) * T.ig[3 * b + 1]; bz = (bz + T.ot[3 * b + 2]) * T.ig[3 * b + 2];
            float l = -(bx * bx + by * by + bz * bz);
            if (delta_row) l -= __ldg(delta_row + b);
            w[b] = l;
            mx = fmaxf(mx, l);
        }
    }
    float Z = 0.f;
    anchor = 0;
    bool found = false;
#pragma unroll
    for (int b = 0; b < BMAX; b++) {
        if (b < B) {
            if (!found && w[b] == mx) { anchor = b; found = true; }      // first arg-max, like torch.argmax
            w[b] = expf(w[b] - mx);
            Z += w[b];
        } else w[b] = 0.f;
    }
    const float inv = 1.0f / Z;
#pragma unroll
    for (int b = 0; b < BMAX; b++) w[b] *= inv;
    entropy = logf(Z);
}

// sign-aligned dual-quaternion blend of frame m (geom_utils.py:66-83): returns the un-normalised QR, QD
template <int BMAX>
__device__ __forceinline__ void blend(const Tables& T, int B, int m, const float (&w)[BMAX], int anchor, Q4& QR, Q4& QD) {
    const float* sr = T.sr + (size_t)m * B * 4;
    const float* sd = T.sd + (size_t)m * B * 4;
    const Q4 qa = ldq(sr + 4 * anchor);
    QR = {0.f, 0.f, 0.f, 0.f}; QD = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int b = 0; b < BMAX; b++) {
        if (b < B) {
            const Q4 r = ldq(sr + 4 * b), dq = ldq(sd + 4 * b);
            const float s = (qdot(qa, r) > 0.f ? 1.f : -1.f) * w[b];
            QR = qadd(QR, qscale(r, s)); QD = qadd(QD, qscale(dq, s));
        }
    }
}

// Recursive-halving warp reduction of 32 values: lane L ends with the sum over the warp of v[L].  31 shuffles for 32
// sums (a plain shuffle tree needs 5 per value) and the 32 results land one per lane, so the shared-memory accumulation
// that follows is ONE conflict-free atomic instruction instead of 32 single-lane ones.
__device__ __forceinline__ float butterfly32(float (&v)[32], int lane) {
#pragma unroll
    for (int off = 16, n = 16; off >= 1; off >>= 1, n >>= 1) {
        const bool hi = lane & off;
#pragma unroll
        for (int i = 0; i < 16; i++) {
            if (i < n) {
                const float keep = hi ? v[i + n] : v[i], send = hi ? v[i] : v[i + n];
                v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
            }
        }
    }
    return v[0];
}

// warp sum, then one shared-memory add per warp (only the 8 warps of a block contend on an address)
__device__ __forceinline__ void acc_table(float* slot, float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0 && v != 0.f) atomicAdd(slot, v);
}
__device__ __forceinline__ void acc_q(float* slot, const Q4& q) {
    acc_table(slot, q.w); acc_table(slot + 1, q.x); acc_table(slot + 2, q.y); acc_table(slot + 3, q.z);
}

// vjp of the blend of frame m: adds dL/dw[b] to gw and reduces dL/dse3_r, dL/dse3_d of frame m over the warp into the
// shared-memory gradients g_sr, g_sd (layout of Tables).  Every lane of the warp must call it (dead lanes with zeros).
template <int BMAX>
__device__ __forceinline__ void blend_vjp(const Tables& T, int B, int m, const float (&w)[BMAX], int anchor, const Q4& gQR,
                                          const Q4& gQD, float (&gw)[BMAX], float* g_sr, float* g_sd) {
    const float* sr = T.sr + (size_t)m * B * 4;
    const float* sd = T.sd + (size_t)m * B * 4;
    const Q4 qa = ldq(sr + 4 * anchor);
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int c4 = 0; c4 < BMAX / 4; c4++) {
        if (4 * c4 < B) {                                        // four bones x (4 + 4) components = 32 sums per butterfly
            float vals[32];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const int b = 4 * c4 + j;
                float ws = 0.f;
                if (b < B) {
                    const Q4 rb = ldq(sr + 4 * b), db = ldq(sd + 4 * b);
                    const float s = qdot(qa, rb) > 0.f ? 1.f : -1.f;
                    gw[b] += s * (qdot(gQR, rb) + qdot(gQD, db));
                    ws = w[b] * s;
                }
                vals[8 * j] = gQR.w * ws; vals[8 * j + 1] = gQR.x * ws; vals[8 * j + 2] = gQR.y * ws; vals[8 * j + 3] = gQR.z * ws;
                vals[8 * j + 4] = gQD.w * ws; vals[8 * j + 5] = gQD.x * ws; vals[8 * j + 6] = gQD.y * ws; vals[8 * j + 7] = gQD.z * ws;
            }
            const float tot = butterfly32(vals, lane);
            const int b = 4 * c4 + (lane >> 3), comp = lane & 7;
            if (b < B && tot != 0.f)
                atomicAdd((comp < 4 ? g_sr : g_sd) + ((size_t)m * B + b) * 4 + (comp & 3), tot);
        }
    }
}

// vjp of the skinning weights of point ps given dL/dw (gw) and dL/dentropy (ge; 0 on a dead lane): softmax, then the
// Gaussian logits.  Writes dL/ddelta to g_delta[ps*B..] (if non-NULL), plus g_d2 * delta_row[b] where delta also feeds a
// term in delta^2 (delta_row non-NULL), adds dL/dx to (gxx, gxy, gxz) and reduces dL/do2b_q, dL/do2b_t, dL/dinv_gauss over
// the warp into g_oq, g_ot, g_ig.  A dead lane (live = false, lv = 0) takes part with zeros: every lane of the warp must
// call it.  bob_warp_bwd_kernel keeps its own inline copy of this loop: calling this function there changes that kernel's
// instruction schedule, which is kept as it was.
template <int BMAX>
__device__ __forceinline__ void skin_vjp(const Tables& T, int B, float x, float y, float z, const float (&w)[BMAX],
                                         const float (&gw)[BMAX], int anchor, float ge, size_t ps, bool live, float lv,
                                         float* __restrict__ g_delta, const float* __restrict__ delta_row, float g_d2, float* g_oq,
                                         float* g_ot, float* g_ig, float& gxx, float& gxy, float& gxz) {
    float dotwg = 0.f;
#pragma unroll
    for (int b = 0; b < BMAX; b++) dotwg += w[b] * gw[b];
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
                    if (g_delta && live) g_delta[ps * B + b] = delta_row ? g_d2 * __ldg(delta_row + b) - gl : -gl;
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
}

}  // namespace
