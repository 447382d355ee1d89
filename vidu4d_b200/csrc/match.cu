// match.cu -- Stage 3's feature-matching reprojection loss ("feat_reproj"), forward and backward (DESIGN.md section 3.5b).
//
// Replaces (behaviour, not code) of the reference's PyTorch chain
//   lab4d/nnutils/deformable_gaussian.py:1436-1486   global_match: scores against C sampled candidates, top-K, softmax at
//                                                    temperature exp(logsigma), prob-weighted canonical xyz
//   lab4d/nnutils/deformable_gaussian.py:1488-1513   forward_project: forward_warp of the matched points (no rotation)
//   lab4d/utils/geom_utils.py:17-30                  pinhole_projection  K x / (z + 1e-6)
//   lab4d/engine/model.py:669-672,915,961-967,994-1012   ||xy_reproj - hxy[..., :2]|| * mask * is_detected, reduced as
//                                                    the mean over the batch's positive values / train_res * feat_reproj_wt
// The reference materialises the (M*H*W, C) fp32 score matrix (1.07 GB at 256^2 x 2 frames x 2048 candidates) and a
// second one of that size in topk's backward.  Here match_fwd streams the candidates through shared memory and keeps a
// sorted top-K per pixel in registers; only K (position, prob, score) triples per pixel reach HBM.
//
// match_fwd   one thread per pixel: 16 features in registers; candidate feature rows gathered (candidate c is surfel
//             cand[c] mod P) into a double-buffered shared-memory ring with cp.async.  Each score is one fp32 FMA chain
//             over the 16 channels in channel order.  Top-K order: larger score first; among EQUAL scores the lower
//             candidate position first (a later candidate never displaces an equal earlier one).  Candidate indices
//             outside [0, M*P) are skipped (their rows are staged as NaN, which never enters the top-K).
// match_bwd   one thread per pixel over the saved top-K; dL/dfeat_cand and dL/dxyz_cand go to a (C,19) shared-memory
//             accumulator per CTA, flushed once per CTA (persistent grid); dL/dlogsigma is block-reduced.  When (C,19)
//             floats exceed the device's opt-in shared memory, a second instantiation adds them to g_cand directly.
// match_scatter adds the (C,19) candidate rows into g_regist_feat (P,16) / g_xyz (P,3) at cand[c] mod P (duplicates sum).
// reproj_fwd  one thread per pixel: skinning weights of the matched point, frame m's dual-quaternion blend, field2cam,
//             the frame's K; per-frame sums and integer counts of v > 0 (block reduction + per-frame atomics).
// reproj_scale one CTA: s = w / (count * train_res) (0 when the batch-wide count is 0), scales the terms, writes the loss.
// reproj_bwd  one thread per pixel: projection VJP, single-point warp VJP (warp_common.cuh); dL/dxyz_matched and dL/ddelta
//             written directly, table gradients reduced butterfly -> shared memory -> one global atomic per value and CTA.
#include <algorithm>

#include "warp_common.cuh"

namespace {

constexpr int FEAT = 16;                // width of the registration feature
constexpr int KMAX = 8;                 // largest num_grad
constexpr int ROW = FEAT + 3;           // candidate gradient row: feature 16, xyz 3
constexpr int MATCH_THREADS = 256;
constexpr int CHUNK = 256;              // candidate rows per shared-memory stage
constexpr int BWD_THREADS = 1024;
constexpr int REPROJ_THREADS = 128;

__device__ __forceinline__ void cp_async4(float* dst, const float* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1() { asm volatile("cp.async.wait_group 1;\n" ::: "memory"); }

struct MatchDims {
    long long N;         // pixels M*H*W
    int P, C, K;
    long long MP;        // M*P: valid candidate indices
};

// stage candidate rows [base, base + CHUNK) of the gathered (C,16) feature matrix into `rows`
__device__ __forceinline__ void stage_rows(float* rows, const MatchDims d, int base, const float* __restrict__ regist_feat,
                                           const int32_t* __restrict__ cand) {
    for (int e = threadIdx.x; e < CHUNK * FEAT; e += blockDim.x) {
        const int r = e / FEAT, c = base + r;
        if (c >= d.C) continue;
        const long long idx = __ldg(cand + c);
        if (idx < 0 || idx >= d.MP) rows[e] = __int_as_float(0x7fffffff);          // NaN: never enters the top-K
        else cp_async4(rows + e, regist_feat + (idx % d.P) * FEAT + (e % FEAT));
    }
}

__global__ void __launch_bounds__(MATCH_THREADS)
match_fwd_kernel(const MatchDims d, const float* __restrict__ feat_px, const float* __restrict__ regist_feat,
                 const float* __restrict__ xyz, const int32_t* __restrict__ cand, const float* __restrict__ logsigma,
                 float* __restrict__ xyz_matched, int32_t* __restrict__ top_idx, float* __restrict__ top_prob,
                 float* __restrict__ top_score) {
    __shared__ __align__(16) float rows[2][CHUNK * FEAT];
    const long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = n < d.N;
    float f[FEAT];
#pragma unroll
    for (int c = 0; c < FEAT; c++) f[c] = live ? __ldg(feat_px + n * FEAT + c) : 0.f;
    // sorted descending; the KMAX - K leading slots hold +inf (never displaced), so the top-K are v[KMAX-K .. KMAX-1] and
    // the entry threshold is always v[KMAX-1] (a static register, no indexed local-memory array)
    float v[KMAX];
    int id[KMAX];
#pragma unroll
    for (int k = 0; k < KMAX; k++) {
        const bool pad = k < KMAX - d.K;
        v[k] = pad ? INFINITY : -INFINITY; id[k] = pad ? -1 : INT_MAX;
    }
    const int nchunks = (d.C + CHUNK - 1) / CHUNK;
    stage_rows(rows[0], d, 0, regist_feat, cand);
    cp_async_commit();
    for (int ch = 0; ch < nchunks; ch++) {
        if (ch + 1 < nchunks) stage_rows(rows[(ch + 1) & 1], d, (ch + 1) * CHUNK, regist_feat, cand);
        cp_async_commit();
        cp_async_wait1();
        __syncthreads();
        const float4* R = reinterpret_cast<const float4*>(rows[ch & 1]);
        const int base = ch * CHUNK, nr = min(CHUNK, d.C - base);
        for (int r = 0; r < nr; r++) {
            const float4 a = R[4 * r], b = R[4 * r + 1], c = R[4 * r + 2], e = R[4 * r + 3];
            float s = f[0] * a.x;
            s = fmaf(f[1], a.y, s); s = fmaf(f[2], a.z, s); s = fmaf(f[3], a.w, s);
            s = fmaf(f[4], b.x, s); s = fmaf(f[5], b.y, s); s = fmaf(f[6], b.z, s); s = fmaf(f[7], b.w, s);
            s = fmaf(f[8], c.x, s); s = fmaf(f[9], c.y, s); s = fmaf(f[10], c.z, s); s = fmaf(f[11], c.w, s);
            s = fmaf(f[12], e.x, s); s = fmaf(f[13], e.y, s); s = fmaf(f[14], e.z, s); s = fmaf(f[15], e.w, s);
            if (s > v[KMAX - 1]) {                                   // rare after the first rows: ~K ln(C/K) insertions
                float cs = s;
                int ci = base + r;
#pragma unroll
                for (int k = 0; k < KMAX; k++) {                     // carry the displaced entry down the sorted list
                    if (cs > v[k] || (cs == v[k] && ci < id[k])) {
                        const float tv = v[k]; const int ti = id[k];
                        v[k] = cs; id[k] = ci; cs = tv; ci = ti;
                    }
                }
            }
        }
        __syncthreads();                                             // the buffer is refilled two chunks later
    }
    if (!live) return;
    const int k0 = KMAX - d.K;                                       // slot of the best candidate
    const float tau = expf(__ldg(logsigma));
    float mx = 0.f;
#pragma unroll
    for (int j = 0; j < KMAX; j++) if (j == k0) mx = v[j] * tau;
    float e[KMAX], Z = 0.f;
#pragma unroll
    for (int j = 0; j < KMAX; j++) {
        e[j] = (j >= k0 && id[j] != INT_MAX) ? expf(v[j] * tau - mx) : 0.f;
        Z += e[j];
    }
    const float iz = Z > 0.f ? 1.f / Z : 0.f;
    float ox = 0.f, oy = 0.f, oz = 0.f;
#pragma unroll
    for (int j = 0; j < KMAX; j++) {
        if (j >= k0) {
            const bool ok = id[j] != INT_MAX;
            const float p = e[j] * iz;
            if (ok) {
                const long long sidx = (long long)__ldg(cand + id[j]) % d.P;
                ox += p * __ldg(xyz + 3 * sidx); oy += p * __ldg(xyz + 3 * sidx + 1); oz += p * __ldg(xyz + 3 * sidx + 2);
            }
            const long long o = n * d.K + (j - k0);
            top_idx[o] = ok ? id[j] : -1;
            top_prob[o] = p;
            top_score[o] = ok ? v[j] : 0.f;
        }
    }
    xyz_matched[3 * n] = ox; xyz_matched[3 * n + 1] = oy; xyz_matched[3 * n + 2] = oz;
}

// SMEM: the (C,19) rows are summed in shared memory and flushed once per CTA.  Without it (C * 19 floats beyond the
// device's opt-in shared memory) every product goes straight to g_cand with a global atomic.
template <bool SMEM>
__global__ void __launch_bounds__(BWD_THREADS)
match_bwd_kernel(const MatchDims d, const float* __restrict__ feat_px, const float* __restrict__ xyz,
                 const int32_t* __restrict__ cand, const float* __restrict__ logsigma, const int32_t* __restrict__ top_idx,
                 const float* __restrict__ top_prob, const float* __restrict__ top_score,
                 const float* __restrict__ g_xyz_matched, float* __restrict__ g_cand, float* __restrict__ g_logsigma) {
    extern __shared__ float acc_smem[];                              // (C,19) candidate gradient rows of this CTA
    __shared__ float red[BWD_THREADS / 32];
    float* const acc = SMEM ? acc_smem : g_cand;
    if constexpr (SMEM) {
        for (int i = threadIdx.x; i < d.C * ROW; i += blockDim.x) acc[i] = 0.f;
        __syncthreads();
    }
    const float tau = expf(__ldg(logsigma));
    float glog = 0.f;
    for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < d.N; n += (long long)gridDim.x * blockDim.x) {
        const float gx = g_xyz_matched[3 * n], gy = g_xyz_matched[3 * n + 1], gz = g_xyz_matched[3 * n + 2];
        if (gx == 0.f && gy == 0.f && gz == 0.f) continue;          // masked-out pixels: nothing to add
        int id[KMAX];
        float p[KMAX], gp[KMAX], dot = 0.f;
#pragma unroll
        for (int k = 0; k < KMAX; k++) {
            id[k] = k < d.K ? top_idx[n * d.K + k] : -1;
            p[k] = 0.f; gp[k] = 0.f;
            if (id[k] >= 0) {
                const long long sidx = (long long)__ldg(cand + id[k]) % d.P;
                p[k] = top_prob[n * d.K + k];
                gp[k] = gx * __ldg(xyz + 3 * sidx) + gy * __ldg(xyz + 3 * sidx + 1) + gz * __ldg(xyz + 3 * sidx + 2);
                dot += p[k] * gp[k];
            }
        }
        float f[FEAT];
#pragma unroll
        for (int c = 0; c < FEAT; c++) f[c] = __ldg(feat_px + n * FEAT + c);
#pragma unroll
        for (int k = 0; k < KMAX; k++) {
            if (id[k] >= 0) {
                const float ds = p[k] * (gp[k] - dot);               // dL / d(score * tau)
                glog += ds * tau * top_score[n * d.K + k];
                const float gs = ds * tau;                           // dL / dscore
                float* row = acc + id[k] * ROW;
#pragma unroll
                for (int c = 0; c < FEAT; c++) atomicAdd(row + c, gs * f[c]);
                atomicAdd(row + FEAT, p[k] * gx); atomicAdd(row + FEAT + 1, p[k] * gy); atomicAdd(row + FEAT + 2, p[k] * gz);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) glog += __shfl_xor_sync(0xffffffffu, glog, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = glog;
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) t += red[w];
        if (t != 0.f) atomicAdd(g_logsigma, t);
    }
    if constexpr (SMEM) {
        for (int i = threadIdx.x; i < d.C * ROW; i += blockDim.x)
            if (acc[i] != 0.f) atomicAdd(g_cand + i, acc[i]);
    }
}

__global__ void __launch_bounds__(256)
match_scatter_kernel(const MatchDims d, const int32_t* __restrict__ cand, const float* __restrict__ g_cand,
                     float* __restrict__ g_regist_feat, float* __restrict__ g_xyz) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= d.C * ROW) return;
    const int c = i / ROW, comp = i - c * ROW;
    const long long idx = __ldg(cand + c);
    const float g = g_cand[i];
    if (idx < 0 || idx >= d.MP || g == 0.f) return;
    const long long s = idx % d.P;
    if (comp < FEAT) atomicAdd(g_regist_feat + s * FEAT + comp, g);
    else atomicAdd(g_xyz + s * 3 + (comp - FEAT), g);
}

struct ReprojDims { int M, HW, B, hs; };   // hs: last dimension of hxy (2 or 3)

// the matched point x of frame m in camera space, projected: also returns what the backward needs
template <int BMAX>
__device__ __forceinline__ void reproj_point(const Tables& T, const ReprojDims d, int m, float x, float y, float z,
                                             const float* __restrict__ delta_row, const float* __restrict__ Km, float (&w)[BMAX],
                                             int& anchor, Q4& q, Q4& qd, float& inv, float (&xt)[3], float (&xc)[3],
                                             float (&h)[3], float& u, float& v) {
    float ent;
    skin_weights<BMAX>(T, d.B, x, y, z, delta_row, w, anchor, ent);
    Q4 QR, QD;
    blend<BMAX>(T, d.B, m, w, anchor, QR, QD);
    inv = rsqrtf(qdot(QR, QR));
    q = qscale(QR, inv); qd = qscale(QD, inv);
    const Q4 t4 = qmul(qd, qconj(q));                               // t = 2 (qd (x) q*)[1:]
    qrot(q, x, y, z, xt[0], xt[1], xt[2]);
    xt[0] += 2.f * t4.x; xt[1] += 2.f * t4.y; xt[2] += 2.f * t4.z;
    qrot(ldq(T.cq + 4 * m), xt[0], xt[1], xt[2], xc[0], xc[1], xc[2]);
    xc[0] += T.ct[3 * m]; xc[1] += T.ct[3 * m + 1]; xc[2] += T.ct[3 * m + 2];
#pragma unroll
    for (int i = 0; i < 3; i++) h[i] = __ldg(Km + 3 * i) * xc[0] + __ldg(Km + 3 * i + 1) * xc[1] + __ldg(Km + 3 * i + 2) * xc[2];
    const float den = h[2] + 1e-6f;
    u = h[0] / den; v = h[1] / den;
}

template <int BMAX>
__global__ void __launch_bounds__(REPROJ_THREADS)
reproj_fwd_kernel(const ReprojDims d, const float* __restrict__ xyz_m, const float* __restrict__ o2b_q,
                  const float* __restrict__ o2b_t, const float* __restrict__ inv_gauss, const float* __restrict__ delta,
                  const float* __restrict__ se3_r, const float* __restrict__ se3_d, const float* __restrict__ cam_q,
                  const float* __restrict__ cam_t, const float* __restrict__ Kmat, const float* __restrict__ hxy,
                  const float* __restrict__ mask, const float* __restrict__ is_detected, float* __restrict__ xy_reproj,
                  float* __restrict__ terms, uint32_t* __restrict__ counts) {
    extern __shared__ float smem[];
    const int m = blockIdx.y;
    load_tables(smem, WarpDims{0, d.B, d.M}, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t);
    __syncthreads();
    Tables T; T.bind(smem, d.B, d.M);
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    float part = 0.f;
    uint32_t cnt = 0u;
    if (i < d.HW) {
        const size_t n = (size_t)m * d.HW + i;
        float w[BMAX], xt[3], xc[3], h[3], u, v, inv;
        int anchor; Q4 q, qd;
        reproj_point<BMAX>(T, d, m, xyz_m[3 * n], xyz_m[3 * n + 1], xyz_m[3 * n + 2], delta ? delta + n * d.B : nullptr,
                           Kmat + 9 * m, w, anchor, q, qd, inv, xt, xc, h, u, v);
        xy_reproj[2 * n] = u; xy_reproj[2 * n + 1] = v;
        const float dx = u - hxy[n * d.hs], dy = v - hxy[n * d.hs + 1];
        const float val = sqrtf(dx * dx + dy * dy) * mask[n] * (is_detected ? __ldg(is_detected + m) : 1.f);
        const bool on = val > 0.f;
        part = on ? val : 0.f;
        cnt = on;
    }
    // block reduction as in feat_loss_kernel (loss.cu): one float and one integer atomic per CTA
    __shared__ float red[REPROJ_THREADS / 32];
    __shared__ uint32_t redc[REPROJ_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        part += __shfl_xor_sync(0xffffffffu, part, o);
        cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    }
    if ((threadIdx.x & 31) == 0) { red[threadIdx.x >> 5] = part; redc[threadIdx.x >> 5] = cnt; }
    __syncthreads();
    if (threadIdx.x == 0) {
        float t = 0.f;
        uint32_t c = 0u;
#pragma unroll
        for (int w = 0; w < REPROJ_THREADS / 32; w++) { t += red[w]; c += redc[w]; }
        if (c) { atomicAdd(terms + m, t); atomicAdd(counts + m, c); }
    }
}

// s = w / (C * train_res) with C the count over the whole batch (the reference's v[v > 0].mean() / train_res * wt)
__global__ void reproj_scale_kernel(int M, float train_res, const float* __restrict__ weight, const uint32_t* __restrict__ counts,
                                    float* __restrict__ terms, float* __restrict__ scale, float* __restrict__ loss) {
    if (threadIdx.x != 0) return;
    unsigned long long c = 0;
    for (int m = 0; m < M; m++) c += counts[m];
    const float s = c ? __ldg(weight) / ((float)c * train_res) : 0.f;
    float l = 0.f;
    for (int m = 0; m < M; m++) { terms[m] *= s; l += terms[m]; }
    *scale = s;
    *loss = l;
}

template <int BMAX>
__global__ void __launch_bounds__(REPROJ_THREADS)
reproj_bwd_kernel(const ReprojDims d, const float* __restrict__ xyz_m, const float* __restrict__ o2b_q,
                  const float* __restrict__ o2b_t, const float* __restrict__ inv_gauss, const float* __restrict__ delta,
                  const float* __restrict__ se3_r, const float* __restrict__ se3_d, const float* __restrict__ cam_q,
                  const float* __restrict__ cam_t, const float* __restrict__ Kmat, const float* __restrict__ hxy,
                  const float* __restrict__ mask, const float* __restrict__ is_detected, const float* __restrict__ scale,
                  const float* __restrict__ g_loss, float* __restrict__ g_xyz_m, float* __restrict__ g_delta,
                  float* __restrict__ g_tables) {
    extern __shared__ float smem[];
    const int B = d.B, M = d.M, m = blockIdx.y, nt = Tables::floats(B, M);
    load_tables(smem, WarpDims{0, B, M}, o2b_q, o2b_t, inv_gauss, se3_r, se3_d, cam_q, cam_t);
    float* gacc = smem + nt;                                        // gradient of every table entry, same layout
    for (int i = threadIdx.x; i < nt; i += blockDim.x) gacc[i] = 0.f;
    __syncthreads();
    Tables T; T.bind(smem, B, M);
    float* g_oq = gacc; float* g_ot = g_oq + B * 4; float* g_ig = g_ot + B * 3; float* g_sr = g_ig + B * 3;
    float* g_sd = g_sr + M * B * 4; float* g_cq = g_sd + M * B * 4; float* g_ct = g_cq + M * 4;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = i < d.HW;                                      // dead lanes take part in the warp sums with zeros
    const size_t n = (size_t)m * d.HW + (live ? i : 0);
    const float lv = live ? 1.f : 0.f;
    const float x = xyz_m[3 * n], y = xyz_m[3 * n + 1], z = xyz_m[3 * n + 2];
    const float* Km = Kmat + 9 * m;
    float w[BMAX], gw[BMAX], xt[3], xc[3], h[3], u, v, inv;
    int anchor; Q4 q, qd;
    reproj_point<BMAX>(T, d, m, x, y, z, delta ? delta + n * B : nullptr, Km, w, anchor, q, qd, inv, xt, xc, h, u, v);
    // ---- loss: v = ||xy - hxy|| * mask * det, counted where v > 0; dL/dv = g_loss * scale there
    const float dx = u - hxy[n * d.hs], dy = v - hxy[n * d.hs + 1];
    const float nrm = sqrtf(dx * dx + dy * dy);
    const float wpx = mask[n] * (is_detected ? __ldg(is_detected + m) : 1.f);
    const float gl = (nrm * wpx > 0.f) ? __ldg(g_loss) * __ldg(scale) * wpx / nrm * lv : 0.f;
    const float gu = gl * dx, gv = gl * dy;
    // ---- projection: u = h0 / (h2 + 1e-6), v = h1 / (h2 + 1e-6), h = K xc
    const float den = h[2] + 1e-6f;
    const float dh0 = gu / den, dh1 = gv / den, dh2 = -(gu * u + gv * v) / den;
    float gc[3];
#pragma unroll
    for (int j = 0; j < 3; j++) gc[j] = __ldg(Km + j) * dh0 + __ldg(Km + 3 + j) * dh1 + __ldg(Km + 6 + j) * dh2;
    // ---- camera: xc = qc xt qc* + tc
    Q4 gqc; float gtx, gty, gtz;
    qrot_vjp(ldq(T.cq + 4 * m), xt[0], xt[1], xt[2], gc[0], gc[1], gc[2], gqc, gtx, gty, gtz);
    acc_q(g_cq + 4 * m, gqc);
    acc_table(g_ct + 3 * m, gc[0]); acc_table(g_ct + 3 * m + 1, gc[1]); acc_table(g_ct + 3 * m + 2, gc[2]);
    // ---- xt = q x q* + t, t = 2 (qd (x) q*)[1:]; normalisation q = QR / |QR|, qd = QD / |QR|
    Q4 gq; float gxx, gxy, gxz;
    qrot_vjp(q, x, y, z, gtx, gty, gtz, gq, gxx, gxy, gxz);
    const Q4 gct = pure(2.f * gtx, 2.f * gty, 2.f * gtz);
    const Q4 gqd = qmul(gct, q);
    gq = qadd(gq, qconj(qmul(qconj(qd), gct)));
    const Q4 gQD = qscale(gqd, inv);
    const Q4 gQR = qscale(qadd(gq, qscale(q, -(qdot(q, gq) + qdot(qd, gqd)))), inv);
#pragma unroll
    for (int b = 0; b < BMAX; b++) gw[b] = 0.f;
    blend_vjp<BMAX>(T, B, m, w, anchor, gQR, gQD, gw, g_sr, g_sd);
    skin_vjp<BMAX>(T, B, x, y, z, w, gw, anchor, 0.f, n, live, lv, g_delta, nullptr, 0.f, g_oq, g_ot, g_ig, gxx, gxy, gxz);
    if (live) { g_xyz_m[3 * n] = gxx; g_xyz_m[3 * n + 1] = gxy; g_xyz_m[3 * n + 2] = gxz; }
    __syncthreads();
    for (int j = threadIdx.x; j < nt; j += blockDim.x)
        if (gacc[j] != 0.f) atomicAdd(g_tables + j, gacc[j]);
}

int check_match(int32_t M, int32_t H, int32_t W, int32_t P, int32_t C, int32_t K) {
    if (M < 1 || H < 1 || W < 1 || P < 1) return sr_fail(SR_EINVAL, "M, H, W and P must be >= 1");
    if (C < 1 || (long long)C > (long long)M * P) return sr_fail(SR_EINVAL, "C must be in [1, M*P], got %d", C);
    if (K < 1 || K > KMAX || K > C) return sr_fail(SR_EINVAL, "K must be in [1, min(8, C = %d)], got %d", C, K);
    return 0;
}

int check_reproj(int32_t M, int32_t H, int32_t W, int32_t B, int32_t hxy_dim, float train_res) {
    if (M < 1 || H < 1 || W < 1) return sr_fail(SR_EINVAL, "M, H and W must be >= 1");
    if (B < 1 || B > 64) return sr_fail(SR_EINVAL, "B must be in [1, 64], got %d", B);
    if (hxy_dim != 2 && hxy_dim != 3) return sr_fail(SR_EINVAL, "hxy_dim must be 2 or 3, got %d", hxy_dim);
    if (!(train_res > 0.f)) return sr_fail(SR_EINVAL, "train_res must be > 0");
    if (sr_bob_warp_table_floats(B, M) * 2 * sizeof(float) > SR_TABLE_SMEM_MAX)
        return sr_fail(SR_EINVAL, "the bone / frame tables of B = %d, M = %d frames do not fit in shared memory", B, M);
    return 0;
}

}  // namespace

extern "C" {

SR_API int sr_global_match_forward(int32_t M, int32_t H, int32_t W, int32_t P, int32_t C, int32_t K, const float* feat_px,
                                   const float* regist_feat, const float* xyz, const int32_t* cand, const float* logsigma,
                                   float* xyz_matched, int32_t* top_idx, float* top_prob, float* top_score, void* stream_) {
    if (int rc = check_match(M, H, W, P, C, K)) return rc;
    if (!feat_px || !regist_feat || !xyz || !cand || !logsigma || !xyz_matched || !top_idx || !top_prob || !top_score)
        return sr_fail(SR_EINVAL, "sr_global_match_forward: a required pointer is NULL");
    const MatchDims d{(long long)M * H * W, P, C, K, (long long)M * P};
    cudaStream_t s = (cudaStream_t)stream_;
    {
        ProfileScope ps("match_fwd", s);
        match_fwd_kernel<<<(unsigned)((d.N + MATCH_THREADS - 1) / MATCH_THREADS), MATCH_THREADS, 0, s>>>(
            d, feat_px, regist_feat, xyz, cand, logsigma, xyz_matched, top_idx, top_prob, top_score);
    }
    return sr_launched(1, "sr_global_match_forward");
}

SR_API int sr_global_match_backward(int32_t M, int32_t H, int32_t W, int32_t P, int32_t C, int32_t K, const float* feat_px,
                                    const float* xyz, const int32_t* cand, const float* logsigma, const int32_t* top_idx,
                                    const float* top_prob, const float* top_score, const float* g_xyz_matched, float* g_cand,
                                    float* g_regist_feat, float* g_xyz, float* g_logsigma, void* stream_) {
    if (int rc = check_match(M, H, W, P, C, K)) return rc;
    if (!feat_px || !xyz || !cand || !logsigma || !top_idx || !top_prob || !top_score || !g_xyz_matched || !g_cand ||
        !g_regist_feat || !g_xyz || !g_logsigma)
        return sr_fail(SR_EINVAL, "sr_global_match_backward: a required pointer is NULL");
    const MatchDims d{(long long)M * H * W, P, C, K, (long long)M * P};
    cudaStream_t s = (cudaStream_t)stream_;
    CK(cudaMemsetAsync(g_cand, 0, (size_t)C * ROW * sizeof(float), s), "sr_global_match_backward: memset(g_cand)");
    CK(cudaMemsetAsync(g_regist_feat, 0, (size_t)P * FEAT * sizeof(float), s), "sr_global_match_backward: memset(g_regist_feat)");
    CK(cudaMemsetAsync(g_xyz, 0, (size_t)P * 3 * sizeof(float), s), "sr_global_match_backward: memset(g_xyz)");
    CK(cudaMemsetAsync(g_logsigma, 0, sizeof(float), s), "sr_global_match_backward: memset(g_logsigma)");
    int dev = 0, sms = 132, per_sm = 1, optin = 0;
    CK(cudaGetDevice(&dev), "sr_global_match_backward: cudaGetDevice");
    CK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev), "sr_global_match_backward: opt-in limit");
    cudaFuncAttributes fa{};
    CK(cudaFuncGetAttributes(&fa, match_bwd_kernel<true>), "sr_global_match_backward: cudaFuncGetAttributes");
    // the (C,19) rows fit beside the kernel's static shared memory up to C = (optin - static) / 76 (3056 on an H100)
    const bool in_smem = (size_t)C * ROW * sizeof(float) + fa.sharedSizeBytes <= (size_t)optin;
    const size_t smem = in_smem ? (size_t)C * ROW * sizeof(float) : 0;
    auto kern = in_smem ? match_bwd_kernel<true> : match_bwd_kernel<false>;
    CK(sr_opt_in_smem(kern, smem), "sr_global_match_backward: shared-memory opt-in");
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, BWD_THREADS, smem);
    // persistent grid: each CTA flushes its (C,19) rows once, so fewer, fuller CTAs mean fewer global reductions
    const long long want = (d.N + BWD_THREADS - 1) / BWD_THREADS;
    const int grid = (int)std::max(1LL, std::min(want, (long long)sms * std::max(per_sm, 1)));
    {
        ProfileScope ps(in_smem ? "match_bwd" : "match_bwd_global", s);   // the profile names the path taken
        kern<<<grid, BWD_THREADS, smem, s>>>(d, feat_px, xyz, cand, logsigma, top_idx, top_prob, top_score, g_xyz_matched,
                                             g_cand, g_logsigma);
    }
    {
        ProfileScope ps("match_scatter", s);
        match_scatter_kernel<<<(C * ROW + 255) / 256, 256, 0, s>>>(d, cand, g_cand, g_regist_feat, g_xyz);
    }
    return sr_launched(2, "sr_global_match_backward");
}

SR_API int sr_reproj_loss_forward(int32_t M, int32_t H, int32_t W, int32_t B, int32_t hxy_dim, float train_res,
                                  const float* xyz_matched, const float* o2b_q, const float* o2b_t, const float* inv_gauss,
                                  const float* delta, const float* se3_r, const float* se3_d, const float* cam_q,
                                  const float* cam_t, const float* Kmat, const float* hxy, const float* mask,
                                  const float* is_detected, const float* weight, float* xy_reproj, float* terms,
                                  uint32_t* counts, float* scale, float* loss, void* stream_) {
    if (int rc = check_reproj(M, H, W, B, hxy_dim, train_res)) return rc;
    if (!xyz_matched || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !Kmat || !hxy || !mask ||
        !weight || !xy_reproj || !terms || !counts || !scale || !loss)
        return sr_fail(SR_EINVAL, "sr_reproj_loss_forward: a required pointer is NULL");
    const ReprojDims d{M, H * W, B, hxy_dim};
    cudaStream_t s = (cudaStream_t)stream_;
    CK(cudaMemsetAsync(terms, 0, (size_t)M * sizeof(float), s), "sr_reproj_loss_forward: memset(terms)");
    CK(cudaMemsetAsync(counts, 0, (size_t)M * sizeof(uint32_t), s), "sr_reproj_loss_forward: memset(counts)");
    const size_t smem = sr_bob_warp_table_floats(B, M) * sizeof(float);
    const dim3 grid((d.HW + REPROJ_THREADS - 1) / REPROJ_THREADS, M);
    auto launch = [&](auto kern) -> int {
        CK(sr_opt_in_smem(kern, smem), "sr_reproj_loss_forward: shared-memory opt-in");
        ProfileScope ps("reproj_fwd", s);
        kern<<<grid, REPROJ_THREADS, smem, s>>>(d, xyz_matched, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t, Kmat,
                                                hxy, mask, is_detected, xy_reproj, terms, counts);
        return 0;
    };
    if (int rc = B <= 32 ? launch(reproj_fwd_kernel<32>) : launch(reproj_fwd_kernel<64>)) return rc;
    {
        ProfileScope ps("reproj_scale", s);
        reproj_scale_kernel<<<1, 32, 0, s>>>(M, train_res, weight, counts, terms, scale, loss);
    }
    return sr_launched(2, "sr_reproj_loss_forward");
}

SR_API int sr_reproj_loss_backward(int32_t M, int32_t H, int32_t W, int32_t B, int32_t hxy_dim, const float* xyz_matched,
                                   const float* o2b_q, const float* o2b_t, const float* inv_gauss, const float* delta,
                                   const float* se3_r, const float* se3_d, const float* cam_q, const float* cam_t,
                                   const float* Kmat, const float* hxy, const float* mask, const float* is_detected,
                                   const float* scale, const float* g_loss, float* g_xyz_matched, float* g_delta,
                                   float* g_tables, void* stream_) {
    if (int rc = check_reproj(M, H, W, B, hxy_dim, 1.f)) return rc;
    if (!xyz_matched || !o2b_q || !o2b_t || !inv_gauss || !se3_r || !se3_d || !cam_q || !cam_t || !Kmat || !hxy || !mask ||
        !scale || !g_loss || !g_xyz_matched || !g_tables)
        return sr_fail(SR_EINVAL, "sr_reproj_loss_backward: a required pointer is NULL");
    if (g_delta && !delta) return sr_fail(SR_EINVAL, "sr_reproj_loss_backward: g_delta without delta");
    const ReprojDims d{M, H * W, B, hxy_dim};
    cudaStream_t s = (cudaStream_t)stream_;
    const size_t nt = sr_bob_warp_table_floats(B, M);
    CK(cudaMemsetAsync(g_tables, 0, nt * sizeof(float), s), "sr_reproj_loss_backward: memset(g_tables)");
    const size_t smem = 2 * nt * sizeof(float);
    const dim3 grid((d.HW + REPROJ_THREADS - 1) / REPROJ_THREADS, M);
    auto launch = [&](auto kern) -> int {
        CK(sr_opt_in_smem(kern, smem), "sr_reproj_loss_backward: shared-memory opt-in");
        ProfileScope ps("reproj_bwd", s);
        kern<<<grid, REPROJ_THREADS, smem, s>>>(d, xyz_matched, o2b_q, o2b_t, inv_gauss, delta, se3_r, se3_d, cam_q, cam_t, Kmat,
                                                hxy, mask, is_detected, scale, g_loss, g_xyz_matched, g_delta, g_tables);
        return 0;
    };
    if (int rc = B <= 32 ? launch(reproj_bwd_kernel<32>) : launch(reproj_bwd_kernel<64>)) return rc;
    return sr_launched(1, "sr_reproj_loss_backward");
}

}  // extern "C"
