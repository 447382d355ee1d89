/*
 * surfel_oracle.c -- CPU restatement of the Gaussian-surfel rasterizer hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  This file is the *checker*: only tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / reference legs may load
 * it.  Nothing under vidu4d_b200/ may import, link or call it; the product path
 * fails loudly when its CUDA library is missing.
 *
 * It restates, in plain scalar C (fp32 arithmetic, every operation rounded on
 * its own: build with -ffp-contract=off), the algorithm of yikaiw/Vidu4D's
 * gs/submodules/diff-surfel-rasterization (abbrev. RAST below):
 *
 *   forward  preprocess   RAST/cuda_rasterizer/forward.cu:166-260
 *            T matrix     RAST/cuda_rasterizer/forward.cu:75-128
 *            AABB         RAST/cuda_rasterizer/forward.cu:133-163
 *            SH colour    RAST/cuda_rasterizer/forward.cu:20-71
 *            frustum      RAST/cuda_rasterizer/auxiliary.h:160-185
 *            quat->R      RAST/cuda_rasterizer/auxiliary.h:188-210
 *            tile rect    RAST/cuda_rasterizer/auxiliary.h:64-74
 *            scan         RAST/cuda_rasterizer/rasterizer_impl.cu:278
 *            key emit     RAST/cuda_rasterizer/rasterizer_impl.cu:70-111
 *            sort         RAST/cuda_rasterizer/rasterizer_impl.cu:301-309 (stable, low 32+bit bits)
 *            tile ranges  RAST/cuda_rasterizer/rasterizer_impl.cu:116-138,311
 *            composite    RAST/cuda_rasterizer/forward.cu:265-463
 *   backward composite    RAST/cuda_rasterizer/backward.cu:143-449
 *            AABB vjp     RAST/cuda_rasterizer/backward.cu:599-649
 *            T matrix vjp RAST/cuda_rasterizer/backward.cu:451-529
 *            quat vjp     RAST/cuda_rasterizer/auxiliary.h:213-257
 *            preprocess   RAST/cuda_rasterizer/backward.cu:533-597
 *            SH vjp       RAST/cuda_rasterizer/backward.cu:20-139
 *   markVisible           RAST/cuda_rasterizer/rasterizer_impl.cu:54-66
 *
 * Parity pinning: the reference ships NO tests / golden vectors for this path
 * (SURVEY.md section 4).  The oracle is pinned instead against outputs of the
 * unmodified reference extension itself (its sm_100a build), made by
 * tests/golden/make_golden.py and committed under tests/golden/ (see DESIGN.md).
 *
 * Numerical notes (why CPU and GPU can differ in the last ulp): the reference
 * uses MUFU-based rsqrtf() (auxiliary.h:190) and libdevice expf(); this file
 * uses 1/sqrtf and libm expf.  Binning decisions (radius ceil, tile rect
 * truncation) are evaluated exactly as the reference writes them, including the
 * accidental double-precision detour through `FilterSize` (auxiliary.h:20,
 * forward.cu:239).  Gradients are accumulated in double (the reference uses
 * unordered fp32 atomics, backward.cu:345-446), so this oracle is the more
 * accurate of the two on sums.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

#define BLOCK_X 16
#define BLOCK_Y 16
#define NEAR_PLANE_F 0.2f

static const float SH_C0 = 0.28209479177387814f;
static const float SH_C1 = 0.4886025119029199f;
static const float SH_C2[5] = {1.0925484305920792f, -1.0925484305920792f, 0.31539156525252005f,
                              -1.0925484305920792f, 0.5462742152960396f};
static const float SH_C3[7] = {-0.5900435899266435f, 2.890611442640554f, -0.4570457994644658f,
                               0.3731763325901154f, -0.4570457994644658f, 1.445305721320277f,
                               -0.5900435899266435f};

/* The reference is compiled with nvcc's default -fmad=true; where its SASS
 * contracts a*b+c into one FFMA we call fmaf() explicitly (see DESIGN.md,
 * "FMA map").  Everything else is separately rounded (-ffp-contract=off). */
#define FMA(a, b, c) fmaf((a), (b), (c))

typedef struct {
    int P, D, M;          /* surfels, active SH degree, SH coeffs per surfel in `shs` */
    int W, H;
    float tanfovx, tanfovy;
    const float *bg;      /* 3 */
    const float *means3D; /* P*3 */
    const float *shs;     /* P*M*3 or NULL */
    const float *colors_precomp; /* P*3 or NULL */
    const float *opacities;      /* P */
    const float *scales;         /* P*2 */
    const float *rotations;      /* P*4 (w,x,y,z) */
    const float *viewmatrix;     /* 16, row-vector convention stored row-major == column-major 4x4 */
    const float *projmatrix;     /* 16 (only feeds dead code in the reference) */
    const float *campos;         /* 3 */
} so_params;

typedef struct {
    int P, W, H, tiles_x, tiles_y, R, bit;
    /* per surfel ("geometry state", rasterizer_impl.cu:155-170) */
    float *depths; uint8_t *clamped; int *radii; float *means2D; float *transMat;
    float *normal_opacity; float *rgb; uint32_t *tiles_touched; uint32_t *point_offsets;
    /* per instance ("binning state", rasterizer_impl.cu:181-194) */
    uint64_t *keys_unsorted; uint32_t *values_unsorted; uint64_t *keys; uint32_t *point_list;
    /* per pixel / tile ("image state", rasterizer_impl.cu:172-179) */
    uint32_t *ranges;     /* tiles*2 */
    float *final_T;       /* 3*N: T, M1, M2 */
    uint32_t *n_contrib;  /* 2*N: last, median */
    float *out_color;     /* 3*N */
    float *out_others;    /* 8*N */
} so_state;

/* rasterizer_impl.cu:35-50 */
static uint32_t higher_msb(uint32_t n) {
    uint32_t msb = sizeof(n) * 4, step = msb;
    while (step > 1) { step /= 2; if (n >> msb) msb += step; else msb -= step; }
    if (n >> msb) msb++;
    return msb;
}

/* auxiliary.h:188-210; returns column-major R (R[c*3+r]) of the NORMALISED quaternion.
 * FMA placement follows the reference's sm_100a SASS (fwd preprocessCUDA 0x7c0-0xac0). */
static void quat_to_rotmat(const float *q, float *R) {
    /* glm names: quat.x=q[0] (w), .y=q[1] (x), .z=q[2] (y), .w=q[3] (z) */
    float n2 = FMA(q[2], q[2], FMA(q[1], q[1], FMA(q[3], q[3], q[0] * q[0])));
    float s = 1.0f / sqrtf(n2); /* reference: rsqrtf() == MUFU.RSQ, may differ in the last ulp */
    float w = q[0] * s, x = q[1] * s, y = q[2] * s, z = q[3] * s;
    float wz = w * z, wy = w * y, wx = w * x, yy = y * y, zz = z * z;
    float t;
    t = yy + zz;          R[0] = 1.f - (t + t);
    t = FMA(x, y, wz);    R[1] = t + t;
    t = FMA(x, z, -wy);   R[2] = t + t;
    t = FMA(x, y, -wz);   R[3] = t + t;
    t = FMA(x, x, zz);    R[4] = 1.f - (t + t);
    t = FMA(y, z, wx);    R[5] = t + t;
    t = FMA(x, z, wy);    R[6] = t + t;
    t = FMA(y, z, -wx);   R[7] = t + t;
    t = FMA(x, x, yy);    R[8] = 1.f - (t + t);
}

/* W (3x3 of the view matrix, column-major cols = viewmat[0..2],[4..6],[8..10]) times v */
static void W_mul(const float *vm, const float *v, float *o) {
    /* glm mat3*vec3, contracted as in the reference SASS: fma(m[2][r],v.z, fma(m[0][r],v.x, m[1][r]*v.y)) */
    o[0] = FMA(v[2], vm[8], FMA(v[0], vm[0], v[1] * vm[4]));
    o[1] = FMA(v[2], vm[9], FMA(v[0], vm[1], v[1] * vm[5]));
    o[2] = FMA(v[2], vm[10], FMA(v[0], vm[2], v[1] * vm[6]));
}
static void Wt_mul(const float *vm, const float *v, float *o) {
    o[0] = vm[0] * v[0] + vm[1] * v[1] + vm[2] * v[2];
    o[1] = vm[4] * v[0] + vm[5] * v[1] + vm[6] * v[2];
    o[2] = vm[8] * v[0] + vm[9] * v[1] + vm[10] * v[2];
}

/* forward.cu:75-128. Returns 0 if culled (cos==0). T: rows Tu,Tv,Tw. */
static int compute_transmat(const float *p_world, const float *quat, const float *scale,
                            const float *vm, float fx, float fy, float cx, float cy,
                            float *T, float *normal) {
    float p_view[3], Rq[9], M0[3], M1[3], tn[3], c0[3], c1[3];
    W_mul(vm, p_world, p_view);
    p_view[0] += vm[12]; p_view[1] += vm[13]; p_view[2] += vm[14];
    quat_to_rotmat(quat, Rq);
    for (int r = 0; r < 3; r++) { c0[r] = Rq[r] * scale[0]; c1[r] = Rq[3 + r] * scale[1]; }
    W_mul(vm, c0, M0);
    W_mul(vm, c1, M1);
    W_mul(vm, Rq + 6, tn);
    float cosv = FMA(-p_view[2], tn[2], FMA(p_view[1], -tn[1], -(p_view[0] * tn[0])));
    if (cosv == 0.0f) return 0;
    float mult = cosv > 0 ? 1.f : -1.f;
    tn[0] *= mult; tn[1] *= mult; tn[2] *= mult;
    /* T = (K [M0 M1 p_view; 0 0 1])^T with K=[[fx,0,cx],[0,fy,cy],[0,0,1]]; SASS 0xed0-0x10e0 */
    T[0] = FMA(M0[2], cx, fx * M0[0]);
    T[1] = FMA(M1[2], cx, fx * M1[0]);
    T[2] = FMA(p_view[2], cx, fx * p_view[0]);
    T[3] = FMA(M0[2], cy, fy * M0[1]);
    T[4] = FMA(M1[2], cy, fy * M1[1]);
    T[5] = FMA(p_view[2], cy, fy * p_view[1]);
    T[6] = M0[2]; T[7] = M1[2]; T[8] = p_view[2];
    normal[0] = tn[0]; normal[1] = tn[1]; normal[2] = tn[2];
    return 1;
}

/* forward.cu:133-163 */
static int compute_aabb(const float *T, float *center, float *extent) {
    const float *Tu = T, *Tv = T + 3, *Tw = T + 6;
    /* SASS 0x1280-0x15f0 of the reference's fwd preprocessCUDA */
    float d = FMA(-Tw[2], Tw[2], FMA(Tw[0], Tw[0], Tw[1] * Tw[1]));
    if (d == 0.0f) return 0;
    float r = 1.0f / d;
    float px = FMA(Tu[2] * Tw[2], -r, FMA(Tu[1] * Tw[1], r, (Tu[0] * Tw[0]) * r));
    float py = FMA(Tv[2] * Tw[2], -r, FMA(Tv[1] * Tw[1], r, (Tv[0] * Tw[0]) * r));
    float nqx = FMA(Tu[2] * Tu[2], r, -FMA(Tu[1] * Tu[1], r, (Tu[0] * Tu[0]) * r)); /* = -dot(f,Tu*Tu) */
    float nqy = FMA(Tv[2] * Tv[2], r, -FMA(Tv[1] * Tv[1], r, (Tv[0] * Tv[0]) * r));
    float h0x = FMA(px, px, nqx), h0y = FMA(py, py, nqy);
    center[0] = px; center[1] = py;
    extent[0] = sqrtf(fmaxf(0.0f, h0x));
    extent[1] = sqrtf(fmaxf(0.0f, h0y));
    return 1;
}

/* auxiliary.h:64-74 */
static void get_rect(const float *p, int max_radius, int gx, int gy, uint32_t *rmin, uint32_t *rmax) {
    float r = (float)max_radius;
    int x0 = (int)((p[0] - r) / (float)BLOCK_X), y0 = (int)((p[1] - r) / (float)BLOCK_Y);
    int x1 = (int)((p[0] + r + (float)BLOCK_X - 1.f) / (float)BLOCK_X);
    int y1 = (int)((p[1] + r + (float)BLOCK_Y - 1.f) / (float)BLOCK_Y);
    if (x0 < 0) x0 = 0; if (y0 < 0) y0 = 0; if (x1 < 0) x1 = 0; if (y1 < 0) y1 = 0;
    rmin[0] = (uint32_t)x0 < (uint32_t)gx ? (uint32_t)x0 : (uint32_t)gx;
    rmin[1] = (uint32_t)y0 < (uint32_t)gy ? (uint32_t)y0 : (uint32_t)gy;
    rmax[0] = (uint32_t)x1 < (uint32_t)gx ? (uint32_t)x1 : (uint32_t)gx;
    rmax[1] = (uint32_t)y1 < (uint32_t)gy ? (uint32_t)y1 : (uint32_t)gy;
}

/* forward.cu:20-71 */
static void sh_to_rgb(int idx, int deg, int M, const float *means, const float *campos,
                      const float *shs, uint8_t *clamped, float *rgb) {
    float dx = means[3 * idx] - campos[0], dy = means[3 * idx + 1] - campos[1], dz = means[3 * idx + 2] - campos[2];
    float len = sqrtf(dx * dx + dy * dy + dz * dz);
    float x = dx / len, y = dy / len, z = dz / len;
    const float *sh = shs + (size_t)idx * M * 3;
    for (int c = 0; c < 3; c++) {
        float r = SH_C0 * sh[c];
        if (deg > 0) {
            r = r - SH_C1 * y * sh[3 + c] + SH_C1 * z * sh[6 + c] - SH_C1 * x * sh[9 + c];
            if (deg > 1) {
                float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
                r = r + SH_C2[0] * xy * sh[12 + c] + SH_C2[1] * yz * sh[15 + c] +
                    SH_C2[2] * (2.0f * zz - xx - yy) * sh[18 + c] + SH_C2[3] * xz * sh[21 + c] +
                    SH_C2[4] * (xx - yy) * sh[24 + c];
                if (deg > 2) {
                    r = r + SH_C3[0] * y * (3.0f * xx - yy) * sh[27 + c] + SH_C3[1] * xy * z * sh[30 + c] +
                        SH_C3[2] * y * (4.0f * zz - xx - yy) * sh[33 + c] +
                        SH_C3[3] * z * (2.0f * zz - 3.0f * xx - 3.0f * yy) * sh[36 + c] +
                        SH_C3[4] * x * (4.0f * zz - xx - yy) * sh[39 + c] +
                        SH_C3[5] * z * (xx - yy) * sh[42 + c] + SH_C3[6] * x * (xx - 3.0f * yy) * sh[45 + c];
                }
            }
        }
        r += 0.5f;
        clamped[3 * idx + c] = (r < 0);
        rgb[3 * idx + c] = r < 0.0f ? 0.0f : r;
    }
}

static void radix_sort_pairs(const uint64_t *kin, const uint32_t *vin, uint64_t *kout, uint32_t *vout,
                             size_t n, int end_bit) {
    /* stable LSD radix sort on bits [0,end_bit): same permutation as cub::DeviceRadixSort::SortPairs */
    uint64_t *ka = (uint64_t *)malloc(n * 8 + 8), *kb = (uint64_t *)malloc(n * 8 + 8);
    uint32_t *va = (uint32_t *)malloc(n * 4 + 4), *vb = (uint32_t *)malloc(n * 4 + 4);
    memcpy(ka, kin, n * 8); memcpy(va, vin, n * 4);
    for (int shift = 0; shift < end_bit; shift += 8) {
        int nb = end_bit - shift < 8 ? end_bit - shift : 8;
        uint32_t mask = (1u << nb) - 1;
        size_t cnt[257]; memset(cnt, 0, sizeof(cnt));
        for (size_t i = 0; i < n; i++) cnt[((ka[i] >> shift) & mask) + 1]++;
        for (int b = 0; b < 256; b++) cnt[b + 1] += cnt[b];
        for (size_t i = 0; i < n; i++) { size_t d = cnt[(ka[i] >> shift) & mask]++; kb[d] = ka[i]; vb[d] = va[i]; }
        uint64_t *tk = ka; ka = kb; kb = tk; uint32_t *tv = va; va = vb; vb = tv;
    }
    memcpy(kout, ka, n * 8); memcpy(vout, va, n * 4);
    free(ka); free(kb); free(va); free(vb);
}

void so_free(so_state *s) {
    if (!s) return;
    free(s->depths); free(s->clamped); free(s->radii); free(s->means2D); free(s->transMat);
    free(s->normal_opacity); free(s->rgb); free(s->tiles_touched); free(s->point_offsets);
    free(s->keys_unsorted); free(s->values_unsorted); free(s->keys); free(s->point_list);
    free(s->ranges); free(s->final_T); free(s->n_contrib); free(s->out_color); free(s->out_others);
    free(s);
}

/*
 * ---- error analysis shared by the knife mask and the rounding-error bounds ----
 *
 * With the per-surfel records taken from the GPU, the only inputs of a pair's arithmetic that can differ between the GPU
 * and this file are G = exp(power) and whatever depends on it.  The ray/splat intersection, rho3d, rho2d, the depth, the
 * rho3d <= rho2d branch and the near-plane test are the same fp32 operations on the same bits on both sides (the GPU's
 * two-division helper is bit-identical to `/`), so they are not knife edges.
 *
 * expf: libdevice expf is within 2 ulp, glibc's within 1 ulp, so the two G differ by at most 3 ulp <= 6u (u = 2^-24,
 * the unit roundoff).  alpha = fl(opacity * G) adds one rounding on each side: |d alpha| <= SO_EU * alpha with
 * SO_EU = 8 (units of u).  1 - alpha then differs by SO_EU u alpha, i.e. SO_EU u alpha / (1 - alpha) relative, and the
 * product T (1 - alpha) adds one rounding on each side; 2 + 8 alpha / (1 - alpha) <= 8 / (1 - alpha).  So after k
 * contributors the two transmittances differ by at most SO_EU u S_k relative, S_k = sum over them of 1 / (1 - alpha_j)
 * (>= k: the margin grows at least with the walk depth, and faster behind near-opaque surfels).
 */
#define SO_U (1.0 / 16777216.0)
#define SO_EU 8.0
/* roundings of one forward term after alpha and T (T alpha x, the distortion's error polynomial) */
#define SO_CF 8.0
/* roundings of one backward term after alpha and T: the longest chain is dL/dalpha (a dozen products and sums), times G
 * and opacity, through 1/pz, the cross products and the pixel-weighted sum of dL/dTw: about 30 */
#define SO_CB 32.0
/* m(d) = a - b/d; both sides round it differently (fp32 rcp vs double), with absolute error ~ u (a + b/d) */
#define SO_MA 1.0020040080160320
#define SO_MB 0.20040080160320642

/* optional outputs of the composite (all NULL: the plain composite) */
typedef struct {
    uint8_t *knife;   /* N: 1 = some pair's expf-dependent decision lies within its margin of the threshold */
    double *walk_S;   /* N: S over every contributor of the pixel (see above) */
    double *fbound;   /* 14*N: per plane, sum over terms of (weight in u) * |term| for colour 3, allmap 8, final_T 3 */
    uint32_t *nblend; /* N: pairs blended into the pixel (without culling: every pair of the tile's list is evaluated) */
} so_fwd_ext;

static inline int so_near(double v, double thr, double rel) { return fabs(v - thr) <= rel * fabs(thr); }

/* per-pixel front-to-back composite, forward.cu:283-462 */
static void composite_pixel(const so_state *s, const float *feat, const float *bg, int px, int py,
                            uint32_t r0, uint32_t r1, const so_fwd_ext *ext) {
    const int W = s->W, H = s->H; const size_t N = (size_t)W * H; const size_t pid = (size_t)W * py + px;
    const float pixx = (float)px + 0.5f, pixy = (float)py + 0.5f;
    float T = 1.0f, C[3] = {0, 0, 0}, D = 0, Nn[3] = {0, 0, 0}, dist1 = 0, dist2 = 0, distortion = 0;
    float median_depth = 0, median_weight = 0, median_contributor = -1.0f;
    uint32_t contributor = 0, last_contributor = 0;
    /* ext: S over the contributors so far, knife flag, bound sums (colour 0-2, allmap 3-10, final_T 11-13) */
    double S = 0.0, fb[14] = {0}, ra[14] = {0};
    int knife = 0;
    uint32_t nblend = 0;
    for (uint32_t i = r0; i < r1; i++) {
        contributor++;
        uint32_t id = s->point_list[i];
        const float *Tu = s->transMat + 9 * (size_t)id, *Tv = Tu + 3, *Tw = Tu + 6;
        /* FMA placement below follows the reference's sm_100a SASS (fwd renderCUDA 0x8e0-0x13e0) */
        float k[3] = {FMA(pixx, Tw[0], -Tu[0]), FMA(pixx, Tw[1], -Tu[1]), FMA(pixx, Tw[2], -Tu[2])};
        float l[3] = {FMA(pixy, Tw[0], -Tv[0]), FMA(pixy, Tw[1], -Tv[1]), FMA(pixy, Tw[2], -Tv[2])};
        float p[3] = {FMA(k[1], l[2], -(k[2] * l[1])), FMA(k[2], l[0], -(k[0] * l[2])), FMA(k[0], l[1], -(k[1] * l[0]))};
        if (p[2] == 0.0f) continue;
        float sx = p[0] / p[2], sy = p[1] / p[2];
        float rho3d = FMA(sx, sx, sy * sy);
        float dx = s->means2D[2 * id] - pixx, dy = s->means2D[2 * id + 1] - pixy;
        float q2 = FMA(dx, dx, dy * dy);
        float rho2d = q2 + q2; /* FilterInvSquare*(..) evaluated in double rounds to exactly 2*q2 (DESIGN.md) */
        float rho = fminf(rho3d, rho2d);
        float depth = (rho3d <= rho2d) ? Tw[2] + FMA(Tw[0], sx, Tw[1] * sy) : Tw[2];
        if (depth < NEAR_PLANE_F) continue;
        const float *no = s->normal_opacity + 4 * (size_t)id;
        float power = rho * -0.5f;
        if (power > 0.0f) continue;
        float alpha = fminf(0.99f, no[3] * expf(power));
        if (ext) {
            /* the three expf-dependent decisions; T before this pair carries S, test_T also this pair's 1 - alpha */
            const double Sk = S + 1.0 / (1.0 - (double)alpha);
            knife |= so_near(alpha, 1.0f / 255.0f, SO_EU * SO_U);
            if (alpha >= 1.0f / 255.0f) {
                knife |= so_near((double)T * (1.0 - (double)alpha), 0.0001f, SO_EU * SO_U * Sk);
                knife |= so_near(T, 0.5f, SO_EU * SO_U * S);
            }
        }
        if (alpha < 1.0f / 255.0f) continue;
        float test_T = T * (1 - alpha);
        if (test_T < 0.0001f) break; /* done = true */
        if (ext) {
            /* each running sum gets w |term| for the term and, for the rounding of the sum itself, the running sum of
             * the magnitudes so far (ra) */
            S += 1.0 / (1.0 - (double)alpha);
            const double w = SO_CF + SO_EU * S, ta = (double)T * alpha, mab = SO_MA + SO_MB / depth;
            double t[14] = {0};
            for (int ch = 0; ch < 3; ch++) t[ch] = ta * fabs(feat[3 * (size_t)id + ch]);
            t[3 + 0] = ta * fabs(depth);
            for (int ch = 0; ch < 3; ch++) t[3 + 2 + ch] = ta * fabs(no[ch]);
            t[3 + 6] = ta * (2.0 * fabs(dist1) * mab + fabs(1.0 - T) * mab * mab + fabs(dist2));
            t[11 + 1] = ta * mab;
            t[11 + 2] = ta * mab * mab;
            for (int k = 0; k < 14; k++) {
                ra[k] += t[k];
                fb[k] += w * t[k] + ra[k];
            }
            if (T > 0.5f) fb[3 + 7] = w * ta;
        }
        float A = 1 - T;
        /* the reference evaluates this mapping in double (FAR_PLANE/NEAR_PLANE are double literals) */
        float m = (float)(fma((double)depth, 100.0, -20.0) / ((double)depth * 99.8));
        float error = FMA(-dist1, m + m, FMA(A, m * m, dist2));
        distortion = FMA(T, alpha * error, distortion);
        if (T > 0.5f) { median_depth = depth; median_weight = T * alpha; median_contributor = (float)contributor; }
        for (int ch = 0; ch < 3; ch++) Nn[ch] = FMA(T, no[ch] * alpha, Nn[ch]);
        D = FMA(T, depth * alpha, D);
        dist1 = FMA(T, alpha * m, dist1);
        dist2 = FMA(T, alpha * (m * m), dist2);
        for (int ch = 0; ch < 3; ch++) C[ch] = FMA(T, alpha * feat[3 * (size_t)id + ch], C[ch]);
        T = test_T;
        last_contributor = contributor;
        nblend++;
    }
    s->final_T[pid] = T; s->final_T[pid + N] = dist1; s->final_T[pid + 2 * N] = dist2;
    s->n_contrib[pid] = last_contributor;
    s->n_contrib[pid + N] = median_contributor < 0 ? 0u : (uint32_t)median_contributor; /* cvt.rzi.u32.f32 saturates */
    for (int ch = 0; ch < 3; ch++) s->out_color[ch * N + pid] = C[ch] + T * bg[ch];
    s->out_others[0 * N + pid] = D;
    s->out_others[1 * N + pid] = 1 - T;
    for (int ch = 0; ch < 3; ch++) s->out_others[(2 + ch) * N + pid] = Nn[ch];
    s->out_others[5 * N + pid] = median_depth;
    s->out_others[6 * N + pid] = distortion;
    s->out_others[7 * N + pid] = median_weight;
    if (ext) {
        /* T, 1 - T and C + T bg: the transmittance's own bound plus one rounding of the last operation; the median
         * depth is exact once the median pair agrees */
        const double wT = (1.0 + SO_EU * S) * T;
        for (int ch = 0; ch < 3; ch++) fb[ch] += wT * fabs(bg[ch]) + ra[ch] + T * fabs(bg[ch]);
        fb[3 + 1] = wT + (1.0 - T);
        fb[11 + 0] = wT;
        if (ext->knife) ext->knife[pid] = (uint8_t)knife;
        if (ext->walk_S) ext->walk_S[pid] = S;
        if (ext->nblend) ext->nblend[pid] = nblend;
        if (ext->fbound)
            for (int k = 0; k < 14; k++) ext->fbound[k * N + pid] = fb[k];
    }
}

/* The composite alone, over a state whose per-surfel records (transMat, means2D, normal_opacity), point_list and ranges
 * are given -- e.g. the GPU's own -- into its final_T, n_contrib, out_color and out_others.  knife / walk_S / fbound /
 * nblend: optional outputs (NULL = not wanted), see so_fwd_ext. */
void so_composite(so_state *s, const float *feat, const float *bg, uint8_t *knife, double *walk_S, double *fbound,
                  uint32_t *nblend) {
    const int tiles = s->tiles_x * s->tiles_y, W = s->W, H = s->H;
    so_fwd_ext e = {knife, walk_S, fbound, nblend};
    const so_fwd_ext *ext = (knife || walk_S || fbound || nblend) ? &e : NULL;
#pragma omp parallel for schedule(dynamic, 1)
    for (int t = 0; t < tiles; t++) {
        int tx = t % s->tiles_x, ty = t / s->tiles_x;
        uint32_t r0 = s->ranges[2 * t], r1 = s->ranges[2 * t + 1];
        for (int y = ty * BLOCK_Y; y < (ty + 1) * BLOCK_Y && y < H; y++)
            for (int x = tx * BLOCK_X; x < (tx + 1) * BLOCK_X && x < W; x++)
                composite_pixel(s, feat, bg, x, y, r0, r1, ext);
    }
}

so_state *so_forward(const so_params *p) {
    const int P = p->P, W = p->W, H = p->H;
    const size_t N = (size_t)W * H;
    so_state *s = (so_state *)calloc(1, sizeof(so_state));
    s->P = P; s->W = W; s->H = H;
    s->tiles_x = (W + BLOCK_X - 1) / BLOCK_X; s->tiles_y = (H + BLOCK_Y - 1) / BLOCK_Y;
    const int tiles = s->tiles_x * s->tiles_y;
    const size_t Pa = P > 0 ? P : 1;
    s->depths = (float *)calloc(Pa, 4); s->clamped = (uint8_t *)calloc(Pa * 3, 1);
    s->radii = (int *)calloc(Pa, 4); s->means2D = (float *)calloc(Pa * 2, 4);
    s->transMat = (float *)calloc(Pa * 9, 4); s->normal_opacity = (float *)calloc(Pa * 4, 4);
    s->rgb = (float *)calloc(Pa * 3, 4); s->tiles_touched = (uint32_t *)calloc(Pa, 4);
    s->point_offsets = (uint32_t *)calloc(Pa, 4);
    s->ranges = (uint32_t *)calloc((size_t)tiles * 2, 4);
    s->final_T = (float *)calloc(N * 3, 4); s->n_contrib = (uint32_t *)calloc(N * 2, 4);
    s->out_color = (float *)calloc(N * 3, 4); s->out_others = (float *)calloc(N * 8, 4);

    const float focal_y = H / (2.0f * p->tanfovy), focal_x = W / (2.0f * p->tanfovx);
    const float cx = (float)W / 2.0f, cy = (float)H / 2.0f;
    const float *vm = p->viewmatrix;

    /* ---- preprocess, forward.cu:166-260 ---- */
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        const float *pw = p->means3D + 3 * (size_t)idx;
        float pvz = FMA(pw[2], vm[10], FMA(pw[0], vm[2], pw[1] * vm[6])) + vm[14]; /* transformPoint4x3 .z, SASS 0x4a0-0x4e0 */
        if (pvz <= 0.2f) continue;
        float normal[3], center[2], extent[2];
        float *T = s->transMat + 9 * (size_t)idx;
        if (!compute_transmat(pw, p->rotations + 4 * (size_t)idx, p->scales + 2 * (size_t)idx, vm,
                              focal_x, focal_y, cx, cy, T, normal)) continue;
        if (!compute_aabb(T, center, extent)) continue;
        /* forward.cu:239: FilterSize is a double literal -> the max/mul/ceil run in double */
        double ext = (double)fmaxf(extent[0], extent[1]);
        if (ext < 0.7071067811865476) ext = 0.7071067811865476;
        float radius = (float)ceil(3.0 * ext);
        uint32_t rmin[2], rmax[2];
        get_rect(center, (int)radius, s->tiles_x, s->tiles_y, rmin, rmax);
        if ((rmax[0] - rmin[0]) * (rmax[1] - rmin[1]) == 0) continue;
        if (p->colors_precomp == NULL)
            sh_to_rgb(idx, p->D, p->M, p->means3D, p->campos, p->shs, s->clamped, s->rgb);
        s->depths[idx] = pvz;
        s->radii[idx] = (int)radius;
        s->means2D[2 * idx] = center[0]; s->means2D[2 * idx + 1] = center[1];
        s->normal_opacity[4 * idx] = normal[0]; s->normal_opacity[4 * idx + 1] = normal[1];
        s->normal_opacity[4 * idx + 2] = normal[2]; s->normal_opacity[4 * idx + 3] = p->opacities[idx];
        s->tiles_touched[idx] = (rmax[1] - rmin[1]) * (rmax[0] - rmin[0]);
    }
    /* ---- inclusive scan, rasterizer_impl.cu:278 ---- */
    uint32_t acc = 0;
    for (int i = 0; i < P; i++) { acc += s->tiles_touched[i]; s->point_offsets[i] = acc; }
    const size_t R = acc; s->R = (int)R;
    const size_t Ra = R > 0 ? R : 1;
    s->keys_unsorted = (uint64_t *)calloc(Ra, 8); s->values_unsorted = (uint32_t *)calloc(Ra, 4);
    s->keys = (uint64_t *)calloc(Ra, 8); s->point_list = (uint32_t *)calloc(Ra, 4);
    /* ---- duplicateWithKeys, rasterizer_impl.cu:70-111 ---- */
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        if (s->radii[idx] <= 0) continue;
        uint32_t off = idx == 0 ? 0 : s->point_offsets[idx - 1];
        uint32_t rmin[2], rmax[2];
        get_rect(s->means2D + 2 * (size_t)idx, s->radii[idx], s->tiles_x, s->tiles_y, rmin, rmax);
        uint32_t dbits; memcpy(&dbits, &s->depths[idx], 4);
        for (uint32_t y = rmin[1]; y < rmax[1]; y++)
            for (uint32_t x = rmin[0]; x < rmax[0]; x++) {
                uint64_t key = (uint64_t)(y * (uint32_t)s->tiles_x + x);
                key <<= 32; key |= dbits;
                s->keys_unsorted[off] = key; s->values_unsorted[off] = (uint32_t)idx; off++;
            }
    }
    /* ---- sort + ranges, rasterizer_impl.cu:301-319 ---- */
    s->bit = (int)higher_msb((uint32_t)tiles);
    radix_sort_pairs(s->keys_unsorted, s->values_unsorted, s->keys, s->point_list, R, 32 + s->bit);
    for (size_t i = 0; i < R; i++) {
        uint32_t cur = (uint32_t)(s->keys[i] >> 32);
        if (i == 0) s->ranges[2 * cur] = 0;
        else {
            uint32_t prev = (uint32_t)(s->keys[i - 1] >> 32);
            if (cur != prev) { s->ranges[2 * prev + 1] = (uint32_t)i; s->ranges[2 * cur] = (uint32_t)i; }
        }
        if (i == R - 1) s->ranges[2 * cur + 1] = (uint32_t)R;
    }
    /* ---- composite, forward.cu:265-463 ---- */
    so_composite(s, p->colors_precomp ? p->colors_precomp : s->rgb, p->bg, NULL, NULL, NULL, NULL);
    return s;
}

/* ------------------------------------------------------------------ backward */

typedef struct {
    double *dT;      /* P*9  dL/dtransMat */
    double *dmean2D; /* P*2  low-pass branch accumulators */
    double *dnormal; /* P*3 */
    double *dopac;   /* P */
    double *dcolor;  /* P*3 */
    /* optional (NULL = not wanted), per surfel in so_chain's accumulator order (SO_A_*):
     *   bnd   sum over contributing pairs of (weight in u) * |t|, |t| the term evaluated on absolute values (no
     *         cancellation), weight = SO_CB + SO_EU (S_all + S_behind) + (256 - pixel's index in its tile)
     *   asum  sum over contributing pairs of |t|
     * walk_S: per pixel S over all its contributors (so_composite's output), required with bnd */
    double *bnd, *asum;
    const double *walk_S;
} so_acc;

/* accumulator order of so_chain: dL/dT 9, dL/dmean2D 2 (low-pass branch), dL/dnormal 3, dL/dopacity 1, dL/dcolour 3 */
#define SO_A_T 0
#define SO_A_M2D 9
#define SO_A_NORMAL 11
#define SO_A_OPAC 14
#define SO_A_COLOR 15
#define SO_NACC 18

static inline void atomic_addd(double *p, double v) {
#pragma omp atomic
    *p += v;
}

/* backward.cu:143-449, one pixel */
static void composite_pixel_bwd(const so_state *s, const float *feat, const float *bg,
                                const float *dL_dpix, const float *dL_doth, int px, int py,
                                uint32_t r0, uint32_t r1, so_acc *g) {
    const int W = s->W, H = s->H; const size_t N = (size_t)W * H; const size_t pid = (size_t)W * py + px;
    const float pixx = (float)px + 0.5f, pixy = (float)py + 0.5f;
    const float T_final = s->final_T[pid];
    float T = T_final;
    const uint32_t len = r1 - r0;
    const int last_contributor = (int)s->n_contrib[pid];
    const int median_contributor = (int)s->n_contrib[pid + N];
    float accum_rec[3] = {0, 0, 0}, dL_dpixel[3], dL_dnormal2D[3];
    for (int c = 0; c < 3; c++) dL_dpixel[c] = dL_dpix[c * N + pid];
    const float dL_ddepth = dL_doth[0 * N + pid], dL_daccum = dL_doth[1 * N + pid], dL_dreg = dL_doth[6 * N + pid];
    for (int c = 0; c < 3; c++) dL_dnormal2D[c] = dL_doth[(2 + c) * N + pid];
    const float dL_dmedian_depth = dL_doth[5 * N + pid], dL_dmax_dweight = dL_doth[7 * N + pid];
    float last_depth = 0, last_normal[3] = {0, 0, 0}, accum_depth_rec = 0, accum_alpha_rec = 0;
    float accum_normal_rec[3] = {0, 0, 0};
    const float final_D = s->final_T[pid + N], final_D2 = s->final_T[pid + 2 * N], final_A = 1 - T_final;
    float last_dL_dT = 0, last_alpha = 0, last_color[3] = {0, 0, 0};
    float bg_dot_dpixel = 0;
    for (int c = 0; c < 3; c++) bg_dot_dpixel += bg[c] * dL_dpixel[c];
    /* bounds: the same recursions on absolute values (suffix _a), S behind the current pair, the pair weight's fixed part */
    const int bound = g->bnd != NULL;
    double lc_a[3] = {0, 0, 0}, acc_a[3] = {0, 0, 0}, ld_a = 0, accd_a = 0, lastdT_a = 0, ln_a[3] = {0, 0, 0}, accn_a[3] = {0, 0, 0};
    double la_prev = 0, S_b = 0, w0 = 0, bgd_a = 0;
    if (bound) {
        const int lx = px % BLOCK_X, ly = py % BLOCK_Y;
        const int local = ((ly / 4) * 2 + lx / 8) * 32 + (ly % 4) * 8 + lx % 8;  /* 8x4 sub-tile order */
        w0 = SO_CB + SO_EU * g->walk_S[pid] + (256 - local);
        for (int c = 0; c < 3; c++) bgd_a += fabs(bg[c]) * fabs(dL_dpixel[c]);
    }

    for (uint32_t contributor = len; contributor-- > 0;) {
        if ((int)contributor >= last_contributor) continue;
        const uint32_t id = s->point_list[r0 + contributor];
        const float *Tu = s->transMat + 9 * (size_t)id, *Tv = Tu + 3, *Tw = Tu + 6;
        /* same geometry / alpha arithmetic as the forward, so the discrete skips agree */
        float k[3] = {FMA(pixx, Tw[0], -Tu[0]), FMA(pixx, Tw[1], -Tu[1]), FMA(pixx, Tw[2], -Tu[2])};
        float l[3] = {FMA(pixy, Tw[0], -Tv[0]), FMA(pixy, Tw[1], -Tv[1]), FMA(pixy, Tw[2], -Tv[2])};
        float p[3] = {FMA(k[1], l[2], -(k[2] * l[1])), FMA(k[2], l[0], -(k[0] * l[2])), FMA(k[0], l[1], -(k[1] * l[0]))};
        if (p[2] == 0.0f) continue;
        float sx = p[0] / p[2], sy = p[1] / p[2];
        float rho3d = FMA(sx, sx, sy * sy);
        float dx = s->means2D[2 * id] - pixx, dy = s->means2D[2 * id + 1] - pixy;
        float q2 = FMA(dx, dx, dy * dy);
        float rho2d = q2 + q2;
        float rho = fminf(rho3d, rho2d);
        float c_d = (rho3d <= rho2d) ? Tw[2] + FMA(Tw[0], sx, Tw[1] * sy) : Tw[2];
        if (c_d < NEAR_PLANE_F) continue;
        const float *no = s->normal_opacity + 4 * (size_t)id;
        float power = rho * -0.5f;
        if (power > 0.0f) continue;
        const float G = expf(power);
        const float alpha = fminf(0.99f, no[3] * G);
        if (alpha < 1.0f / 255.0f) continue;

        T = T / (1.f - alpha);
        const float dchannel_dcolor = alpha * T;
        float dL_dalpha = 0.0f;
        for (int ch = 0; ch < 3; ch++) {
            const float c = feat[3 * (size_t)id + ch];
            accum_rec[ch] = last_alpha * last_color[ch] + (1.f - last_alpha) * accum_rec[ch];
            last_color[ch] = c;
            dL_dalpha += (c - accum_rec[ch]) * dL_dpixel[ch];
            atomic_addd(&g->dcolor[3 * (size_t)id + ch], (double)(dchannel_dcolor * dL_dpixel[ch]));
        }
        float dL_dz = 0.0f, dL_dweight = 0;
        /* double detour as in the reference (backward.cu:351-352) */
        float m_d = (float)((100.0 * (double)c_d - 100.0 * 0.2) / ((100.0 - 0.2) * (double)c_d));
        float dmd_dd = (float)((100.0 * 0.2) / ((100.0 - 0.2) * (double)c_d * (double)c_d));
        if ((int)contributor == median_contributor - 1) { dL_dz += dL_dmedian_depth; dL_dweight += dL_dmax_dweight; }
        dL_dweight += (final_D2 + m_d * m_d * final_A - 2 * m_d * final_D) * dL_dreg;
        dL_dalpha += dL_dweight - last_dL_dT;
        last_dL_dT = dL_dweight * alpha + (1 - alpha) * last_dL_dT;
        float dL_dmd = 2.0f * (T * alpha) * (m_d * final_A - final_D) * dL_dreg;
        dL_dz += dL_dmd * dmd_dd;
        accum_depth_rec = last_alpha * last_depth + (1.f - last_alpha) * accum_depth_rec;
        last_depth = c_d;
        dL_dalpha += (c_d - accum_depth_rec) * dL_ddepth;
        accum_alpha_rec = last_alpha * 1.0f + (1.f - last_alpha) * accum_alpha_rec;
        dL_dalpha += (1 - accum_alpha_rec) * dL_daccum;
        for (int ch = 0; ch < 3; ch++) {
            accum_normal_rec[ch] = last_alpha * last_normal[ch] + (1.f - last_alpha) * accum_normal_rec[ch];
            last_normal[ch] = no[ch];
            dL_dalpha += (no[ch] - accum_normal_rec[ch]) * dL_dnormal2D[ch];
            atomic_addd(&g->dnormal[3 * (size_t)id + ch], (double)(alpha * T * dL_dnormal2D[ch]));
        }
        dL_dalpha *= T;
        last_alpha = alpha;
        dL_dalpha += (-T_final / (1.f - alpha)) * bg_dot_dpixel;
        const float dL_dG = no[3] * dL_dalpha;
        dL_dz += alpha * T * dL_ddepth;
        if (rho3d <= rho2d) {
            float dL_dsx = dL_dG * -G * sx + dL_dz * Tw[0];
            float dL_dsy = dL_dG * -G * sy + dL_dz * Tw[1];
            float dsx_pz = dL_dsx / p[2], dsy_pz = dL_dsy / p[2];
            float dL_dp[3] = {dsx_pz, dsy_pz, -(dsx_pz * sx + dsy_pz * sy)};
            float dL_dk[3] = {l[1] * dL_dp[2] - l[2] * dL_dp[1], l[2] * dL_dp[0] - l[0] * dL_dp[2],
                              l[0] * dL_dp[1] - l[1] * dL_dp[0]};
            float dL_dl[3] = {dL_dp[1] * k[2] - dL_dp[2] * k[1], dL_dp[2] * k[0] - dL_dp[0] * k[2],
                              dL_dp[0] * k[1] - dL_dp[1] * k[0]};
            float dz_dTw[3] = {sx, sy, 1.0f};
            for (int c = 0; c < 3; c++) {
                atomic_addd(&g->dT[9 * (size_t)id + c], (double)(-dL_dk[c]));
                atomic_addd(&g->dT[9 * (size_t)id + 3 + c], (double)(-dL_dl[c]));
                atomic_addd(&g->dT[9 * (size_t)id + 6 + c],
                            (double)(pixx * dL_dk[c] + pixy * dL_dl[c] + dL_dz * dz_dTw[c]));
            }
        } else {
            float dG_ddelx = -G * 2.0f * dx, dG_ddely = -G * 2.0f * dy;
            atomic_addd(&g->dmean2D[2 * (size_t)id], (double)(dL_dG * dG_ddelx));
            atomic_addd(&g->dmean2D[2 * (size_t)id + 1], (double)(dL_dG * dG_ddely));
            atomic_addd(&g->dT[9 * (size_t)id + 8], (double)dL_dz);
        }
        atomic_addd(&g->dopac[id], (double)(G * dL_dalpha));
        if (bound) {
            /* the pair's terms once more, on absolute values: every sum of signed parts becomes the sum of their
             * magnitudes, so |t| bounds the size of everything a rounding in t is relative to */
            S_b += 1.0 / (1.0 - (double)alpha);
            const double w = w0 + SO_EU * S_b, aT = (double)alpha * T;
            const double mab = SO_MA + SO_MB / c_d, dmd_a = SO_MB / ((double)c_d * c_d);
            const int med = (int)contributor == median_contributor - 1;
            double dla = 0, dz_a = med ? fabs(dL_dmedian_depth) : 0.0;
            double dw_a = (fabs(final_D2) + mab * mab * fabs(final_A) + 2 * mab * fabs(final_D)) * fabs(dL_dreg);
            if (med) dw_a += fabs(dL_dmax_dweight);
            for (int ch = 0; ch < 3; ch++) {
                acc_a[ch] = la_prev * lc_a[ch] + (1 - la_prev) * acc_a[ch];
                lc_a[ch] = fabs(feat[3 * (size_t)id + ch]);
                dla += (lc_a[ch] + acc_a[ch]) * fabs(dL_dpixel[ch]);
            }
            dla += dw_a + lastdT_a;
            lastdT_a = dw_a * alpha + (1 - alpha) * lastdT_a;
            dz_a += 2 * aT * (mab * fabs(final_A) + fabs(final_D)) * fabs(dL_dreg) * dmd_a;
            accd_a = la_prev * ld_a + (1 - la_prev) * accd_a;
            ld_a = fabs(c_d);
            dla += (ld_a + accd_a) * fabs(dL_ddepth);
            dla += (1 + accum_alpha_rec) * fabs(dL_daccum);
            for (int ch = 0; ch < 3; ch++) {
                accn_a[ch] = la_prev * ln_a[ch] + (1 - la_prev) * accn_a[ch];
                ln_a[ch] = fabs(no[ch]);
                dla += (ln_a[ch] + accn_a[ch]) * fabs(dL_dnormal2D[ch]);
            }
            dla = dla * T + T_final / (1.0 - alpha) * bgd_a;
            la_prev = alpha;
            dz_a += aT * fabs(dL_ddepth);
            const double dG_a = fabs(no[3]) * dla;
            double t[SO_NACC] = {0};
            if (rho3d <= rho2d) {
                const double dsx = dG_a * G * fabs(sx) + dz_a * fabs(Tw[0]), dsy = dG_a * G * fabs(sy) + dz_a * fabs(Tw[1]);
                const double dpx = dsx / fabs(p[2]), dpy = dsy / fabs(p[2]), dpz = dpx * fabs(sx) + dpy * fabs(sy);
                const double dk[3] = {fabs(l[1]) * dpz + fabs(l[2]) * dpy, fabs(l[2]) * dpx + fabs(l[0]) * dpz,
                                      fabs(l[0]) * dpy + fabs(l[1]) * dpx};
                const double dl[3] = {dpy * fabs(k[2]) + dpz * fabs(k[1]), dpz * fabs(k[0]) + dpx * fabs(k[2]),
                                      dpx * fabs(k[1]) + dpy * fabs(k[0])};
                const double dzw[3] = {fabs(sx), fabs(sy), 1.0};
                for (int c = 0; c < 3; c++) {
                    t[SO_A_T + c] = dk[c];
                    t[SO_A_T + 3 + c] = dl[c];
                    t[SO_A_T + 6 + c] = pixx * dk[c] + pixy * dl[c] + dz_a * dzw[c];
                }
            } else {
                t[SO_A_M2D] = dG_a * G * 2 * fabs(dx);
                t[SO_A_M2D + 1] = dG_a * G * 2 * fabs(dy);
                t[SO_A_T + 8] = dz_a;
            }
            for (int ch = 0; ch < 3; ch++) {
                t[SO_A_NORMAL + ch] = aT * fabs(dL_dnormal2D[ch]);
                t[SO_A_COLOR + ch] = aT * fabs(dL_dpixel[ch]);
            }
            t[SO_A_OPAC] = G * dla;
            for (int c = 0; c < SO_NACC; c++)
                if (t[c] != 0.0) {
                    atomic_addd(&g->bnd[SO_NACC * (size_t)id + c], w * t[c]);
                    atomic_addd(&g->asum[SO_NACC * (size_t)id + c], t[c]);
                }
        }
    }
}

/* auxiliary.h:125-135 */
static void dnormvdv3(const float *v, const float *dv, float *o) {
    float sum2 = v[0] * v[0] + v[1] * v[1] + v[2] * v[2];
    float inv = 1.0f / sqrtf(sum2 * sum2 * sum2);
    o[0] = ((+sum2 - v[0] * v[0]) * dv[0] - v[1] * v[0] * dv[1] - v[2] * v[0] * dv[2]) * inv;
    o[1] = (-v[0] * v[1] * dv[0] + (sum2 - v[1] * v[1]) * dv[1] - v[2] * v[1] * dv[2]) * inv;
    o[2] = (-v[0] * v[2] * dv[0] - v[1] * v[2] * dv[1] + (sum2 - v[2] * v[2]) * dv[2]) * inv;
}

/* backward.cu:20-139.  dL_dcolor: 3 floats (already the summed per-surfel value). Adds into dmeans; writes the
 * surfel's dL/dSH row o (M*3 floats). */
static void sh_bwd(int idx, int deg, int M, const float *means, const float *campos, const float *shs,
                   const uint8_t *clamped, const float *dL_dcolor, float *dL_dmean, float *o) {
    float dox = means[3 * idx] - campos[0], doy = means[3 * idx + 1] - campos[1], doz = means[3 * idx + 2] - campos[2];
    float len = sqrtf(dox * dox + doy * doy + doz * doz);
    float x = dox / len, y = doy / len, z = doz / len;
    const float *sh = shs + (size_t)idx * M * 3;
    float dRGB[3];
    for (int c = 0; c < 3; c++) dRGB[c] = dL_dcolor[c] * (clamped[3 * idx + c] ? 0.f : 1.f);
    float dRGBdx[3] = {0, 0, 0}, dRGBdy[3] = {0, 0, 0}, dRGBdz[3] = {0, 0, 0};
#define SETSH(k, w) for (int c = 0; c < 3; c++) o[3 * (k) + c] = (w) * dRGB[c]
    SETSH(0, SH_C0);
    if (deg > 0) {
        SETSH(1, -SH_C1 * y); SETSH(2, SH_C1 * z); SETSH(3, -SH_C1 * x);
        for (int c = 0; c < 3; c++) {
            dRGBdx[c] = -SH_C1 * sh[9 + c]; dRGBdy[c] = -SH_C1 * sh[3 + c]; dRGBdz[c] = SH_C1 * sh[6 + c];
        }
        if (deg > 1) {
            float xx = x * x, yy = y * y, zz = z * z, xy = x * y, yz = y * z, xz = x * z;
            SETSH(4, SH_C2[0] * xy); SETSH(5, SH_C2[1] * yz); SETSH(6, SH_C2[2] * (2.f * zz - xx - yy));
            SETSH(7, SH_C2[3] * xz); SETSH(8, SH_C2[4] * (xx - yy));
            for (int c = 0; c < 3; c++) {
                dRGBdx[c] += SH_C2[0] * y * sh[12 + c] + SH_C2[2] * 2.f * -x * sh[18 + c] + SH_C2[3] * z * sh[21 + c] +
                             SH_C2[4] * 2.f * x * sh[24 + c];
                dRGBdy[c] += SH_C2[0] * x * sh[12 + c] + SH_C2[1] * z * sh[15 + c] + SH_C2[2] * 2.f * -y * sh[18 + c] +
                             SH_C2[4] * 2.f * -y * sh[24 + c];
                dRGBdz[c] += SH_C2[1] * y * sh[15 + c] + SH_C2[2] * 2.f * 2.f * z * sh[18 + c] + SH_C2[3] * x * sh[21 + c];
            }
            if (deg > 2) {
                SETSH(9, SH_C3[0] * y * (3.f * xx - yy)); SETSH(10, SH_C3[1] * xy * z);
                SETSH(11, SH_C3[2] * y * (4.f * zz - xx - yy));
                SETSH(12, SH_C3[3] * z * (2.f * zz - 3.f * xx - 3.f * yy));
                SETSH(13, SH_C3[4] * x * (4.f * zz - xx - yy)); SETSH(14, SH_C3[5] * z * (xx - yy));
                SETSH(15, SH_C3[6] * x * (xx - 3.f * yy));
                for (int c = 0; c < 3; c++) {
                    dRGBdx[c] += (SH_C3[0] * sh[27 + c] * 3.f * 2.f * xy + SH_C3[1] * sh[30 + c] * yz +
                                  SH_C3[2] * sh[33 + c] * -2.f * xy + SH_C3[3] * sh[36 + c] * -3.f * 2.f * xz +
                                  SH_C3[4] * sh[39 + c] * (-3.f * xx + 4.f * zz - yy) +
                                  SH_C3[5] * sh[42 + c] * 2.f * xz + SH_C3[6] * sh[45 + c] * 3.f * (xx - yy));
                    dRGBdy[c] += (SH_C3[0] * sh[27 + c] * 3.f * (xx - yy) + SH_C3[1] * sh[30 + c] * xz +
                                  SH_C3[2] * sh[33 + c] * (-3.f * yy + 4.f * zz - xx) +
                                  SH_C3[3] * sh[36 + c] * -3.f * 2.f * yz + SH_C3[4] * sh[39 + c] * -2.f * xy +
                                  SH_C3[5] * sh[42 + c] * -2.f * yz + SH_C3[6] * sh[45 + c] * -3.f * 2.f * xy);
                    dRGBdz[c] += (SH_C3[1] * sh[30 + c] * xy + SH_C3[2] * sh[33 + c] * 4.f * 2.f * yz +
                                  SH_C3[3] * sh[36 + c] * 3.f * (2.f * zz - xx - yy) +
                                  SH_C3[4] * sh[39 + c] * 4.f * 2.f * xz + SH_C3[5] * sh[42 + c] * (xx - yy));
                }
            }
        }
    }
#undef SETSH
    float ddir[3] = {dRGBdx[0] * dRGB[0] + dRGBdx[1] * dRGB[1] + dRGBdx[2] * dRGB[2],
                     dRGBdy[0] * dRGB[0] + dRGBdy[1] * dRGB[1] + dRGBdy[2] * dRGB[2],
                     dRGBdz[0] * dRGB[0] + dRGBdz[1] * dRGB[1] + dRGBdz[2] * dRGB[2]};
    float dorig[3] = {dox, doy, doz}, dm[3];
    dnormvdv3(dorig, ddir, dm);
    dL_dmean[0] += dm[0]; dL_dmean[1] += dm[1]; dL_dmean[2] += dm[2];
}

/* one surfel's rows of the backward's outputs */
typedef struct {
    float *m2d, *col, *op, *m3d, *tm, *sh, *sc, *rot, *nrm;
} so_row;

static so_row row_of(int idx, int M, float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity, float *dL_dmeans3D,
                     float *dL_dtransMat, float *dL_dsh, float *dL_dscales, float *dL_drotations, float *dL_dnormal) {
    so_row o = {dL_dmeans2D + 3 * (size_t)idx, dL_dcolors + 3 * (size_t)idx, dL_dopacity + idx, dL_dmeans3D + 3 * (size_t)idx,
                dL_dtransMat + 9 * (size_t)idx, dL_dsh + (size_t)idx * M * 3, dL_dscales + 2 * (size_t)idx,
                dL_drotations + 4 * (size_t)idx, dL_dnormal + 3 * (size_t)idx};
    return o;
}

/* The per-surfel part of the backward from one surfel's accumulators a[] (SO_A_* order): the AABB vjp, the
 * computeTransMat vjp, the quaternion vjp and the SH vjp.  Linear in a[] for fixed surfel inputs.  Rows other than the
 * colour, opacity, normal and transMat ones are left alone for an invisible surfel (the caller zero-fills them). */
static void chain_one(const so_params *p, const so_state *s, int idx, const float *a, so_row o) {
    const int W = p->W, H = p->H;
    const float focal_y = H / (2.0f * p->tanfovy), focal_x = W / (2.0f * p->tanfovx);
    const float Wh = focal_x * p->tanfovx, Hh = focal_y * p->tanfovy; /* backward.cu:683-684 */
    const float *vm = p->viewmatrix;
    for (int c = 0; c < 3; c++) {
        o.col[c] = a[SO_A_COLOR + c];
        o.nrm[c] = a[SO_A_NORMAL + c];
    }
    *o.op = a[SO_A_OPAC];
    float dT[9];
    for (int c = 0; c < 9; c++) dT[c] = a[SO_A_T + c];
    if (!(s->radii[idx] > 0)) { for (int c = 0; c < 9; c++) o.tm[c] = dT[c]; return; }
    /* ---- computeAABB vjp, backward.cu:599-649 ---- */
    const float *T = s->transMat + 9 * (size_t)idx;
    const float *Tu = T, *Tv = T + 3, *Tw = T + 6;
    const float dmx = a[SO_A_M2D], dmy = a[SO_A_M2D + 1];
    float d = Tw[0] * Tw[0] + Tw[1] * Tw[1] - Tw[2] * Tw[2];
    float inv = 1.0f / d;
    float f[3] = {inv, inv, -inv};
    float dL_dT0[3], dL_dT1[3], dL_dT3[3], dL_df[3];
    for (int c = 0; c < 3; c++) {
        dL_dT0[c] = dmx * f[c] * Tw[c];
        dL_dT1[c] = dmy * f[c] * Tw[c];
        dL_dT3[c] = dmx * f[c] * Tu[c] + dmy * f[c] * Tv[c];
        dL_df[c] = (dmx * Tu[c] * Tw[c]) + (dmy * Tv[c] * Tw[c]);
    }
    float dL_dd = (float)((double)(dL_df[0] * f[0] + dL_df[1] * f[1] + dL_df[2] * f[2]) * (-1.0 / (double)d));
    const float sg[3] = {1.f, 1.f, -1.f};
    for (int c = 0; c < 3; c++) dL_dT3[c] += dL_dd * (sg[c] * Tw[c] * 2.0f);
    for (int c = 0; c < 3; c++) { dT[c] += dL_dT0[c]; dT[3 + c] += dL_dT1[c]; dT[6 + c] += dL_dT3[c]; }
    for (int c = 0; c < 9; c++) o.tm[c] = dT[c];
    o.m2d[0] = dT[2] * T[8] * Wh;     /* densification proxy, backward.cu:645-648 */
    o.m2d[1] = dT[5] * T[8] * Hh;
    /* ---- computeTransMat vjp, backward.cu:451-529 ---- */
    const float *quat = p->rotations + 4 * (size_t)idx, *scale = p->scales + 2 * (size_t)idx;
    const float *pw = p->means3D + 3 * (size_t)idx;
    const float fx = focal_x, fy = focal_y, cx = Wh, cy = Hh; /* intrins, backward.cu:570 */
    float Rq[9]; quat_to_rotmat(quat, Rq);
    float pv[3]; W_mul(vm, pw, pv); pv[0] += vm[12]; pv[1] += vm[13]; pv[2] += vm[14];
    /* dL_dM column j = K^T (dTu[j], dTv[j], dTw[j]) */
    float dM[3][3];
    for (int j = 0; j < 3; j++) {
        dM[j][0] = fx * dT[j];
        dM[j][1] = fy * dT[3 + j];
        dM[j][2] = cx * dT[j] + cy * dT[3 + j] + dT[6 + j];
    }
    float dRS0[3], dRS1[3], dpw[3], dtn[3];
    Wt_mul(vm, dM[0], dRS0); Wt_mul(vm, dM[1], dRS1); Wt_mul(vm, dM[2], dpw);
    float dn[3] = {o.nrm[0], o.nrm[1], o.nrm[2]};
    Wt_mul(vm, dn, dtn);
    float tn[3]; W_mul(vm, Rq + 6, tn);
    float cosv = (-tn[0]) * pv[0] + (-tn[1]) * pv[1] + (-tn[2]) * pv[2];
    float mult = cosv > 0 ? 1.f : -1.f;
    dtn[0] *= mult; dtn[1] *= mult; dtn[2] *= mult;
    /* v_R column-major: col0 = dRS0*sx, col1 = dRS1*sy, col2 = dtn */
    float vR[3][3];
    for (int r = 0; r < 3; r++) { vR[0][r] = dRS0[r] * scale[0]; vR[1][r] = dRS1[r] * scale[1]; vR[2][r] = dtn[r]; }
    /* quat_to_rotmat_vjp, auxiliary.h:213-257 (gradient w.r.t. the normalised quaternion) */
    float sN = 1.0f / sqrtf(quat[3] * quat[3] + quat[0] * quat[0] + quat[1] * quat[1] + quat[2] * quat[2]);
    float w = quat[0] * sN, x = quat[1] * sN, y = quat[2] * sN, z = quat[3] * sN;
    o.rot[0] = 2.f * (x * (vR[1][2] - vR[2][1]) + y * (vR[2][0] - vR[0][2]) + z * (vR[0][1] - vR[1][0]));
    o.rot[1] = 2.f * (-2.f * x * (vR[1][1] + vR[2][2]) + y * (vR[0][1] + vR[1][0]) +
                      z * (vR[0][2] + vR[2][0]) + w * (vR[1][2] - vR[2][1]));
    o.rot[2] = 2.f * (x * (vR[0][1] + vR[1][0]) - 2.f * y * (vR[0][0] + vR[2][2]) +
                      z * (vR[1][2] + vR[2][1]) + w * (vR[2][0] - vR[0][2]));
    o.rot[3] = 2.f * (x * (vR[0][2] + vR[2][0]) + y * (vR[1][2] + vR[2][1]) -
                      2.f * z * (vR[0][0] + vR[1][1]) + w * (vR[0][1] - vR[1][0]));
    o.sc[0] = dRS0[0] * Rq[0] + dRS0[1] * Rq[1] + dRS0[2] * Rq[2];
    o.sc[1] = dRS1[0] * Rq[3] + dRS1[1] * Rq[4] + dRS1[2] * Rq[5];
    o.m3d[0] = dpw[0]; o.m3d[1] = dpw[1]; o.m3d[2] = dpw[2];
    if (p->shs) sh_bwd(idx, p->D, p->M, p->means3D, p->campos, p->shs, s->clamped, o.col, o.m3d, o.sh);
}

/* so_backward's per-surfel part on given accumulators acc (P*18 floats, SO_A_* order).  Outputs as so_backward's. */
void so_chain(const so_params *p, const so_state *s, const float *acc, float *dL_dmeans2D, float *dL_dcolors,
              float *dL_dopacity, float *dL_dmeans3D, float *dL_dtransMat, float *dL_dsh, float *dL_dscales,
              float *dL_drotations, float *dL_dnormal) {
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < p->P; idx++)
        chain_one(p, s, idx, acc + SO_NACC * (size_t)idx,
                  row_of(idx, p->M, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh, dL_dscales,
                         dL_drotations, dL_dnormal));
}

/*
 * Propagates per-accumulator bounds B (P*18 doubles, SO_A_* order) through the per-surfel chain evaluated on absolute
 * values: every input replaced by its magnitude, every difference by a sum, every divisor d by |d|^2 / (the divisor on
 * absolute values) -- the standard running-error shadow.  The chain is linear in the accumulators, so the result bounds
 * sum_j |d out / d acc_j| B_j, and the chain's own fp32 roundings are relative to it (not to the possibly much smaller
 * |d out / d acc_j|: the basis polynomials, W^T dM, dRS . R and the quaternion vjp all cancel).  Outputs: doubles,
 * shaped as so_backward's.
 */
void so_chain_bound(const so_params *p, const so_state *s, const double *B, double *b_m2d, double *b_col, double *b_op,
                    double *b_m3d, double *b_tm, double *b_sh, double *b_sc, double *b_rot, double *b_nrm) {
    const int M = p->M, W = p->W, H = p->H;
    const double focal_y = H / (2.0f * p->tanfovy), focal_x = W / (2.0f * p->tanfovx);
    const double Wh = fabs((float)focal_x * p->tanfovx), Hh = fabs((float)focal_y * p->tanfovy);
    double vm[16];
    for (int i = 0; i < 16; i++) vm[i] = fabs(p->viewmatrix[i]);
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < p->P; idx++) {
        const double *A = B + SO_NACC * (size_t)idx;
        for (int c = 0; c < 3; c++) {
            b_col[3 * (size_t)idx + c] = A[SO_A_COLOR + c];
            b_nrm[3 * (size_t)idx + c] = A[SO_A_NORMAL + c];
        }
        b_op[idx] = A[SO_A_OPAC];
        double tm[9];
        for (int c = 0; c < 9; c++) tm[c] = A[SO_A_T + c];
        if (!(s->radii[idx] > 0)) { for (int c = 0; c < 9; c++) b_tm[9 * (size_t)idx + c] = tm[c]; continue; }
        /* AABB vjp */
        double T[9];
        for (int c = 0; c < 9; c++) T[c] = fabs(s->transMat[9 * (size_t)idx + c]);
        const float *Tf = s->transMat + 9 * (size_t)idx;
        const double d = (double)Tf[6] * Tf[6] + (double)Tf[7] * Tf[7] - (double)Tf[8] * Tf[8];
        const double inv_a = (T[6] * T[6] + T[7] * T[7] + T[8] * T[8]) / (d * d);
        const double dmx = A[SO_A_M2D], dmy = A[SO_A_M2D + 1];
        double df = 0;
        for (int c = 0; c < 3; c++) df += (dmx * T[c] * T[6 + c] + dmy * T[3 + c] * T[6 + c]) * inv_a;
        const double dd = df * inv_a;
        for (int c = 0; c < 3; c++) {
            tm[c] += dmx * inv_a * T[6 + c];
            tm[3 + c] += dmy * inv_a * T[6 + c];
            tm[6 + c] += dmx * inv_a * T[c] + dmy * inv_a * T[3 + c] + dd * 2 * T[6 + c];
        }
        for (int c = 0; c < 9; c++) b_tm[9 * (size_t)idx + c] = tm[c];
        b_m2d[3 * (size_t)idx] = tm[2] * T[8] * Wh;
        b_m2d[3 * (size_t)idx + 1] = tm[5] * T[8] * Hh;
        /* computeTransMat vjp: dM = K^T dT, W^T, the rotation of the normalised quaternion */
        double dM[3][3], dRS[3][3], dtn[3];
        for (int j = 0; j < 3; j++) {
            dM[j][0] = focal_x * tm[j];
            dM[j][1] = focal_y * tm[3 + j];
            dM[j][2] = Wh * tm[j] + Hh * tm[3 + j] + tm[6 + j];
        }
        for (int j = 0; j < 3; j++)
            for (int r = 0; r < 3; r++) dRS[j][r] = vm[4 * r] * dM[j][0] + vm[4 * r + 1] * dM[j][1] + vm[4 * r + 2] * dM[j][2];
        for (int r = 0; r < 3; r++)
            dtn[r] = vm[4 * r] * A[SO_A_NORMAL] + vm[4 * r + 1] * A[SO_A_NORMAL + 1] + vm[4 * r + 2] * A[SO_A_NORMAL + 2];
        const float *q = p->rotations + 4 * (size_t)idx, *sc = p->scales + 2 * (size_t)idx;
        const double qn = sqrt((double)q[0] * q[0] + (double)q[1] * q[1] + (double)q[2] * q[2] + (double)q[3] * q[3]);
        const double w = fabs(q[0] / qn), x = fabs(q[1] / qn), y = fabs(q[2] / qn), z = fabs(q[3] / qn);
        const double R[6] = {1 + 2 * (y * y + z * z), 2 * (x * y + w * z), 2 * (x * z + w * y),
                             2 * (x * y + w * z), 1 + 2 * (x * x + z * z), 2 * (y * z + w * x)};
        double v[3][3];
        for (int r = 0; r < 3; r++) { v[0][r] = dRS[0][r] * fabs(sc[0]); v[1][r] = dRS[1][r] * fabs(sc[1]); v[2][r] = dtn[r]; }
        double *ro = b_rot + 4 * (size_t)idx;
        ro[0] = 2 * (x * (v[1][2] + v[2][1]) + y * (v[2][0] + v[0][2]) + z * (v[0][1] + v[1][0]));
        ro[1] = 2 * (2 * x * (v[1][1] + v[2][2]) + y * (v[0][1] + v[1][0]) + z * (v[0][2] + v[2][0]) + w * (v[1][2] + v[2][1]));
        ro[2] = 2 * (x * (v[0][1] + v[1][0]) + 2 * y * (v[0][0] + v[2][2]) + z * (v[1][2] + v[2][1]) + w * (v[2][0] + v[0][2]));
        ro[3] = 2 * (x * (v[0][2] + v[2][0]) + y * (v[1][2] + v[2][1]) + 2 * z * (v[0][0] + v[1][1]) + w * (v[0][1] + v[1][0]));
        b_sc[2 * (size_t)idx] = dRS[0][0] * R[0] + dRS[0][1] * R[1] + dRS[0][2] * R[2];
        b_sc[2 * (size_t)idx + 1] = dRS[1][0] * R[3] + dRS[1][1] * R[4] + dRS[1][2] * R[5];
        double *m3 = b_m3d + 3 * (size_t)idx;
        for (int r = 0; r < 3; r++) m3[r] = dRS[2][r];
        if (!p->shs) continue;
        /* SH vjp: the basis polynomials and their derivatives on absolute values, then the direction normalisation */
        const float *mw = p->means3D + 3 * (size_t)idx;
        const double ox = (double)mw[0] - p->campos[0], oy = (double)mw[1] - p->campos[1], oz = (double)mw[2] - p->campos[2];
        const double sum2 = ox * ox + oy * oy + oz * oz, len = sqrt(sum2);
        const double X = fabs(ox / len), Y = fabs(oy / len), Z = fabs(oz / len), xx = X * X, yy = Y * Y, zz = Z * Z;
        const int deg = p->D;
        const double wa[16] = {SH_C0, SH_C1 * Y, SH_C1 * Z, SH_C1 * X,
                               fabs(SH_C2[0]) * X * Y, fabs(SH_C2[1]) * Y * Z, fabs(SH_C2[2]) * (2 * zz + xx + yy),
                               fabs(SH_C2[3]) * X * Z, fabs(SH_C2[4]) * (xx + yy),
                               fabs(SH_C3[0]) * Y * (3 * xx + yy), fabs(SH_C3[1]) * X * Y * Z,
                               fabs(SH_C3[2]) * Y * (4 * zz + xx + yy), fabs(SH_C3[3]) * Z * (2 * zz + 3 * xx + 3 * yy),
                               fabs(SH_C3[4]) * X * (4 * zz + xx + yy), fabs(SH_C3[5]) * Z * (xx + yy),
                               fabs(SH_C3[6]) * X * (xx + 3 * yy)};
        const int used = (deg + 1) * (deg + 1) < M ? (deg + 1) * (deg + 1) : M;
        double dRGB[3];
        for (int c = 0; c < 3; c++) dRGB[c] = s->clamped[3 * (size_t)idx + c] ? 0.0 : A[SO_A_COLOR + c];
        double *bs = b_sh + (size_t)idx * M * 3;
        for (int k = 0; k < used; k++)
            for (int c = 0; c < 3; c++) bs[3 * k + c] = wa[k] * dRGB[c];
        const float *shf = p->shs + (size_t)idx * M * 3;
        double dd3[3] = {0, 0, 0};
        for (int c = 0; c < 3; c++) {
#define SA(k) fabs((double)shf[3 * (k) + c])
            double gx = 0, gy = 0, gz = 0;
            if (deg > 0) { gx = SH_C1 * SA(3); gy = SH_C1 * SA(1); gz = SH_C1 * SA(2); }
            if (deg > 1) {
                gx += fabs(SH_C2[0]) * Y * SA(4) + fabs(SH_C2[2]) * 2 * X * SA(6) + fabs(SH_C2[3]) * Z * SA(7) + fabs(SH_C2[4]) * 2 * X * SA(8);
                gy += fabs(SH_C2[0]) * X * SA(4) + fabs(SH_C2[1]) * Z * SA(5) + fabs(SH_C2[2]) * 2 * Y * SA(6) + fabs(SH_C2[4]) * 2 * Y * SA(8);
                gz += fabs(SH_C2[1]) * Y * SA(5) + fabs(SH_C2[2]) * 4 * Z * SA(6) + fabs(SH_C2[3]) * X * SA(7);
            }
            if (deg > 2) {
                gx += fabs(SH_C3[0]) * SA(9) * 6 * X * Y + fabs(SH_C3[1]) * SA(10) * Y * Z + fabs(SH_C3[2]) * SA(11) * 2 * X * Y +
                      fabs(SH_C3[3]) * SA(12) * 6 * X * Z + fabs(SH_C3[4]) * SA(13) * (3 * xx + 4 * zz + yy) +
                      fabs(SH_C3[5]) * SA(14) * 2 * X * Z + fabs(SH_C3[6]) * SA(15) * 3 * (xx + yy);
                gy += fabs(SH_C3[0]) * SA(9) * 3 * (xx + yy) + fabs(SH_C3[1]) * SA(10) * X * Z +
                      fabs(SH_C3[2]) * SA(11) * (3 * yy + 4 * zz + xx) + fabs(SH_C3[3]) * SA(12) * 6 * Y * Z +
                      fabs(SH_C3[4]) * SA(13) * 2 * X * Y + fabs(SH_C3[5]) * SA(14) * 2 * Y * Z + fabs(SH_C3[6]) * SA(15) * 6 * X * Y;
                gz += fabs(SH_C3[1]) * SA(10) * X * Y + fabs(SH_C3[2]) * SA(11) * 8 * Y * Z +
                      fabs(SH_C3[3]) * SA(12) * 3 * (2 * zz + xx + yy) + fabs(SH_C3[4]) * SA(13) * 8 * X * Z +
                      fabs(SH_C3[5]) * SA(14) * (xx + yy);
            }
#undef SA
            dd3[0] += gx * dRGB[c]; dd3[1] += gy * dRGB[c]; dd3[2] += gz * dRGB[c];
        }
        const double vx = fabs(ox), vy = fabs(oy), vz = fabs(oz), inv32 = 1.0 / sqrt(sum2 * sum2 * sum2);
        m3[0] += ((sum2 + vx * vx) * dd3[0] + vy * vx * dd3[1] + vz * vx * dd3[2]) * inv32;
        m3[1] += (vx * vy * dd3[0] + (sum2 + vy * vy) * dd3[1] + vz * vy * dd3[2]) * inv32;
        m3[2] += (vx * vz * dd3[0] + vy * vz * dd3[1] + (sum2 + vz * vz) * dd3[2]) * inv32;
    }
}

/*
 * Outputs (all float, caller-allocated, zero-initialised by the caller):
 *   dL_dmeans2D P*3, dL_dcolors P*3, dL_dopacity P, dL_dmeans3D P*3, dL_dtransMat P*9,
 *   dL_dsh P*M*3, dL_dscales P*2, dL_drotations P*4, dL_dnormal P*3
 * Optional (NULL = not wanted, zero-initialised by the caller): acc P*18 doubles, the accumulators in SO_A_* order;
 * bnd, asum P*18 doubles, the bound sums of so_acc, which need walk_S (so_composite's output).
 */
void so_backward_ex(const so_params *p, const so_state *s, const float *dL_dpix, const float *dL_doth,
                    float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity, float *dL_dmeans3D,
                    float *dL_dtransMat, float *dL_dsh, float *dL_dscales, float *dL_drotations,
                    float *dL_dnormal, const double *walk_S, double *acc, double *bnd, double *asum) {
    const int P = p->P, W = p->W, H = p->H;
    const int tiles = s->tiles_x * s->tiles_y;
    so_acc g;
    const size_t Pa = P > 0 ? P : 1;
    g.dT = (double *)calloc(Pa * 9, 8); g.dmean2D = (double *)calloc(Pa * 2, 8);
    g.dnormal = (double *)calloc(Pa * 3, 8); g.dopac = (double *)calloc(Pa, 8); g.dcolor = (double *)calloc(Pa * 3, 8);
    g.bnd = walk_S ? bnd : NULL; g.asum = asum; g.walk_S = walk_S;
    const float *feat = p->colors_precomp ? p->colors_precomp : s->rgb;
#pragma omp parallel for schedule(dynamic, 1)
    for (int t = 0; t < tiles; t++) {
        int tx = t % s->tiles_x, ty = t / s->tiles_x;
        uint32_t r0 = s->ranges[2 * t], r1 = s->ranges[2 * t + 1];
        if (r1 == r0) continue;
        for (int y = ty * BLOCK_Y; y < (ty + 1) * BLOCK_Y && y < H; y++)
            for (int x = tx * BLOCK_X; x < (tx + 1) * BLOCK_X && x < W; x++)
                composite_pixel_bwd(s, feat, p->bg, dL_dpix, dL_doth, x, y, r0, r1, &g);
    }
#pragma omp parallel for schedule(static)
    for (int idx = 0; idx < P; idx++) {
        double a64[SO_NACC];
        for (int c = 0; c < 9; c++) a64[SO_A_T + c] = g.dT[9 * idx + c];
        for (int c = 0; c < 2; c++) a64[SO_A_M2D + c] = g.dmean2D[2 * idx + c];
        for (int c = 0; c < 3; c++) {
            a64[SO_A_NORMAL + c] = g.dnormal[3 * idx + c];
            a64[SO_A_COLOR + c] = g.dcolor[3 * idx + c];
        }
        a64[SO_A_OPAC] = g.dopac[idx];
        float a[SO_NACC];
        for (int c = 0; c < SO_NACC; c++) a[c] = (float)a64[c];
        if (acc) memcpy(acc + SO_NACC * (size_t)idx, a64, sizeof(a64));
        chain_one(p, s, idx, a, row_of(idx, p->M, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh,
                                       dL_dscales, dL_drotations, dL_dnormal));
    }
    free(g.dT); free(g.dmean2D); free(g.dnormal); free(g.dopac); free(g.dcolor);
}

void so_backward(const so_params *p, const so_state *s, const float *dL_dpix, const float *dL_doth,
                 float *dL_dmeans2D, float *dL_dcolors, float *dL_dopacity, float *dL_dmeans3D,
                 float *dL_dtransMat, float *dL_dsh, float *dL_dscales, float *dL_drotations,
                 float *dL_dnormal) {
    so_backward_ex(p, s, dL_dpix, dL_doth, dL_dmeans2D, dL_dcolors, dL_dopacity, dL_dmeans3D, dL_dtransMat, dL_dsh,
                   dL_dscales, dL_drotations, dL_dnormal, NULL, NULL, NULL, NULL);
}

/* rasterizer_impl.cu:54-66 + auxiliary.h:160-185 */
void so_mark_visible(int P, const float *means3D, const float *vm, uint8_t *present) {
    for (int i = 0; i < P; i++) {
        const float *pw = means3D + 3 * (size_t)i;
        float z = FMA(pw[2], vm[10], FMA(pw[0], vm[2], pw[1] * vm[6])) + vm[14];
        present[i] = z > 0.2f;
    }
}

int so_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}
