// outlier.cu -- radius outlier filter: keep a point iff more than nb_points points lie strictly closer than `radius`.
//
// Replaces (behaviour, not code) the Open3D call of Stage 3's periodic outlier filter (lab4d/engine/trainer.py:573-588,
// `pcd.remove_radius_outlier(nb_points=20, radius=0.004)`), which runs on the host after a D2H copy of every surfel.
//
// Semantics (DESIGN.md section 3.9):
//   count_i = #{ j in [0,P) : d2(i,j) < r2 }, j = i included;
//   d2 = ((xi-xj)^2 + (yi-yj)^2) + (zi-zj)^2 in float64, every difference, product and sum rounded on its own;
//   r2 = radius * radius in float64;  keep_i = count_i > nb_points.
// A point with a NaN or Inf coordinate has d2 = NaN or Inf to every point, itself included: it counts for nobody and
// is never kept.
//
// Grid: every point gets a cell (floor(x / h), floor(y / h), floor(z / h)), each axis clamped to a signed 21-bit range and
// packed into a 63-bit key; the points are radix-sorted by key (cub), so the three z-adjacent cells of one (x, y) column
// are one contiguous key range, found by binary search.  No bounding box, no host synchronisation: scratch is sized
// from P alone and the whole call can be captured in a CUDA graph.  Far points (strays) clamp into the border cells,
// where they only cost candidate checks; the exact predicate decides every pair.
#include <cmath>
#include <cub/device/device_radix_sort.cuh>
#include "common.cuh"

namespace {

constexpr int RO_BITS = 21;                                  // per axis: cell indices in [-2^20, 2^20)
constexpr double RO_CMIN = -(double)(1 << (RO_BITS - 1));
constexpr double RO_CMAX = (double)((1 << (RO_BITS - 1)) - 1);
constexpr int RO_THREADS = 256;
constexpr size_t RO_CUB_SLACK = size_t(1) << 20;

// Cell edge h = r * (1 + 2^-20).  Why two points closer than r never land two cells apart on an axis: with t = fl(x * inv_h),
// inv_h = fl(1 / h), the error of inv_h is relative and common to both points, so it scales their difference by at most
// (1 + 2^-53); each product adds at most half an ulp of t, which is 2^-32 where |t| < 2^22.  d2 < r2 in float64 means
// d < r * (1 + 2^-50) (a handful of roundings on each side), hence, where both |t| < 2^22,
//     |ti - tj| < (1 + 2^-50) * (1 + 2^-53) / (1 + 2^-20) + 2 * 2^-32 < 1,
// and floor() keeps the difference <= 1.  Where one |t| >= 2^22, the other is > 2^21 on the same side (the relative
// rounding is far below 1 / 2), and both clamp to the same border index.  Clamping is monotone, so it never separates
// adjacent indices.  fmax / fmin map a NaN to the lower bound, which only puts a point that counts for nobody into a cell.
__device__ __forceinline__ int ro_cell(float x, double inv_h) {
    const double t = floor(__dmul_rn((double)x, inv_h));
    return (int)fmin(fmax(t, RO_CMIN), RO_CMAX);
}
__device__ __forceinline__ uint64_t ro_key(int cx, int cy, int cz) {
    const uint64_t o = uint64_t(1) << (RO_BITS - 1);
    return ((uint64_t)(cx + o) << (2 * RO_BITS)) | ((uint64_t)(cy + o) << RO_BITS) | (uint64_t)(cz + o);
}

__global__ void __launch_bounds__(RO_THREADS)
ro_key_kernel(int P, const float* __restrict__ pts, double inv_h, uint64_t* __restrict__ keys, int* __restrict__ idx) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    keys[i] = ro_key(ro_cell(x, inv_h), ro_cell(y, inv_h), ro_cell(z, inv_h));
    idx[i] = i;
}

// the points in key order, so that the candidates of one column are read contiguously
__global__ void __launch_bounds__(RO_THREADS)
ro_gather_kernel(int P, const float* __restrict__ pts, const int* __restrict__ idx, float4* __restrict__ sorted) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const size_t i = (size_t)idx[k];
    sorted[k] = make_float4(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2], 0.f);
}

__device__ __forceinline__ int ro_lower_bound(const uint64_t* __restrict__ keys, int n, uint64_t k) {
    int lo = 0, hi = n;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(keys + mid) < k) lo = mid + 1; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ double ro_d2(float4 a, float4 b) {
    const double dx = __dsub_rn((double)a.x, (double)b.x), dy = __dsub_rn((double)a.y, (double)b.y),
                 dz = __dsub_rn((double)a.z, (double)b.z);
    return __dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz));
}

// One thread per point, in key order (neighbouring threads search neighbouring cells).  Counting stops at
// nb_points + 1: only the decision is needed, and clone-densified duplicates make the dense cells dense.
__global__ void __launch_bounds__(RO_THREADS)
ro_query_kernel(int P, const float4* __restrict__ sorted, const uint64_t* __restrict__ keys, const int* __restrict__ idx,
                double inv_h, double r2, long long cap, uint8_t* __restrict__ keep, int32_t* __restrict__ counts) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= P) return;
    const float4 p = sorted[k];
    long long n = 0;
    if (isfinite(p.x) && isfinite(p.y) && isfinite(p.z)) {
        const int cx = ro_cell(p.x, inv_h), cy = ro_cell(p.y, inv_h), cz = ro_cell(p.z, inv_h);
        const int z0 = max(cz - 1, (int)RO_CMIN), z1 = min(cz + 1, (int)RO_CMAX);
        for (int dx = -1; dx <= 1 && n < cap; dx++) {
            const int x = cx + dx;
            if (x < (int)RO_CMIN || x > (int)RO_CMAX) continue;
            for (int dy = -1; dy <= 1 && n < cap; dy++) {
                const int y = cy + dy;
                if (y < (int)RO_CMIN || y > (int)RO_CMAX) continue;
                const int b = ro_lower_bound(keys, P, ro_key(x, y, z0));
                const int e = ro_lower_bound(keys, P, ro_key(x, y, z1) + 1);
                for (int m = b; m < e && n < cap; m++)
                    if (ro_d2(p, sorted[m]) < r2) n++;
            }
        }
    }
    const int i = idx[k];
    keep[i] = n >= cap ? 1 : 0;
    if (counts) counts[i] = (int32_t)(n < cap ? n : cap);
}

struct RoLayout {
    size_t keys[2], idx[2], sorted, cub, total;
};
RoLayout ro_layout(int32_t P) {
    RoLayout L{};
    const size_t n = P > 0 ? (size_t)P : 0;
    size_t o = 0;
    L.keys[0] = o; o = sr_align_up(o + n * 8);
    L.keys[1] = o; o = sr_align_up(o + n * 8);
    L.idx[0] = o;  o = sr_align_up(o + n * 4);
    L.idx[1] = o;  o = sr_align_up(o + n * 4);
    L.sorted = o;  o = sr_align_up(o + n * 16);
    // cub's radix sort with double buffers needs a look-back or spine of about one 32-bit word per digit per tile of
    // items (< 4 bytes per item) and a few KB of histograms; sr_radius_outlier_mask checks cub's own figure against this
    L.cub = o;     o = sr_align_up(o + n * 4 + RO_CUB_SLACK);
    L.total = n ? o : 0;
    return L;
}

}  // namespace

extern "C" {

SR_API int64_t sr_radius_outlier_scratch_bytes(int32_t P) { return P > 0 ? (int64_t)ro_layout(P).total : 0; }

SR_API int sr_radius_outlier_mask(int32_t P, const float* points, double radius, int32_t nb_points, uint8_t* keep,
                                  int32_t* counts, void* scratch, int64_t scratch_bytes, void* stream_) {
    if (P < 0) return sr_fail(SR_EINVAL, "P must be >= 0, got %d", P);
    if (nb_points < 0) return sr_fail(SR_EINVAL, "nb_points must be >= 0, got %d", nb_points);
    if (!(radius > 0.0) || !std::isfinite(radius)) return sr_fail(SR_EINVAL, "radius must be finite and > 0");
    if (P == 0) return 0;
    if (!points || !keep || !scratch) return sr_fail(SR_EINVAL, "sr_radius_outlier_mask: a required pointer is NULL");
    const RoLayout L = ro_layout(P);
    if (scratch_bytes < (int64_t)L.total)
        return sr_fail(SR_EINVAL, "scratch holds fewer bytes than sr_radius_outlier_scratch_bytes(%d)", P);
    const double h = radius * (1.0 + 0x1p-20), inv_h = 1.0 / h, r2 = radius * radius;
    char* base = (char*)scratch;
    cub::DoubleBuffer<uint64_t> keys((uint64_t*)(base + L.keys[0]), (uint64_t*)(base + L.keys[1]));
    cub::DoubleBuffer<int> idx((int*)(base + L.idx[0]), (int*)(base + L.idx[1]));
    size_t cub_bytes = 0;
    if (cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, keys, idx, (int)P, 0, 3 * RO_BITS) != cudaSuccess)
        return sr_fail(SR_ECUDA, "sr_radius_outlier_mask: cub radix sort size query failed");
    if (cub_bytes > L.total - L.cub)
        return sr_fail(SR_ECUDA, "sr_radius_outlier_mask: cub needs more temporary storage than reserved for P = %d", P);
    cudaStream_t s = (cudaStream_t)stream_;
    const int nb = (P + RO_THREADS - 1) / RO_THREADS;
    {
        ProfileScope ps("outlier_key", s);
        ro_key_kernel<<<nb, RO_THREADS, 0, s>>>(P, points, inv_h, keys.Current(), idx.Current());
    }
    {
        ProfileScope ps("outlier_sort", s);
        size_t tb = L.total - L.cub;
        if (cub::DeviceRadixSort::SortPairs(base + L.cub, tb, keys, idx, (int)P, 0, 3 * RO_BITS, s) != cudaSuccess)
            return sr_fail(SR_ECUDA, "sr_radius_outlier_mask: cub radix sort failed");
    }
    float4* sorted = (float4*)(base + L.sorted);
    {
        ProfileScope ps("outlier_gather", s);
        ro_gather_kernel<<<nb, RO_THREADS, 0, s>>>(P, points, idx.Current(), sorted);
    }
    {
        ProfileScope ps("outlier_query", s);
        ro_query_kernel<<<nb, RO_THREADS, 0, s>>>(P, sorted, keys.Current(), idx.Current(), inv_h, r2, (long long)nb_points + 1,
                                                  keep, counts);
    }
    sr_count_launch(3);
    return cudaGetLastError() == cudaSuccess ? 0 : SR_ECUDA;
}

}  // extern "C"
