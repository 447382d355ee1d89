// knn.cu -- mean squared distance to the 3 nearest neighbours of every point (surfel-scale initialisation).
//
// Replaces (behaviour, not code) of gs/submodules/simple-knn/simple_knn.cu:132-218 (`distCUDA2`), which the reference
// calls once when the surfels are created (gs/scene/gaussian_model.py:139-140: scales = log(sqrt(dist2))).  The
// reference sorts the points along a Morton curve and scans boxes of 1024 with a box-distance reject test; here the
// points are binned into a uniform grid (counting sort: count -> scan -> scatter) and every point searches growing cubic
// shells of cells until its third-nearest distance is provably final.  Exact 3-NN, same result: (d0 + d1 + d2) / 3 with
// the three smallest squared distances to OTHER points (duplicates count with distance 0, as in the reference).
#include <cfloat>

#include "common.cuh"

namespace {

struct Grid {
    float minx, miny, minz, inv_h, h;
    int nx, ny, nz;
};
__device__ __forceinline__ int3 cell_of(const Grid& g, float x, float y, float z) {
    int cx = (int)((x - g.minx) * g.inv_h), cy = (int)((y - g.miny) * g.inv_h), cz = (int)((z - g.minz) * g.inv_h);
    cx = min(max(cx, 0), g.nx - 1); cy = min(max(cy, 0), g.ny - 1); cz = min(max(cz, 0), g.nz - 1);
    return make_int3(cx, cy, cz);
}
__device__ __forceinline__ int cell_id(const Grid& g, int3 c) { return (c.z * g.ny + c.y) * g.nx + c.x; }

__global__ void knn_count_kernel(const Grid g, int P, const float* __restrict__ pts, int* __restrict__ cell, int* __restrict__ count) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int c = cell_id(g, cell_of(g, pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2]));
    cell[i] = c;
    atomicAdd(count + c, 1);
}
__global__ void knn_scatter_kernel(int P, const int* __restrict__ cell, const int* __restrict__ start, int* __restrict__ cursor,
                                   int* __restrict__ order) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const int c = cell[i];
    order[start[c] + atomicAdd(cursor + c, 1)] = i;
}
__device__ __forceinline__ void k_best(float (&best)[3], float d) {
#pragma unroll
    for (int j = 0; j < 3; j++) if (best[j] > d) { const float t = best[j]; best[j] = d; d = t; }
}
__global__ void knn_query_kernel(const Grid g, int P, const float* __restrict__ pts, const int* __restrict__ start,
                                 const int* __restrict__ count, const int* __restrict__ order, float* __restrict__ out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= P) return;
    const float x = pts[3 * (size_t)i], y = pts[3 * (size_t)i + 1], z = pts[3 * (size_t)i + 2];
    const int3 c = cell_of(g, x, y, z);
    // FLT_MAX, as simple_knn.cu: with fewer than three other points the mean is (d0 + d1 + FLT_MAX) / 3 (3 points) or
    // Inf (1 or 2 points)
    float best[3] = {FLT_MAX, FLT_MAX, FLT_MAX};
    const int rmax = max(g.nx, max(g.ny, g.nz));
    for (int r = 0; r <= rmax; r++) {
        // cells at Chebyshev distance exactly r from the point's own cell
        for (int dz = -r; dz <= r; dz++) {
            const int cz = c.z + dz;
            if (cz < 0 || cz >= g.nz) continue;
            for (int dy = -r; dy <= r; dy++) {
                const int cy = c.y + dy;
                if (cy < 0 || cy >= g.ny) continue;
                const bool face = (abs(dz) == r) || (abs(dy) == r);
                for (int dx = -r; dx <= r; dx += (face ? 1 : max(2 * r, 1))) {      // interior rows: only the two end cells
                    const int cx = c.x + dx;
                    if (cx < 0 || cx >= g.nx) continue;
                    const int cid = (cz * g.ny + cy) * g.nx + cx;
                    const int s = start[cid], n = count[cid];
                    for (int k = 0; k < n; k++) {
                        const int j = order[s + k];
                        if (j == i) continue;
                        const float ex = pts[3 * (size_t)j] - x, ey = pts[3 * (size_t)j + 1] - y, ez = pts[3 * (size_t)j + 2] - z;
                        k_best(best, ex * ex + ey * ey + ez * ez);
                    }
                }
            }
        }
        // every unscanned point lies at least r * h away (the point sits inside its own cell): stop once the third-nearest
        // distance found so far cannot be beaten
        const float reach = (float)r * g.h;
        if (best[2] <= reach * reach) break;
    }
    out[i] = (best[0] + best[1] + best[2]) / 3.0f;
}

// exclusive scan of the cell counts (cells can be millions; a single-block chunked scan is plenty for an
// initialisation-time routine)
__global__ void __launch_bounds__(1024)
knn_scan_kernel(const int* __restrict__ cnt, int* __restrict__ st, long long n) {
    __shared__ int wtot[32];
    __shared__ int carry;
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (long long base = 0; base < n; base += 1024) {
        const long long i = base + threadIdx.x;
        const int v = i < n ? cnt[i] : 0;
        int inc = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, inc, o); if ((threadIdx.x & 31) >= o) inc += t; }
        if ((threadIdx.x & 31) == 31) wtot[threadIdx.x >> 5] = inc;
        __syncthreads();
        if (threadIdx.x < 32) {
            const int w = wtot[threadIdx.x];
            int winc = w;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, winc, o); if (threadIdx.x >= o) winc += t; }
            wtot[threadIdx.x] = winc - w;
        }
        __syncthreads();
        const int excl = carry + wtot[threadIdx.x >> 5] + inc - v;
        if (i < n) st[i] = excl;
        __syncthreads();
        if (threadIdx.x == 1023) carry = excl + v;
        __syncthreads();
    }
}

}  // namespace

extern "C" {

/* Mean of the three smallest squared distances from every point to the other points (simple_knn.cu:147-183).
 * points[P*3], out[P]; bbox_min/max: HOST float[3] bounding box of the points; scratch: device int32[2*P + 3*cells] with
 * cells = sr_knn_cells(P, bbox): the caller zero-fills nothing (done here). */
SR_API int64_t sr_knn_cells(int32_t P, const float* bbox_min, const float* bbox_max, float* h_out, int32_t* dims_out) {
    if (P <= 0 || !bbox_min || !bbox_max) return 0;
    double ex = fmax((double)bbox_max[0] - bbox_min[0], 1e-12), ey = fmax((double)bbox_max[1] - bbox_min[1], 1e-12),
           ez = fmax((double)bbox_max[2] - bbox_min[2], 1e-12);
    // ~2 points per cell of the bounding volume; surface-like clouds leave most cells empty, which only costs memory
    double h = cbrt(ex * ey * ez / fmax(P / 2.0, 1.0));
    h = fmax(h, fmax(ex, fmax(ey, ez)) / 512.0);              // at most 512 cells per axis
    int nx = (int)(ex / h) + 1, ny = (int)(ey / h) + 1, nz = (int)(ez / h) + 1;
    while ((int64_t)nx * ny * nz > (int64_t)(1 << 26)) { h *= 1.26; nx = (int)(ex / h) + 1; ny = (int)(ey / h) + 1; nz = (int)(ez / h) + 1; }
    if (h_out) *h_out = (float)h;
    if (dims_out) { dims_out[0] = nx; dims_out[1] = ny; dims_out[2] = nz; }
    return (int64_t)nx * ny * nz;
}

SR_API int sr_knn_mean_dist2(int32_t P, const float* points, const float* bbox_min, const float* bbox_max, float* out,
                             int32_t* scratch, void* stream_) {
    if (P < 0) return sr_fail(SR_EINVAL, "sr_knn_mean_dist2: P must be >= 0, got %d", P);
    if (P == 0) return 0;
    if (!points || !bbox_min || !bbox_max || !out || !scratch) return sr_fail(SR_EINVAL, "sr_knn_mean_dist2: a required pointer is NULL");
    float h; int dims[3];
    const int64_t cells = sr_knn_cells(P, bbox_min, bbox_max, &h, dims);
    Grid g{bbox_min[0], bbox_min[1], bbox_min[2], 1.0f / h, h, dims[0], dims[1], dims[2]};
    cudaStream_t s = (cudaStream_t)stream_;
    int* cell = scratch; int* order = cell + P; int* count = order + P; int* start = count + cells; int* cursor = start + cells;
    CK(cudaMemsetAsync(count, 0, (size_t)cells * 3 * sizeof(int), s), "sr_knn_mean_dist2: memset(scratch)");
    const int nb = (P + 255) / 256;
    knn_count_kernel<<<nb, 256, 0, s>>>(g, P, points, cell, count);
    knn_scan_kernel<<<1, 1024, 0, s>>>(count, start, (long long)cells);
    knn_scatter_kernel<<<nb, 256, 0, s>>>(P, cell, start, cursor, order);
    knn_query_kernel<<<nb, 256, 0, s>>>(g, P, points, start, count, order, out);
    return sr_launched(4, "sr_knn_mean_dist2");
}

}  // extern "C"
