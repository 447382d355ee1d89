// post_common.cuh -- camera / ray helpers shared by the fused post-processing (postprocess.cu) and the fused
// post-processing + loss kernels (loss.cu).  gs/utils/point_utils.py:9-21, gs/gaussian_renderer/__init__.py:121-145.
#pragma once
#include "common.cuh"

namespace post {

struct PostCam {
    float R[9];        // W = world_view_transform[:3,:3] (row-major), used as  rend_normal = W @ n
    float A[9];        // camera-to-world rotation (inverse of the affine view matrix's 3x3), row-major
    float o[3];        // camera-to-world translation (ray origin)
    float fx, fy, cx, cy;
};

// world_view_transform is W2C^T (row-vector convention).  c2w = inverse(W2C) by the adjugate formula.  ox, oy: the
// principal point minus (W/2, H/2) in pixels (0 = the image centre, as point_utils.py:12-13 builds K).
__device__ __forceinline__ PostCam load_cam(const float* __restrict__ wvt, int W, int H, float tanx, float tany, float ox = 0.f,
                                            float oy = 0.f) {
    PostCam c;
    float m[16];
#pragma unroll
    for (int i = 0; i < 16; i++) m[i] = __ldg(wvt + i);
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) c.R[i * 3 + j] = m[i * 4 + j];
    // W2C = wvt^T :  B[i][j] = m[j*4+i],  t[i] = m[12+i]
    float B[9];
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
        for (int j = 0; j < 3; j++) B[i * 3 + j] = m[j * 4 + i];
    const float t0 = m[12], t1 = m[13], t2 = m[14];
    // rows of B: r0,r1,r2 ; inverse columns = cross(r1,r2), cross(r2,r0), cross(r0,r1) / det
    const float c0x = B[4] * B[8] - B[5] * B[7], c0y = B[5] * B[6] - B[3] * B[8], c0z = B[3] * B[7] - B[4] * B[6];
    const float c1x = B[7] * B[2] - B[8] * B[1], c1y = B[8] * B[0] - B[6] * B[2], c1z = B[6] * B[1] - B[7] * B[0];
    const float c2x = B[1] * B[5] - B[2] * B[4], c2y = B[2] * B[3] - B[0] * B[5], c2z = B[0] * B[4] - B[1] * B[3];
    const float inv = 1.0f / (B[0] * c0x + B[1] * c0y + B[2] * c0z);
    c.A[0] = c0x * inv; c.A[1] = c1x * inv; c.A[2] = c2x * inv;
    c.A[3] = c0y * inv; c.A[4] = c1y * inv; c.A[5] = c2y * inv;
    c.A[6] = c0z * inv; c.A[7] = c1z * inv; c.A[8] = c2z * inv;
    c.o[0] = -(c.A[0] * t0 + c.A[1] * t1 + c.A[2] * t2);
    c.o[1] = -(c.A[3] * t0 + c.A[4] * t1 + c.A[5] * t2);
    c.o[2] = -(c.A[6] * t0 + c.A[7] * t1 + c.A[8] * t2);
    c.fx = W / (2.0f * tanx); c.fy = H / (2.0f * tany); c.cx = W * 0.5f + ox; c.cy = H * 0.5f + oy;
    return c;
}

__device__ __forceinline__ void ray_dir(const PostCam& c, int x, int y, float& dx, float& dy, float& dz) {
    // (x, y, 1) K^-1, then rotated to world: integer pixel coordinates, as point_utils.py:14-16 builds the grid
    const float u = ((float)x - c.cx) / c.fx, v = ((float)y - c.cy) / c.fy;
    dx = c.A[0] * u + c.A[1] * v + c.A[2];
    dy = c.A[3] * u + c.A[4] * v + c.A[5];
    dz = c.A[6] * u + c.A[7] * v + c.A[8];
}

__device__ __forceinline__ float nan_to_num00(float v) {   // torch.nan_to_num(v, 0, 0): nan -> 0, +inf -> 0, -inf -> lowest
    if (isnan(v)) return 0.f;
    if (isinf(v)) return v > 0.f ? 0.f : -3.4028234663852886e38f;
    return v;
}


}  // namespace post
