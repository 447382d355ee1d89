// surfel_geom.cuh -- a surfel's rotation matrix and the world-to-view transform, in the forward preprocess's rounding.
// One copy, shared by the preprocess (preprocess.cu) and the tracking kernel (track.cu), so that a tracked point moves
// with the surfel exactly as the rasterizer places it.
#pragma once
#include "common.cuh"

namespace sgeo {
namespace rn {
__device__ __forceinline__ float fm(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float fa(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float ff(float a, float b, float c) { return __fmaf_rn(a, b, c); }
}  // namespace rn

struct View { float m[16]; };
__device__ __forceinline__ View load_view(const float* __restrict__ vm) {
    View v;
#pragma unroll
    for (int i = 0; i < 16; i++) v.m[i] = __ldg(vm + i);
    return v;
}
// view-space z exactly as transformPoint4x3 contracts it in the reference build
__device__ __forceinline__ float view_z(const View& c, float x, float y, float z) {
    return rn::fa(rn::ff(z, c.m[10], rn::ff(x, c.m[2], rn::fm(y, c.m[6]))), c.m[14]);
}
// glm mat3(W) * v
__device__ __forceinline__ float3 w_mul(const View& c, float3 v) {
    return make_float3(rn::ff(v.z, c.m[8], rn::ff(v.x, c.m[0], rn::fm(v.y, c.m[4]))),
                       rn::ff(v.z, c.m[9], rn::ff(v.x, c.m[1], rn::fm(v.y, c.m[5]))),
                       rn::ff(v.z, c.m[10], rn::ff(v.x, c.m[2], rn::fm(v.y, c.m[6]))));
}

// computeTransMat's rotation matrix R (row-major) of the quaternion q = (w,x,y,z); glm names .x=w .y=x .z=y .w=z
__device__ __forceinline__ void rot_matrix(float4 q, float R[9]) {
    const float n2 = rn::ff(q.z, q.z, rn::ff(q.y, q.y, rn::ff(q.w, q.w, rn::fm(q.x, q.x))));
    const float s = rsqrtf(n2);
    const float w = rn::fm(q.x, s), x = rn::fm(q.y, s), y = rn::fm(q.z, s), z = rn::fm(q.w, s);
    const float wz = rn::fm(w, z), wy = rn::fm(w, y), wx = rn::fm(w, x), yy = rn::fm(y, y), zz = rn::fm(z, z);
    float t;
    t = rn::fa(yy, zz);        R[0] = rn::fa(1.f, -rn::fa(t, t));
    t = rn::ff(x, y, wz);      R[1] = rn::fa(t, t);
    t = rn::ff(x, z, -wy);     R[2] = rn::fa(t, t);
    t = rn::ff(x, y, -wz);     R[3] = rn::fa(t, t);
    t = rn::ff(x, x, zz);      R[4] = rn::fa(1.f, -rn::fa(t, t));
    t = rn::ff(y, z, wx);      R[5] = rn::fa(t, t);
    t = rn::ff(x, z, wy);      R[6] = rn::fa(t, t);
    t = rn::ff(y, z, -wx);     R[7] = rn::fa(t, t);
    t = rn::ff(x, x, yy);      R[8] = rn::fa(1.f, -rn::fa(t, t));
}

}  // namespace sgeo
