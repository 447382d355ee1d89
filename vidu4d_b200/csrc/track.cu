// track.cu -- dense point tracking on the anchors of the forward-only walk (include/surfel_track.h).
//
// A pixel of frame s is the weighted blend of up to K surfels, each hit at a known point (u, v) of its disc
// (composite_fwd.cu, Stats::ANCHORS).  Those surfels' position and orientation in every frame t are known, so is the
// pixel's point there: X_t = sum_k w_k (mean_t + u_k s_u t_u,t + v_k s_v t_v,t) / sum_k w_k, projected through frame
// t's camera.  One thread per (query, target frame): queries in the caller's order on x, the target on y, so that dense
// queries in raster order read neighbouring anchor words and share the surfel rows of each frame in L1 and L2.  Nothing
// is written but the outputs.
#include "common.cuh"
#include "surfel_geom.cuh"
#include "../../include/surfel_camera.h"
#include "../../include/surfel_track.h"

namespace {
using namespace sgeo;
using rn::fa;
using rn::ff;
using rn::fm;

struct TrackArgs {
    int N, T, S, P, K, W, H;
    const int32_t* queries;
    const int32_t* ids; const float* weights; const float* uv; long long stride;   // elements
    const float* means3D; long long means_stride;                                     // floats, 0 = shared
    const float2* scales;
    const float4* rotations; long long rot_stride;                                    // floats, 0 = shared
    const float* depth; float depth_tol;
    float2* xy; float* z; uint8_t* visible; float* coverage;
};

__global__ void __launch_bounds__(256) track_kernel(const TrackArgs a, const CamParams c0, const FrameStrides fs) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    const int t = blockIdx.y;
    if (n >= a.N) return;
    const size_t out = (size_t)n * a.T + t;
    const int s = __ldg(a.queries + 3 * (size_t)n), x = __ldg(a.queries + 3 * (size_t)n + 1),
              y = __ldg(a.queries + 3 * (size_t)n + 2);
    float sx = 0.f, sy = 0.f, sz = 0.f, sw = 0.f;
    bool ok = s >= 0 && s < a.S && x >= 0 && x < a.W && y >= 0 && y < a.H;
    if (ok) {
        const size_t HW = (size_t)a.W * a.H, pix = (size_t)a.W * y + x;
        const int32_t* ids = a.ids + (size_t)s * a.stride + pix;
        const float* ws = a.weights + (size_t)s * a.stride + pix;
        const float* uv = a.uv + 2 * (size_t)s * a.stride + pix;
        const float* mu = a.means3D + (size_t)t * a.means_stride;
        const float4* rot = a.rotations + (size_t)t * (a.rot_stride / 4);
        for (int k = 0; k < a.K; k++) {
            const int32_t id = __ldg(ids + k * HW);
            if (id < 0) continue;                       // an empty slot
            if (id >= a.P) { ok = false; break; }
            const float w = __ldg(ws + k * HW);
            const float u = __ldg(uv + 2 * k * HW), v = __ldg(uv + (2 * k + 1) * HW);
            float R[9];
            rot_matrix(__ldg(rot + id), R);
            const float2 sc = __ldg(a.scales + id);
            const float au = fm(u, sc.x), av = fm(v, sc.y);
            // mean + au t_u + av t_v: t_u = (R[0], R[1], R[2]) and t_v = (R[3], R[4], R[5]), the columns the
            // preprocess scales into M0 and M1
            const float px = ff(av, R[3], ff(au, R[0], __ldg(mu + 3 * (size_t)id)));
            const float py = ff(av, R[4], ff(au, R[1], __ldg(mu + 3 * (size_t)id + 1)));
            const float pz = ff(av, R[5], ff(au, R[2], __ldg(mu + 3 * (size_t)id + 2)));
            sx = ff(w, px, sx); sy = ff(w, py, sy); sz = ff(w, pz, sz);
            sw = fa(sw, w);
        }
        ok = ok && sw > 0.0f;
    }
    if (t == 0) a.coverage[n] = ok ? sw : 0.0f;
    if (!ok) {
        a.xy[out] = make_float2(__int_as_float(0x7fffffff), __int_as_float(0x7fffffff));
        a.z[out] = __int_as_float(0x7fffffff);
        a.visible[out] = 0;
        return;
    }
    const CamParams c = cam_of_frame(c0, fs, t);
    const View V = load_view(c.vm);
    const float3 X = make_float3(__fdiv_rn(sx, sw), __fdiv_rn(sy, sw), __fdiv_rn(sz, sw));
    const float3 p0 = w_mul(V, X);
    const float vx = fa(p0.x, V.m[12]), vy = fa(p0.y, V.m[13]), vz = fa(p0.z, V.m[14]);
    const float px = ff(c.focal_x, __fdiv_rn(vx, vz), c.cx);
    const float py = ff(c.focal_y, __fdiv_rn(vy, vz), c.cy);
    bool vis = vz >= 0.2f && px >= 0.0f && px < (float)a.W && py >= 0.0f && py < (float)a.H;
    if (vis && a.depth) {
        const float d = __ldg(a.depth + (size_t)t * a.W * a.H + (size_t)a.W * (int)py + (int)px);
        vis = fabsf(fa(vz, -d)) <= fm(a.depth_tol, vz);
    }
    a.xy[out] = make_float2(px, py);
    a.z[out] = vz;
    a.visible[out] = vis ? 1 : 0;
}

}  // namespace

extern "C" int sr_track_pixels(int32_t N, int32_t T, int32_t S, int32_t P, int32_t K, int32_t width, int32_t height,
                               const int32_t* queries, const int32_t* anchor_ids, const float* anchor_weights,
                               const float* anchor_uv, int64_t anchor_stride, const float* means3D,
                               int64_t means3D_stride, const float* scales, const float* rotations,
                               int64_t rotations_stride, const float* viewmatrix, float tan_fovx, float tan_fovy,
                               const float* cameras, const float* depth, float depth_tolerance, float* xy, float* z,
                               uint8_t* visible, float* coverage, void* stream) {
    if (N < 0 || T < 0 || S < 0 || P < 0) return sr_fail(SR_EINVAL, "track: N, T, S and P must be >= 0");
    if (T > 65535) return sr_fail(SR_EINVAL, "track: T must be <= 65535, got %d", T);
    if (K != 1 && K != 2 && K != 4 && K != 8) return sr_fail(SR_EINVAL, "track: K must be 1, 2, 4 or 8, got %d", K);
    if (width <= 0 || height <= 0 || width > 65535 || height > 65535)
        return sr_fail(SR_EINVAL, "track: image size must be in [1, 65535]");
    if (anchor_stride < (int64_t)K * width * height) return sr_fail(SR_EINVAL, "track: anchor frame stride must be >= K*H*W");
    if (means3D_stride != 0 && means3D_stride < 3ll * P)
        return sr_fail(SR_EINVAL, "track: means3D frame stride must be 0 or >= 3*P floats");
    if (rotations_stride != 0 && (rotations_stride < 4ll * P || rotations_stride % 4 != 0))
        return sr_fail(SR_EINVAL, "track: rotations frame stride must be 0 or a multiple of 4 that is >= 4*P floats");
    if (!(depth_tolerance >= 0.0f)) return sr_fail(SR_EINVAL, "track: depth_tolerance must be >= 0");
    if (!cameras && !(tan_fovx > 0.0f && tan_fovy > 0.0f))
        return sr_fail(SR_EINVAL, "track: tan_fovx and tan_fovy must be positive without a camera table");
    if (N == 0 || T == 0) return 0;
    if (!queries || !xy || !z || !visible || !coverage) return sr_fail(SR_EINVAL, "track: query or output pointer is NULL");
    if (!anchor_ids || !anchor_weights || !anchor_uv) return sr_fail(SR_EINVAL, "track: anchor pointer is NULL");
    if (P > 0 && (!means3D || !scales || !rotations)) return sr_fail(SR_EINVAL, "track: surfel pointer is NULL");
    if (!viewmatrix) return sr_fail(SR_EINVAL, "track: viewmatrix is NULL");
    if (((uintptr_t)queries & 3) || ((uintptr_t)anchor_ids & 3) || ((uintptr_t)anchor_weights & 3) ||
        ((uintptr_t)anchor_uv & 3) || ((uintptr_t)means3D & 3) || ((uintptr_t)viewmatrix & 3) ||
        ((uintptr_t)cameras & 3) || ((uintptr_t)depth & 3) || ((uintptr_t)z & 3) || ((uintptr_t)coverage & 3))
        return sr_fail(SR_EINVAL, "track: float and int32 arrays must be 4-byte aligned");
    if (((uintptr_t)scales & 7) || ((uintptr_t)xy & 7)) return sr_fail(SR_EINVAL, "track: scales and xy must be 8-byte aligned");
    if ((uintptr_t)rotations & 15) return sr_fail(SR_EINVAL, "track: rotations must be 16-byte aligned");

    // the forward's camera: make_cam's intrinsics, or cam_of_frame's per-frame table rows
    sr_frame f{};
    f.P = P; f.width = width; f.height = height; f.tan_fovx = tan_fovx; f.tan_fovy = tan_fovy;
    sr_frame_cameras fc{};
    if (cameras) { fc.frame = f; fc.frame.flags = SR_FRAME_CAMERAS; fc.cameras = cameras; }
    const CamParams cam = make_cam(cameras ? &fc.frame : &f, viewmatrix, nullptr, nullptr);
    FrameStrides fs{};
    fs.frames = T; fs.vm = 16 * sizeof(float);
    TrackArgs a{N, T, S, P, K, width, height, queries, anchor_ids, anchor_weights, anchor_uv, anchor_stride,
                means3D, means3D_stride, reinterpret_cast<const float2*>(scales), reinterpret_cast<const float4*>(rotations),
                rotations_stride, depth, depth_tolerance, reinterpret_cast<float2*>(xy), z, visible, coverage};
    {
        ProfileScope ps("track_pixels", (cudaStream_t)stream);
        track_kernel<<<dim3((unsigned)((N + 255) / 256), (unsigned)T), 256, 0, (cudaStream_t)stream>>>(a, cam, fs);
    }
    return sr_launched(1, "track_pixels");
}
