/*
 * surfel_raster.h -- C ABI of the H100-native Gaussian-surfel rasterizer.
 *
 * This is the drop-in boundary for the hot path of yikaiw/Vidu4D's Stage-3
 * ("dynamic Gaussian surfels"): it replaces
 *
 *     CudaRasterizer::Rasterizer::forward      RAST/cuda_rasterizer/rasterizer.h:33-59
 *     CudaRasterizer::Rasterizer::backward     RAST/cuda_rasterizer/rasterizer.h:61-87
 *     CudaRasterizer::Rasterizer::markVisible  RAST/cuda_rasterizer/rasterizer.h:25-31
 *
 * (RAST = gs/submodules/diff-surfel-rasterization) which the reference reaches
 * through its pybind module `_C` (RAST/ext.cpp:15-19, RAST/rasterize_points.cu:39-261).
 * Plain pointers and sizes only -- no torch types.  All pointers are DEVICE
 * pointers unless stated; `stream` is a cudaStream_t passed as void* (NULL = the
 * legacy default stream, which is what the reference always uses).
 *
 * Differences from the reference interface, on purpose:
 *   - The reference grows its three scratch buffers through std::function
 *     callbacks and blocks on a D2H copy of `num_rendered` in the middle of
 *     forward() (rasterizer_impl.cu:282).  Here the caller sizes the buffers up
 *     front with the sr_*_bytes() queries; the instance buffer has a CAPACITY and
 *     forward() never synchronises: `num_rendered` lands in a caller-supplied
 *     (pinned) host word asynchronously.  If the capacity is too small the frame
 *     is not rendered and SR_STATUS_OVERFLOW is reported through `status`
 *     (see sr_forward()).
 *   - `transMat_precomp` ("cov3D_precomp" at the Python level) is rejected: the
 *     reference's own path for it leaves the normal uninitialised
 *     (forward.cu:214-218) and nothing in Vidu4D uses it.
 *   - The opaque buffer layouts are ours (see DESIGN.md, "HBM layout"); use
 *     sr_debug_view() to look inside them in tests.
 *
 * Every function returns 0 on success, a negative SR_E* code on error;
 * sr_last_error() returns a human-readable message for the calling thread.
 */
#ifndef SURFEL_RASTER_H_
#define SURFEL_RASTER_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SR_ABI_VERSION 3

#if defined(__GNUC__)
#define SR_API __attribute__((visibility("default")))
#else
#define SR_API
#endif

#define SR_EINVAL   (-1)   /* bad argument (shape, null pointer, unsupported option) */
#define SR_ECUDA    (-2)   /* a CUDA runtime call or launch failed */
#define SR_ECAPACITY (-3)  /* instance capacity exceeded (only from the synchronous helpers) */

/* bits of the device/host status word written by sr_forward() */
#define SR_STATUS_OK        0u
#define SR_STATUS_OVERFLOW  1u   /* num_rendered > capacity: nothing was binned or composited */
#define SR_STATUS_PREFILTER 4u   /* prefiltered was set but a surfel was culled (the reference __trap()s) */

/* One frame's static description (GaussianRasterizationSettings,
 * RAST/diff_surfel_rasterization/__init__.py:158-170, plus P/M). */
typedef struct sr_frame {
    int32_t P;             /* number of surfels */
    int32_t sh_degree;     /* active SH degree D (0..3) */
    int32_t sh_coeffs;     /* M = shs.size(1); 0 when colors_precomp is used */
    int32_t width, height;
    float   tan_fovx, tan_fovy;
    float   scale_modifier;  /* accepted and ignored, exactly like the reference (forward.cu:95) */
    int32_t prefiltered;     /* if set, a culled surfel is an error in the reference (__trap); we report it via status bit 2 */
    int32_t debug;           /* if set, synchronise + check after every launch (auxiliary.h:271-278) */
    uint32_t flags;          /* reserved, must be 0 */
} sr_frame;

/* ---- buffer sizing (replaces required<GeometryState/ImageState/BinningState>, rasterizer_impl.h:66-72) */
SR_API size_t sr_geom_bytes(int32_t P);
SR_API size_t sr_image_bytes(int32_t width, int32_t height);
/* 136 B per instance of capacity (sort ping/pong, sorted record stream, per-pixel contribution masks kept for the
 * backward) + 1 KB per 16x16 tile: the SAME (capacity, width, height) must be passed to the backward. */
SR_API size_t sr_binning_bytes(int64_t capacity /* max instances */, int32_t width, int32_t height);

/*
 * Forward.  Replaces Rasterizer::forward (rasterizer_impl.cu:198-342).
 *
 *   background[3], means3D[P*3], shs[P*M*3] | colors_precomp[P*3] (exactly one non-NULL),
 *   opacities[P], scales[P*2], rotations[P*4] (w,x,y,z), viewmatrix[16], projmatrix[16], campos[3]
 *   out_color[3*H*W], out_others[8*H*W], radii[P] (int32)           -- written
 *   geom/binning/image buffers: caller-allocated, sizes from sr_*_bytes()
 *   capacity: number of instances the binning buffer was sized for
 *   num_rendered_dev: device uint32[2] -> {num_rendered, status}; also copied
 *       asynchronously to num_rendered_host (pinned host uint32[2]) if non-NULL.
 */
SR_API int sr_forward(const sr_frame* f,
               const float* background, const float* means3D, const float* shs,
               const float* colors_precomp, const float* opacities, const float* scales,
               const float* rotations, const float* viewmatrix, const float* projmatrix,
               const float* campos,
               float* out_color, float* out_others, int32_t* radii,
               void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
               uint32_t* num_rendered_dev, uint32_t* num_rendered_host, void* stream);

/*
 * Backward.  Replaces Rasterizer::backward (rasterizer_impl.cu:346-448).
 * Inputs as in forward plus dL_dout_color[3*H*W], dL_dout_others[8*H*W] and the
 * three buffers the forward filled.  Outputs (all fully written, no need to zero):
 *   dL_dmeans2D[P*3] (the densification proxy of backward.cu:645-648; z = 0),
 *   dL_dcolors[P*3], dL_dopacity[P], dL_dmeans3D[P*3], dL_dtransMat[P*9],
 *   dL_dsh[P*M*3], dL_dscales[P*2], dL_drotations[P*4]
 */
SR_API int sr_backward(const sr_frame* f,
                const float* background, const float* means3D, const float* shs,
                const float* colors_precomp, const float* scales, const float* rotations,
                const float* viewmatrix, const float* projmatrix, const float* campos,
                const int32_t* radii,
                const float* dL_dout_color, const float* dL_dout_others,
                void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
                float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                void* stream);

/*
 * Batched entry points (SURVEY.md section 8(f) row N1): M independent frames -- different cameras, and optionally
 * different surfel sets, as in Stage 3 where every frame rasterizes its own bob-warped copy of the canonical surfels
 * (lab4d/nnutils/deformable_gaussian.py:1175-1188 loops frames in Python) -- in ONE launch set: every kernel of the
 * path gets a frame dimension, so a step costs the same ~15 launches whatever M is and the GPU sees M x the CTAs.
 *
 * Layout: viewmatrix[M*16], projmatrix[M*16], campos[M*3]; out_color[M*3*H*W], out_others[M*8*H*W], radii[M*P];
 * geom/binning/image buffers are M consecutive per-frame buffers of sr_*_bytes() each (same capacity for every frame);
 * num_rendered_dev / num_rendered_host are uint32[M*2] = {num_rendered, status} per frame.  Per-surfel inputs are
 * addressed as base + frame * stride (in floats; sr_batch), stride 0 = shared by all frames.  background[3] is shared.
 * Backward: dL_dout_color[M*3*H*W], dL_dout_others[M*8*H*W]; every gradient output is written per frame, (M, P, .)
 * -- except, with SR_BATCH_SUM_SHARED, those of shared inputs, which are (P, .) sums over the frames; dL_dmeans2D is always
 * per frame; dL_dtransMat may be NULL in the batched call (it is only a by-product);
 * grad_scale (optional DEVICE scalar, NULL = 1) multiplies dL_dout_* -- the upstream scalar of a fused loss.
 * sr_forward / sr_backward are the M = 1 case.
 */
#define SR_BATCH_SUM_SHARED 1u   /* backward: an input shared by the frames (stride 0) gets ONE gradient (P, .), the sum over
                                    the frames, accumulated inside the per-surfel kernel and written once -- instead of
                                    (M, P, .) per-frame gradients the caller would have to reduce */
typedef struct sr_batch {
    int32_t frames;                                   /* M >= 1 */
    uint32_t flags;                                   /* SR_BATCH_* */
    int64_t means3D, shs, colors_precomp, opacities, scales, rotations;   /* floats between consecutive frames; 0 = shared */
} sr_batch;

SR_API int sr_forward_batch(const sr_frame* f, const sr_batch* b,
               const float* background, const float* means3D, const float* shs,
               const float* colors_precomp, const float* opacities, const float* scales,
               const float* rotations, const float* viewmatrix, const float* projmatrix,
               const float* campos,
               float* out_color, float* out_others, int32_t* radii,
               void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
               uint32_t* num_rendered_dev, uint32_t* num_rendered_host, void* stream);

SR_API int sr_backward_batch(const sr_frame* f, const sr_batch* b,
                const float* background, const float* means3D, const float* shs,
                const float* colors_precomp, const float* scales, const float* rotations,
                const float* viewmatrix, const float* projmatrix, const float* campos,
                const int32_t* radii,
                const float* dL_dout_color, const float* dL_dout_others, const float* grad_scale,
                void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
                float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations,
                void* stream);

/* Replaces Rasterizer::markVisible (rasterizer_impl.cu:141-153): present[i] = p_view.z > 0.2 */
SR_API int sr_mark_visible(int32_t P, const float* means3D, const float* viewmatrix, const float* projmatrix,
                    uint8_t* present, void* stream);

/* ---- introspection for tests: byte offsets of the sub-arrays inside our opaque buffers */
typedef struct sr_debug_layout {
    /* geometry buffer (per surfel) */
    size_t surfel_rec;      /* float[P*20]  packed record, see DESIGN.md */
    size_t depths;          /* float[P]     view-space z (sort key low word) */
    size_t tiles_touched;   /* uint32[P] */
    size_t point_offsets;   /* uint32[P]    inclusive scan of tiles_touched */
    size_t clamped;         /* uint8[P]     bit c set = colour channel c clamped at 0 */
    /* binning buffer (per instance); the sorted arrays live in ping or pong: read `sorted_sel` first */
    size_t keys[2];         /* uint64[capacity] x2 */
    size_t values[2];       /* uint32[capacity] x2 */
    size_t sort_ctl;        /* uint32[..]: [0]=sorted_sel (0/1) after forward */
    size_t inst_rec;        /* float[capacity*20] per-instance record stream */
    size_t contrib;         /* uint32[((capacity>>5)+tiles+1)*256] per (32-instance stage, 8x4 sub-tile, pixel) contribution masks */
    /* image buffer */
    size_t final_T;         /* float[3*N]  T, M1, M2 */
    size_t n_contrib;       /* uint32[2*N] last, median */
    size_t ranges;          /* uint32[tiles*2] */
    size_t sub_last;        /* uint32[tiles*8] deepest contributor (list position + 1) per 8x4 sub-tile */
} sr_debug_layout;
SR_API int sr_debug_view(int32_t P, int32_t width, int32_t height, int64_t capacity, sr_debug_layout* out);

/*
 * Fused post-processing of `allmap` (SURVEY.md section 8(f) row N1): everything gs/gaussian_renderer/__init__.py:121-162
 * and gs/utils/point_utils.py:9-37 compute from the rasterizer's 8 planes, in one pass each way.
 * world_view_transform is the camera's (4,4) W2C^T exactly as GaussianRasterizationSettings.viewmatrix.
 * forward writes acc[HW], rend_normal[3HW], rend_dist[HW], depth_median[HW], depth_expected[HW], surf_depth[HW],
 * surf_normal[3HW]; backward takes their gradients and writes g_allmap[8HW] (fully, no need to zero).
 */
SR_API int sr_post_forward(int32_t W, int32_t H, float tan_fovx, float tan_fovy, float depth_ratio, const float* allmap,
                           const float* world_view_transform, float* acc, float* rend_normal, float* rend_dist,
                           float* depth_median, float* depth_expected, float* surf_depth, float* surf_normal, void* stream);
SR_API int sr_post_backward(int32_t W, int32_t H, float tan_fovx, float tan_fovy, float depth_ratio, const float* allmap,
                            const float* world_view_transform, const float* surf_depth, const float* g_acc,
                            const float* g_rend_normal, const float* g_rend_dist, const float* g_depth_median,
                            const float* g_depth_expected, const float* g_surf_depth, const float* g_surf_normal,
                            float* g_allmap, void* stream);

/*
 * Stage-3 image losses fused with the render() post-processing, forward and backward in one pass, M frames per call
 * (SURVEY.md section 8(f) row N1).  Replaces lab4d/engine/model.py:674-692 (masked L1), :649-653 (mask loss), :817-842
 * (normal + distortion regularisers) on top of gs/gaussian_renderer/__init__.py:121-145 and, optionally, the
 * learnable-background composite of lab4d/nnutils/deformable_gaussian.py:188-190.
 *   color[M*3*HW], allmap[M*8*HW] (the rasterizer's outputs), world_view_transform[M*16], target_rgb[M*3*HW];
 *   vis2d[M*HW] (NULL = all visible), mask_gt[M*HW] (NULL = no mask term), mask_wt[M*HW] (NULL = 1),
 *   learnable_bkgd[3] (NULL = none).
 * Writes loss_terms[M*4] = weighted {rgb, mask, normal, dist} per frame (means over the frame's pixels), and the gradient
 * of their sum: dL_dcolor[M*3*HW], dL_dallmap[M*8*HW] (fully written), dL_dbkgd[M*3] (if non-NULL).
 * surf_depth_scratch: M*HW floats.
 */
SR_API int sr_render_loss_batch(int32_t M, int32_t W, int32_t H, float tan_fovx, float tan_fovy, float depth_ratio,
                                const float* color, const float* allmap, const float* world_view_transform,
                                const float* target_rgb, const float* vis2d, const float* mask_gt, const float* mask_wt,
                                const float* learnable_bkgd, float w_rgb, float w_mask, float lambda_normal, float lambda_dist,
                                float* loss_terms, float* dL_dcolor, float* dL_dallmap, float* dL_dbkgd,
                                float* surf_depth_scratch, void* stream);

/*
 * Fused bob-skinning warp (SURVEY.md section 8(f) rows N2/N3): canonical surfels -> every frame's camera space.
 * Replaces the PyTorch chain of lab4d/nnutils/deformable_gaussian.py:1395-1434 (forward_warp), :1033-1046
 * (apply_qt_to_gaussian), lab4d/nnutils/warping.py:378-444 (SkinningWarp.forward, forward direction),
 * lab4d/nnutils/skinning.py:89-142 (Gaussian skinning logits), lab4d/utils/geom_utils.py:48-92 (sign-aligned
 * dual-quaternion blend) and the quaternion helper kernels of lab4d/third_party/quaternion/src/quaternion.cu.
 *   xyz[P*3], rot[P*4] (w,x,y,z): canonical surfels;  o2b_q[B*4], o2b_t[B*3]: object->bone transform of the rest pose;
 *   inv_gauss[B*3] = exp(-log_gauss);  delta[P*B] or NULL;  se3_r, se3_d[M*B*4]: per frame and bone dual quaternion
 *   t_articulation o rest_articulation^-1;  cam_q[M*4], cam_t[M*3]: field2cam.   B <= 64.
 * forward writes xyz_cam[M*P*3], rot_cam[M*P*4] (feed them to sr_forward_batch with per-frame strides) and
 * skin_entropy[P] (may be NULL).  backward takes their gradients (g_entropy may be NULL) and writes g_xyz[P*3], g_rot[P*4],
 * g_delta[P*B] (if non-NULL) and g_tables[sr_bob_warp_table_floats(B, M)] = gradients of {o2b_q, o2b_t, inv_gauss, se3_r,
 * se3_d, cam_q, cam_t} in that order (zeroed inside).
 */
SR_API size_t sr_bob_warp_table_floats(int32_t B, int32_t M);
SR_API int sr_bob_warp_forward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* rot, const float* o2b_q,
                               const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                               const float* se3_d, const float* cam_q, const float* cam_t, float* xyz_cam, float* rot_cam,
                               float* skin_entropy, void* stream);
SR_API int sr_bob_warp_backward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* rot, const float* o2b_q,
                                const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                const float* se3_d, const float* cam_q, const float* cam_t, const float* g_xyz_cam,
                                const float* g_rot_cam, const float* g_entropy, float* g_xyz, float* g_rot, float* g_delta,
                                float* g_tables, void* stream);

/*
 * Optimizer-side kernels over the FLAT surfel parameter buffer (SURVEY.md section 8(f) row N4): the Adam step of every
 * surfel parameter group in one launch (lab4d/engine/trainer.py:243-253,585-586; torch.optim.Adam semantics), and
 * densify / prune as one gather into new buffers (gs/scene/gaussian_model.py:291-446).  See csrc/optim.cu.
 */
SR_API int sr_adam_flat(int32_t n_groups, const int64_t* begin, const float* lr, float beta1, float beta2, float eps,
                        int64_t step, float grad_scale, float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                        void* stream);
SR_API int sr_surfel_compact(int32_t n_groups, const int32_t* width, const int64_t* old_begin, const int64_t* new_begin,
                             int32_t xyz_group, int32_t scaling_group, int32_t P_new, const int32_t* src, const uint8_t* kind,
                             const int32_t* child_slot, const float* child_xyz, const float* child_scaling, const float* p_old,
                             const float* m_old, const float* v_old, float* p_new, float* m_new, float* v_new, void* stream);

/*
 * Mean squared distance of every point to its 3 nearest neighbours: `distCUDA2` of gs/submodules/simple-knn
 * (simple_knn.cu:132-218), used once to initialise the surfel scales (gs/scene/gaussian_model.py:139-140).
 * sr_knn_cells() gives the grid size for a bounding box (host floats); scratch = device int32[2*P + 3*cells].
 */
SR_API int64_t sr_knn_cells(int32_t P, const float* bbox_min, const float* bbox_max, float* h_out, int32_t* dims_out);
SR_API int sr_knn_mean_dist2(int32_t P, const float* points, const float* bbox_min, const float* bbox_max, float* out,
                             int32_t* scratch, void* stream);

SR_API int sr_abi_version(void);
SR_API const char* sr_last_error(void);
/* number of kernel launches issued by this library since load (bench.py's `gpu_launches`) */
SR_API uint64_t sr_launch_count(void);
/* per-kernel device timing for bench.py's roofline: CUDA events on the launching stream around every kernel */
SR_API void sr_set_profiling(int on);
SR_API const char* sr_get_profile(void);   /* JSON {"kernel": {"ms": total, "count": n}}; synchronises */

#ifdef __cplusplus
}
#endif
#endif /* SURFEL_RASTER_H_ */
