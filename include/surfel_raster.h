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

#define SR_ABI_VERSION 10

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
 * Forward and backward.  Replace Rasterizer::forward (rasterizer_impl.cu:198-342) and Rasterizer::backward
 * (rasterizer_impl.cu:346-448), batched (SURVEY.md section 8(f) row N1): M independent frames -- different cameras, and
 * optionally different surfel sets, as in Stage 3 where every frame rasterizes its own bob-warped copy of the canonical
 * surfels (lab4d/nnutils/deformable_gaussian.py:1175-1188 loops frames in Python) -- in ONE launch set: every kernel of
 * the path gets a frame dimension, so a step costs the same ~15 launches whatever M is and the GPU sees M x the CTAs.
 * One frame, as the reference renders it, is the M = 1 case: sr_batch {1, 0, 0, ...}.
 *
 * Inputs: background[bg_channels], means3D[P*3], shs[P*sh_coeffs*3] | colors_precomp[P*3] (exactly one non-NULL),
 *   opacities[P], scales[P*2], rotations[P*4] (w,x,y,z), features[P*F]; viewmatrix[M*16], projmatrix[M*16], campos[M*3].
 *   Per-surfel inputs are addressed as base + frame * stride (in floats; sr_batch, features_stride), stride 0 = shared
 *   by all frames.
 * Forward writes frame m's 3 colour planes at out_color + m * out_color_stride, its F feature planes at out_features +
 *   m * out_features_stride (strides in floats), out_others[M*8*H*W] and radii[M*P] (int32).
 *   geom/binning/image buffers: caller-allocated, M consecutive per-frame buffers of sr_*_bytes() each; capacity: the
 *   number of instances each frame's binning buffer was sized for (the same for every frame).
 *   num_rendered_dev: device uint32[M*2] -> {num_rendered, status} per frame; also copied asynchronously to
 *   num_rendered_host (pinned host uint32[M*2]) if non-NULL.
 * Backward takes the forward's inputs, dL_dout_color / dL_dout_features (strided as out_color / out_features),
 *   dL_dout_others[M*8*H*W] and the three buffers the forward filled.  Outputs (all fully written, no need to zero):
 *   dL_dmeans2D (the densification proxy of backward.cu:645-648; z = 0), dL_dcolors[P*3], dL_dopacity[P],
 *   dL_dmeans3D[P*3], dL_dtransMat[P*9], dL_dsh[P*sh_coeffs*3], dL_dscales[P*2], dL_drotations[P*4], dL_dfeatures[P*F],
 *   each per frame, (M, P, .) -- except, with SR_BATCH_SUM_SHARED, those of shared inputs, which are (P, .) sums over
 *   the frames; dL_dmeans2D and dL_dtransMat are always per frame.  dL_dtransMat (a by-product) may be NULL unless
 *   M == 1 without SR_BATCH_SUM_SHARED.  grad_scale (optional DEVICE scalar, NULL = 1) multiplies dL_dout_color and
 *   dL_dout_others -- the upstream scalar of a fused loss; features_grad_scale (likewise) multiplies dL_dout_features.
 *
 * F = 0 is the plain rasterizer: features NULL, bg_channels 3, and packed colour (out_color_stride / dL_dout_color_stride
 * 0 or 3*H*W).  1 <= F <= 32 composites per-surfel FEATURE channels next to the colour -- the 16+2+3+1-channel vector of
 * lab4d/nnutils/deformable_gaussian.py:1182-1207 (registration feature, flow, normal, Gaussian mask), which the
 * reference rasterizer (NUM_CHANNELS 3) cannot render:
 *   features are independent of where the colour comes from (shs or colors_precomp);
 *   background[bg_channels]: 3 (the feature planes get a zero background) or 3+F (feature plane f gets background[3+f]);
 *   out_color_stride >= 3*H*W, so that colour and features can share one (M, 3+F, H, W) tensor (stride (3+F)*H*W,
 *       features at out_color + 3*H*W); out_features_stride >= F*H*W.
 * Feature plane f = sum_i T_i alpha_i features[i, f] + T_final bg_f over exactly the colour's contributors, weights and
 * FMA order: a feature column equal to a colour column gives a bit-identical plane.  The colour, out_others, radii and
 * the three buffers are those F = 0 writes.  dL_dfeatures is zeroed inside; invisible surfels get 0.  The feature planes'
 * gradient reaches dL_dmeans3D / dL_dscales / dL_drotations / dL_dopacity / dL_dmeans2D through alpha, as the colour
 * planes' does.  The background gets no gradient.
 */
#define SR_BATCH_SUM_SHARED 1u   /* backward: an input shared by the frames (stride 0) gets ONE gradient (P, .), the sum over
                                    the frames, accumulated inside the per-surfel kernel and written once -- instead of
                                    (M, P, .) per-frame gradients the caller would have to reduce */
typedef struct sr_batch {
    int32_t frames;                                   /* M >= 1 */
    uint32_t flags;                                   /* SR_BATCH_* */
    int64_t means3D, shs, colors_precomp, opacities, scales, rotations;   /* floats between consecutive frames; 0 = shared */
} sr_batch;

SR_API int sr_forward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
               const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
               const float* scales, const float* rotations, const float* features, int32_t F, int64_t features_stride,
               const float* viewmatrix, const float* projmatrix, const float* campos,
               float* out_color, int64_t out_color_stride, float* out_features, int64_t out_features_stride,
               float* out_others, int32_t* radii,
               void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
               uint32_t* num_rendered_dev, uint32_t* num_rendered_host, void* stream);

SR_API int sr_backward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                const float* means3D, const float* shs, const float* colors_precomp, const float* scales,
                const float* rotations, const float* features, int32_t F, int64_t features_stride,
                const float* viewmatrix, const float* projmatrix, const float* campos, const int32_t* radii,
                const float* dL_dout_color, int64_t dL_dout_color_stride,
                const float* dL_dout_features, int64_t dL_dout_features_stride,
                const float* dL_dout_others, const float* grad_scale, const float* features_grad_scale,
                void* geom_buffer, void* binning_buffer, void* image_buffer, int64_t capacity,
                float* dL_dmeans2D, float* dL_dcolors, float* dL_dopacity, float* dL_dmeans3D,
                float* dL_dtransMat, float* dL_dsh, float* dL_dscales, float* dL_drotations, float* dL_dfeatures,
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
 * Stage-3 losses on the rasterizer's FEATURE planes (sr_forward with F > 0), forward and gradient, M frames per call.
 * Replaces lab4d/engine/model.py:663-667 (feature reconstruction) and :742-745 (Gaussian-mask consistency) with their
 * masking (:952-967) and reduction (:1000-1012):
 *   feature:        v = ||features[c] - target[c]||_2 over c < Cf, times mask_gt and is_detected[frame]
 *   reg_gauss_mask: v = (features[gauss_mask_channel] - alpha)^2, alpha = allmap plane 1 (no gradient), unmasked
 *   term k = weights[k] * mean of v over the pixels of the WHOLE batch where v > 0 (0 if there is none).
 *   features[M*F*HW]; target[M*Cf*HW] (NULL = no feature term, Cf must then be 0; else 1 <= Cf <= F and mask_gt[M*HW]
 *   is required); is_detected[M] (NULL = 1); allmap[M*8*HW]; gauss_mask_channel in [Cf, F), or -1 = no term;
 *   weights[2] = {feature, reg_gauss_mask} DEVICE floats, read at run time (they may change between graph replays).
 * Writes feature_terms[M*2] = each frame's share of the two weighted terms (their sum over frames is the term),
 * counts[M*2] = each frame's number of pixels with v > 0, and dL_dfeatures[M*F*HW] = the gradient of the sum of the
 * two terms (fully written: 0 on channels no term reads).  Two kernels; no allocation, no host synchronisation.
 */
SR_API int sr_feature_loss_batch(int32_t M, int32_t W, int32_t H, int32_t F, int32_t Cf, int32_t gauss_mask_channel,
                                 const float* features, const float* target, const float* mask_gt, const float* is_detected,
                                 const float* allmap, const float* weights, float* feature_terms, uint32_t* counts,
                                 float* dL_dfeatures, void* stream);

/*
 * Fused bob-skinning warp (SURVEY.md section 8(f) rows N2/N3): canonical surfels -> every frame's camera space.
 * Replaces the PyTorch chain of lab4d/nnutils/deformable_gaussian.py:1395-1434 (forward_warp), :1033-1046
 * (apply_qt_to_gaussian), lab4d/nnutils/warping.py:378-444 (SkinningWarp.forward, forward direction),
 * lab4d/nnutils/skinning.py:89-142 (Gaussian skinning logits), lab4d/utils/geom_utils.py:48-92 (sign-aligned
 * dual-quaternion blend) and the quaternion helper kernels of lab4d/third_party/quaternion/src/quaternion.cu.
 *   xyz[P*3], rot[P*4] (w,x,y,z): canonical surfels;  o2b_q[B*4], o2b_t[B*3]: object->bone transform of the rest pose;
 *   inv_gauss[B*3] = exp(-log_gauss);  delta[P*B] or NULL;  se3_r, se3_d[M*B*4]: per frame and bone dual quaternion
 *   t_articulation o rest_articulation^-1;  cam_q[M*4], cam_t[M*3]: field2cam.   B <= 64.
 * forward writes xyz_cam[M*P*3], rot_cam[M*P*4] (feed them to sr_forward with per-frame strides) and
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
 * Stage 3's feature-matching reprojection loss ("feat_reproj"), in two halves, because the caller's delta-skinning MLP
 * runs on the matched points between them.  See csrc/match.cu and DESIGN.md section 3.5b.
 *
 * sr_global_match_*: replaces lab4d/nnutils/deformable_gaussian.py:1436-1486 (global_match with num_grad = K) without
 * the (M*H*W, C) score matrix.  feat_px[M*H*W*16] pixel features; regist_feat[P*16], xyz[P*3] canonical surfels;
 * cand[C] int32 candidate indices into the M-fold expanded surfels (candidate c is surfel cand[c] mod P; indices outside
 * [0, M*P) are skipped); logsigma[1] DEVICE float (the temperature is exp(logsigma), read at run time).
 * Per pixel: the K highest scores feat_px . regist_feat[cand[c] mod P] (fp32 FMA chain in channel order; among equal
 * scores the lower candidate position c wins), softmax of score * exp(logsigma) over them, and
 * xyz_matched[M*H*W*3] = sum of prob * xyz.  top_idx / top_prob / top_score[M*H*W*K] (candidate position, -1 if none)
 * are for the backward.  The backward takes g_xyz_matched and writes g_regist_feat[P*16], g_xyz[P*3] and g_logsigma[1]
 * (all zeroed inside; duplicate surfels among the candidates sum); g_cand[C*19] is scratch.  feat_px gets no gradient.
 * SR_EINVAL: a NULL required pointer, M, H, W or P < 1, C outside [1, M*P], K outside [1, min(8, C)].
 *
 * sr_reproj_loss_*: replaces lab4d/nnutils/deformable_gaussian.py:1488-1513 (forward_project: forward_warp of the matched
 * points with no rotation, then lab4d/utils/geom_utils.py:17-30 pinhole_projection) and the feat_reproj term of
 * lab4d/engine/model.py:669-672 (||xy_reproj - hxy[..., :2]||), :915,961-967 (times mask and is_detected) and :994-1012
 * (mean over the batch's positive values, / train_res, * feat_reproj_wt).  The warp tables are those of
 * sr_bob_warp_forward (B <= 64); delta[M*H*W*B] or NULL; Kmat[M*9] row-major intrinsics; hxy[M*H*W*hxy_dim]
 * (hxy_dim 2 or 3; the first two are read); mask[M*H*W]; is_detected[M] or NULL (= 1); weight[1] DEVICE float.
 * Forward writes xy_reproj[M*H*W*2], terms[M] (each frame's share of the weighted term), counts[M] (pixels with v > 0),
 * scale[1] = weight / (total count * train_res) (0 if the count is 0) and loss[1] = sum of terms.  Backward takes
 * g_loss[1] (DEVICE float) and scale, and writes g_xyz_matched[M*H*W*3], g_delta[M*H*W*B] (if non-NULL) and
 * g_tables[sr_bob_warp_table_floats(B, M)] in sr_bob_warp_backward's order (zeroed inside).  Kmat and hxy get no gradient.
 * SR_EINVAL: a NULL required pointer, M, H or W < 1, B outside [1, 64], hxy_dim not 2 or 3, train_res <= 0.
 * No call allocates or synchronises with the host.
 */
SR_API int sr_global_match_forward(int32_t M, int32_t H, int32_t W, int32_t P, int32_t C, int32_t K, const float* feat_px,
                                   const float* regist_feat, const float* xyz, const int32_t* cand, const float* logsigma,
                                   float* xyz_matched, int32_t* top_idx, float* top_prob, float* top_score, void* stream);
SR_API int sr_global_match_backward(int32_t M, int32_t H, int32_t W, int32_t P, int32_t C, int32_t K, const float* feat_px,
                                    const float* xyz, const int32_t* cand, const float* logsigma, const int32_t* top_idx,
                                    const float* top_prob, const float* top_score, const float* g_xyz_matched, float* g_cand,
                                    float* g_regist_feat, float* g_xyz, float* g_logsigma, void* stream);
SR_API int sr_reproj_loss_forward(int32_t M, int32_t H, int32_t W, int32_t B, int32_t hxy_dim, float train_res,
                                  const float* xyz_matched, const float* o2b_q, const float* o2b_t, const float* inv_gauss,
                                  const float* delta, const float* se3_r, const float* se3_d, const float* cam_q,
                                  const float* cam_t, const float* Kmat, const float* hxy, const float* mask,
                                  const float* is_detected, const float* weight, float* xy_reproj, float* terms,
                                  uint32_t* counts, float* scale, float* loss, void* stream);
SR_API int sr_reproj_loss_backward(int32_t M, int32_t H, int32_t W, int32_t B, int32_t hxy_dim, const float* xyz_matched,
                                   const float* o2b_q, const float* o2b_t, const float* inv_gauss, const float* delta,
                                   const float* se3_r, const float* se3_d, const float* cam_q, const float* cam_t,
                                   const float* Kmat, const float* hxy, const float* mask, const float* is_detected,
                                   const float* scale, const float* g_loss, float* g_xyz_matched, float* g_delta,
                                   float* g_tables, void* stream);

/*
 * Stage 3's deformation-cycle regulariser with the backward warp's skin-entropy and delta-skin terms (csrc/cycle.cu,
 * DESIGN.md section 3.5c).  Replaces lab4d/nnutils/deformable_gaussian.py:1272-1275,1517-1574 (cycle_loss: :738-764
 * cam_to_field, then lab4d/nnutils/warping.py:378-444 SkinningWarp.forward with backward=True, then apply_qt_to_gaussian
 * and |x_cycled - x|), and lab4d/engine/model.py:850-853 (reg_deform_cyc, reg_delta_skin, reg_skin_entropy) with their
 * :994-1012 reduction (v[v > 0].mean() times the term's weight).
 *   xyz[P*3]: canonical surfels;  xyz_cam[M*P*3]: the same surfels in every frame's camera space (sr_bob_warp_forward's
 *   output);  o2b_q[M*B*4], o2b_t[M*B*3]: object->bone transform of each frame's t_articulation;  inv_gauss[B*3] =
 *   exp(-log_gauss);  delta[M*P*B] or NULL: the frame-conditioned delta skinning term;  se3_r, se3_d[M*B*4]: per frame
 *   and bone dual quaternion rest_articulation o t_articulation^-1;  cam_q[M*4], cam_t[M*3]: field2cam;
 *   weights[3] DEVICE floats {reg_deform_cyc, reg_delta_skin, reg_skin_entropy} read at run time.
 * Per frame m and surfel p: v = {|x_cycled - xyz[p]|, mean_b delta^2 (0 without delta), logsumexp - max of the logits}.
 * Forward writes terms[M*3] (each frame's share of each weighted term), counts[M*3] (values > 0), scale[3] =
 * weights / (total count) (0 where the count is 0) and loss[1] = sum of terms.  Backward takes scale and g_loss[1]
 * (DEVICE float); a value > 0 gets g_loss * scale_k, a value = 0 none.  It writes g_xyz_cam[M*P*3], g_xyz[P*3],
 * g_delta[M*P*B] (if non-NULL) and g_tables[sr_cycle_loss_table_floats(B, M)] = gradients of {o2b_q, o2b_t, inv_gauss,
 * se3_r, se3_d, cam_q, cam_t} in that order (zeroed inside).
 * SR_EINVAL: a NULL required pointer, P < 0, M < 1, B outside [1, 64], tables of (B, M) beyond 200 KB of shared memory
 * (twice sr_cycle_loss_table_floats floats; at B = 64 that is M <= 26), g_delta without delta.
 * No call allocates or synchronises with the host.
 */
SR_API size_t sr_cycle_loss_table_floats(int32_t B, int32_t M);
SR_API int sr_cycle_loss_forward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* xyz_cam, const float* o2b_q,
                                 const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                 const float* se3_d, const float* cam_q, const float* cam_t, const float* weights, float* terms,
                                 uint32_t* counts, float* scale, float* loss, void* stream);
SR_API int sr_cycle_loss_backward(int32_t P, int32_t B, int32_t M, const float* xyz, const float* xyz_cam, const float* o2b_q,
                                  const float* o2b_t, const float* inv_gauss, const float* delta, const float* se3_r,
                                  const float* se3_d, const float* cam_q, const float* cam_t, const float* scale,
                                  const float* g_loss, float* g_xyz_cam, float* g_xyz, float* g_delta, float* g_tables,
                                  void* stream);

/*
 * Stage 3's per-surfel feature rows (csrc/feature_rows.cu, DESIGN.md section 3.5d): the (M,P,Cf+6) rows the rasterizer
 * composites next to the colour.  Replaces lab4d/nnutils/deformable_gaussian.py:1106-1182 (query_field's normal, flow,
 * flow scale and row concatenation), :817-883 (compute_flow with flip_pair), :1742-1769 with lab4d/nnutils/warping.py:463-495
 * and lab4d/utils/transforms.py:28-40 (the Gaussian-bone density), with their autograd.
 *   regist[P*Cf] (may be NULL when Cf = 0; 8-byte alignment suffices);  xyz[P*3]: canonical surfels;  scaling[P*2]: the
 *   two tangent scales;  xyz_cam[M*P*3], rot_cam[M*P*4]: sr_bob_warp_forward's outputs;  Kmat[M*9]: intrinsics (all
 *   three rows used);  cam_q[M*4]: field2cam's quaternion;  centres[B*3]: translations of the rest bones;  beta[1] =
 *   exp(logibeta).  All DEVICE float32.
 * Row (m, p) = [regist[p] | flow[m,p] / s | normal[m,p] | density[p]], with
 *   flow[m,p] = pi(K[m'], xyz_cam[m',p]) - pi(K[m], xyz_cam[m,p]), pi(K,x) = (Kx)[0:2] / (Kx)[2], m' = m xor 1 (M = 1:
 *   m' = m, flow 0);  s = max |flow| over all M*P*2 values + 1e-6 (= max(max(flow), |min(flow)|) + 1e-6);
 *   normal = cam_q[m] (rot_cam[m,p] e_a rot_cam[m,p]*) cam_q[m]*, e_a = e_x or e_y, the arg-min of the two scales (e_x on
 *   ties), quaternions not normalised;  density = beta * max_b exp(-0.5 |xyz - centres[b]|^2 / 0.01^2).
 * Forward writes rows[M*P*(Cf+6)], density[P], flow_scale[1] = s and aux[3] (uint32: the bits of max |flow|, the number
 * of flow values equal to +max|flow| and to -max|flow|; keep it for the backward).  Rows are bit-identical run to run.
 * Backward takes g_rows[M*P*(Cf+6)], g_density[P] or NULL and g_flow_scale[1] (DEVICE) or NULL.  dL/ds (the caller's
 * g_flow_scale plus the rows' -sum(g * flow) / s^2) reaches the tied extreme flow values as torch's autograd sends it:
 * halved when both +max|flow| and -max|flow| occur, then spread evenly over the equal elements, times -1 for the
 * minimum's.  It writes g_regist[P*Cf], g_xyz[P*3], g_xyz_cam[M*P*3], g_rot_cam[M*P*4] directly and g_tables[M*4 + B*3 + 2]
 * = gradients of {cam_q, centres, beta} in that order, then one float of scratch (zeroed inside).
 * SR_EINVAL, before any device work: a NULL required pointer (the per-surfel arrays may be NULL when P = 0), P < 0, M not
 * 1 and not even or above 1024, B outside [1, 64], Cf < 0 or Cf + 6 > 32.  No call allocates or synchronises with the host.
 */
SR_API int sr_feature_rows_forward(int32_t P, int32_t M, int32_t B, int32_t Cf, const float* regist, const float* xyz,
                                   const float* scaling, const float* xyz_cam, const float* rot_cam, const float* Kmat,
                                   const float* cam_q, const float* centres, const float* beta, float* rows, float* density,
                                   float* flow_scale, uint32_t* aux, void* stream);
SR_API int sr_feature_rows_backward(int32_t P, int32_t M, int32_t B, int32_t Cf, const float* xyz, const float* scaling,
                                    const float* xyz_cam, const float* rot_cam, const float* Kmat, const float* cam_q,
                                    const float* centres, const float* beta, const float* flow_scale, const uint32_t* aux,
                                    const float* g_rows, const float* g_density, const float* g_flow_scale, float* g_regist,
                                    float* g_xyz, float* g_xyz_cam, float* g_rot_cam, float* g_tables, void* stream);

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

/*
 * Radius outlier filter (csrc/outlier.cu, DESIGN.md section 3.9): Stage 3's periodic
 * `pcd.remove_radius_outlier(nb_points=20, radius=0.004)` (lab4d/engine/trainer.py:573-588) on the device.
 *   count_i = #{ j in [0,P) : d2(i,j) < r2 }, j = i included, with
 *   d2 = ((xi-xj)^2 + (yi-yj)^2) + (zi-zj)^2: coordinates widened to float64, every difference, product and sum rounded
 *   on its own (no FMA contraction), and r2 = radius * radius in float64.
 *   keep[i] = count_i > nb_points (1 / 0); counts[i] (nullable) = min(count_i, nb_points + 1).
 * A point with a NaN or Inf coordinate is nobody's neighbour, not even its own: it is never kept and changes no other
 * count.  nb_points = 0 keeps every finite point.  This is Open3D's RemoveRadiusOutliers as we understand it (a KD-tree
 * radius search with a strict < on the squared distance, the query point counted, kept iff the count exceeds nb_points);
 * it was not checked against Open3D itself.  The two can differ only on pairs at distance exactly `radius`.
 * points[P*3] (DEVICE float32), keep[P], counts[P]; scratch: DEVICE, at least sr_radius_outlier_scratch_bytes(P) bytes,
 * which depends on P alone.  Counts are integers, so the result is bit-identical run to run and independent of the
 * order of the points.  No allocation, no host synchronisation: the call can be captured in a CUDA graph.
 * SR_EINVAL, before any device work: P < 0, nb_points < 0, radius not finite or <= 0, scratch_bytes below the size
 * query, a NULL points / keep / scratch.  P = 0 does nothing.
 */
SR_API int64_t sr_radius_outlier_scratch_bytes(int32_t P);
SR_API int sr_radius_outlier_mask(int32_t P, const float* points, double radius, int32_t nb_points, uint8_t* keep,
                                  int32_t* counts, void* scratch, int64_t scratch_bytes, void* stream);

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
