/*
 * surfel_camera.h -- per-frame intrinsics for the batched rasterizer and the fused Stage-3 loss pass.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer, whose prototypes stay as they are.
 *
 * Without it every frame of a batch shares one field of view (sr_frame.tan_fovx / tan_fovy, host floats) and the
 * principal point is the image centre (W/2, H/2), as in the reference.  Stage 3 learns a focal length per frame and
 * projects with a full K elsewhere, so a batch needs each frame's own intrinsics, read from device memory: a captured
 * step then renders with whatever the table holds at replay.
 *
 * The table: cameras[M*4], DEVICE float32, frame m's row = (tan_fovx, tan_fovy, cx_off, cy_off).
 *   tan_fov*:  what sr_frame.tan_fov* means (tan of half the field of view);
 *   c*_off:    the principal point minus (W/2, H/2), in pixels.
 * For a pinhole K = [[fx, 0, cx], [0, fy, cy], [0, 0, 1]]: tan_fovx = W / (2 fx), tan_fovy = H / (2 fy),
 * cx_off = cx - W/2, cy_off = cy - H/2.
 * Each kernel derives frame m's intrinsics from its row with the scalar path's own operations and adds the offsets, so a
 * row holding the scalar tangents and zero offsets gives bit-identical results.  The rows are read as four scalar loads
 * (float alignment suffices).  Their values are not checked on the device: a non-finite or non-positive tangent gives
 * what the same scalar would give.  Nothing computes a gradient with respect to the table.
 */
#ifndef SURFEL_CAMERA_H_
#define SURFEL_CAMERA_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bit of sr_frame.flags.  When set, the sr_frame passed to sr_forward / sr_backward is the `frame` member of an
 * sr_frame_cameras, and every frame of the batch reads its intrinsics from `cameras`; tan_fovx / tan_fovy of the
 * sr_frame are not read.  The bit set with cameras == NULL is SR_EINVAL, before any device work. */
#define SR_FRAME_CAMERAS 1u

typedef struct sr_frame_cameras {
    sr_frame frame;           /* frame.flags has SR_FRAME_CAMERAS set */
    const float* cameras;     /* DEVICE [M*4], M = sr_batch.frames */
} sr_frame_cameras;

/* sr_render_loss_batch with frame m's intrinsics read from cameras[m*4 .. m*4+3] (DEVICE) instead of the shared
 * tan_fovx / tan_fovy: the ray grid of depth_to_normal uses fx = W / (2 tan_fovx), cx = W/2 + cx_off (likewise y).
 * The same kernels as sr_render_loss_batch; SR_EINVAL for a NULL cameras, with its other checks. */
SR_API int sr_render_loss_batch_cameras(int32_t M, int32_t W, int32_t H, const float* cameras, float depth_ratio,
                                        const float* color, const float* allmap, const float* world_view_transform,
                                        const float* target_rgb, const float* vis2d, const float* mask_gt,
                                        const float* mask_wt, const float* learnable_bkgd, float w_rgb, float w_mask,
                                        float lambda_normal, float lambda_dist, float* loss_terms, float* dL_dcolor,
                                        float* dL_dallmap, float* dL_dbkgd, float* surf_depth_scratch, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_CAMERA_H_ */
