/*
 * surfel_track.h -- dense point tracking through a rendered sequence: a pixel of one frame, anchored on the surfels it
 * blends (sr_render_forward_anchors, surfel_render.h), followed into every other frame as those surfels move.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path; its own header because surfel_raster.h is the drop-in boundary of the reference
 * rasterizer, whose prototypes stay as they are.
 */
#ifndef SURFEL_TRACK_H_
#define SURFEL_TRACK_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* For every query n and target frame t:
 *
 *   X = sum_k w_k (mean_t + u_k s_u t_u,t + v_k s_v t_v,t) / sum_k w_k
 *
 * over the query's non-empty anchor slots k (id >= 0): w_k, (u_k, v_k) and the surfel id_k from the anchors of the
 * query's frame at its pixel; mean_t, the rotation's first two columns t_u,t and t_v,t, and the scale s of surfel id_k in
 * frame t, as the forward preprocess builds them.  X is projected through frame t's view and intrinsics (the forward's:
 * tan_fovx / tan_fovy and the centred principal point, or row t of `cameras`) into the rasterizer's continuous pixel
 * coordinates, where pixel (x, y) is centred at (x + 0.5, y + 0.5).
 *
 *   N           queries; T target frames; S anchor frames; P surfels; K anchor slots (1, 2, 4 or 8); image W x H
 *   queries     DEVICE (N, 3) int32: (anchor frame, x, y)
 *   anchor_ids, anchor_weights   DEVICE (S, K, H, W) at + s*anchor_stride elements
 *   anchor_uv   DEVICE (S, K, 2, H, W) at + 2*s*anchor_stride elements
 *   anchor_stride  >= K*H*W
 *   means3D     DEVICE (T, P, 3) at + t*means3D_stride floats (0: one (P, 3) array for every frame)
 *   scales      DEVICE (P, 2), shared by every frame
 *   rotations   DEVICE (T, P, 4) at + t*rotations_stride floats (0: shared), 16-byte aligned
 *   viewmatrix  DEVICE (T, 16): each frame's world_view_transform
 *   cameras     optional DEVICE (T, 4) table of surfel_camera.h; with it tan_fovx / tan_fovy are not read
 *   depth       optional DEVICE (T, H, W): e.g. render()'s surf_depth of each target frame
 * Outputs (overwritten):
 *   xy          DEVICE (N, T, 2): the projected point
 *   z           DEVICE (N, T): its view depth
 *   visible     DEVICE (N, T) bytes: 1 when z >= 0.2, 0 <= x < W, 0 <= y < H and, with depth,
 *               |z - depth[t, floor(y), floor(x)]| <= depth_tolerance * z
 *   coverage    DEVICE (N): sum_k w_k, to compare with the pixel's accumulated alpha
 * A query with no anchored surfel, an anchor frame or pixel out of range, or an id >= P gets coverage 0, NaN for xy and
 * z and visible 0, for every target; the kernel reads nothing out of bounds and the host does not synchronise.
 * Grid: queries in the caller's order on x, the target frame on y; N = 0 or T = 0 launches nothing. */
SR_API int sr_track_pixels(int32_t N, int32_t T, int32_t S, int32_t P, int32_t K, int32_t width, int32_t height,
                           const int32_t* queries, const int32_t* anchor_ids, const float* anchor_weights,
                           const float* anchor_uv, int64_t anchor_stride, const float* means3D, int64_t means3D_stride,
                           const float* scales, const float* rotations, int64_t rotations_stride,
                           const float* viewmatrix, float tan_fovx, float tan_fovy, const float* cameras,
                           const float* depth, float depth_tolerance, float* xy, float* z, uint8_t* visible,
                           float* coverage, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_TRACK_H_ */
