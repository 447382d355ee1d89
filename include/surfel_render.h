/*
 * surfel_render.h -- forward-only rendering of many frames: a trained sequence rendered for viewing or evaluation.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer, whose prototypes stay as they are.
 *
 * sr_forward keeps, per frame, what its backward reads: the per-surfel gradient accumulator, the per-(stage, pixel)
 * contribution masks, final_T, n_contrib and each sub-tile's deepest contributor; with F > 0 feature channels a second
 * pass re-walks the recorded contributors.  sr_render_forward writes the same outputs, bit for bit, keeps none of that
 * state, and composites the F feature channels inside the colour's walk.  Its scratch is one arena per frame, smaller
 * than sr_forward's three buffers by exactly those arrays.
 */
#ifndef SURFEL_RENDER_H_
#define SURFEL_RENDER_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bytes of one frame's forward-only arena: sr_geom_bytes(P) + sr_binning_bytes(capacity, W, H) + sr_image_bytes(W, H)
 * less the arrays only a backward reads (the geometry's gradient accumulator, the binning's contribution masks, the
 * image's final_T, n_contrib and sub_last).  An M-frame call takes M of them, consecutively. */
SR_API size_t sr_render_bytes(int32_t P, int64_t capacity, int32_t width, int32_t height);

/* sr_forward's arguments and outputs (an sr_frame, or an sr_frame_cameras of surfel_camera.h; an sr_batch with per-input
 * strides; F in 0..32 with a background of 3 or 3+F values), with one arena of M * sr_render_bytes(P, capacity, W, H)
 * bytes, 16-byte aligned, instead of the three scratch buffers.  Colour, out_others, the feature planes and radii are
 * bit-identical to sr_forward's.  capacity, num_rendered_dev / num_rendered_host and the SR_STATUS_* words mean what
 * they mean for sr_forward: an overflowed frame is not rendered, and the caller re-runs it with a larger capacity.
 * P = 0 zero-fills the colour, feature and out_others planes.  Nothing is kept for a backward. */
SR_API int sr_render_forward(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                             const float* means3D, const float* shs, const float* colors_precomp, const float* opacities,
                             const float* scales, const float* rotations, const float* features, int32_t F,
                             int64_t features_stride, const float* viewmatrix, const float* projmatrix, const float* campos,
                             float* out_color, int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                             float* out_others, int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev,
                             uint32_t* num_rendered_host, void* stream);

/* Per-surfel contribution statistics, DEVICE arrays of P words each.  A pair (frame, pixel, surfel) contributes when the
 * composite blends it; its weight is w = T * alpha rounded once to float32 (the feature plane of a feature equal to 1),
 * and its quantised weight q(w) = round-to-nearest-even(w * 2^32), an integer below 2^32.  Over the contributing pairs:
 *   weight_q[s]    sum of q(w)                        (unsigned 64-bit)
 *   max_weight[s]  max of w, as its float32 bits      (non-negative floats order as unsigned integers)
 *   pixels[s]      number of pairs                    (unsigned 64-bit)
 * All three are integer sums or maxima: exact, and independent of the order in which pairs, frames or calls add. */
typedef struct sr_contrib {
    uint64_t* weight_q;
    uint32_t* max_weight;
    uint64_t* pixels;
} sr_contrib;

/* sr_render_forward, which it is in every argument, output and check, that also ADDS every rendered frame's contributing
 * pairs into `contrib` (never cleared here).  An overflowed frame is not composited and adds nothing: re-running it
 * alone with a larger capacity adds it once (re-running a whole call would add its other frames twice).  With P > 0 the
 * three pointers must be non-NULL, weight_q and pixels 8-byte aligned, max_weight 4-byte aligned.  contrib = NULL is
 * sr_render_forward: the same kernels and bits. */
SR_API int sr_render_forward_contrib(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                                     const float* means3D, const float* shs, const float* colors_precomp,
                                     const float* opacities, const float* scales, const float* rotations,
                                     const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
                                     const float* projmatrix, const float* campos, float* out_color,
                                     int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                                     float* out_others, int32_t* radii, void* arena, int64_t capacity,
                                     uint32_t* num_rendered_dev, uint32_t* num_rendered_host, const sr_contrib* contrib,
                                     void* stream);

/* Foreground masks and the per-surfel share of the contribution statistics that lands on background pixels.
 *   mask         DEVICE bytes: frame m's H*W pixels, row-major, at mask + m * mask_stride; nonzero = foreground
 *   mask_stride  bytes between consecutive frames' masks, >= H*W
 *   weight_bg_q  DEVICE [P] (unsigned 64-bit): sum of q(w) over the contributing pairs on background pixels
 *   pixels_bg    DEVICE [P] (unsigned 64-bit): the number of those pairs
 * Integer sums, like sr_contrib's: exact and independent of the order of pairs, frames or calls. */
typedef struct sr_contrib_mask {
    const uint8_t* mask;
    int64_t mask_stride;
    uint64_t* weight_bg_q;
    uint64_t* pixels_bg;
} sr_contrib_mask;

/* sr_render_forward_contrib, which it is in every argument, output and check, that also ADDS every rendered frame's
 * contributing pairs on background pixels into mask->weight_bg_q and mask->pixels_bg (never cleared here).  contrib's
 * three words get exactly the bits sr_render_forward_contrib gives, and so do the rendered outputs.  An overflowed frame
 * adds nothing.  mask = NULL, or mask->mask = NULL, is sr_render_forward_contrib: the same kernels and bits.  Otherwise
 * contrib must be non-NULL, mask_stride >= H*W and, with P > 0, weight_bg_q and pixels_bg non-NULL and 8-byte aligned. */
SR_API int sr_render_forward_contrib_masked(const sr_frame* f, const sr_batch* b, const float* background,
                                            int32_t bg_channels, const float* means3D, const float* shs,
                                            const float* colors_precomp, const float* opacities, const float* scales,
                                            const float* rotations, const float* features, int32_t F,
                                            int64_t features_stride, const float* viewmatrix, const float* projmatrix,
                                            const float* campos, float* out_color, int64_t out_color_stride,
                                            float* out_features, int64_t out_features_stride, float* out_others,
                                            int32_t* radii, void* arena, int64_t capacity, uint32_t* num_rendered_dev,
                                            uint32_t* num_rendered_host, const sr_contrib* contrib,
                                            const sr_contrib_mask* mask, void* stream);

/* Per-pixel maps lifted onto the surfels: each surfel's blending-weighted sum of C caller-supplied channels.
 *   values         DEVICE floats: frame m's (C, H, W) planes, row-major, at values + m * values_stride
 *   C              channels, 1..32
 *   values_stride  floats between consecutive frames' values, >= C*H*W
 *   scale_log2     s, in SR_LIFT_SCALE_MIN..SR_LIFT_SCALE_MAX.  A caller whose values stay within |v| <= B picks
 *                  s = 32 - ceil(log2 B) once and keeps it for every call that adds into the same sums
 *   sums           DEVICE [P * C] (signed 64-bit, row-major (P, C)): over the contributing pairs of surfel i,
 *                  sums[i*C + c] += q,  q = round-to-nearest-even(fl(w * v) * 2^s),  fl(w * v) the float32 product of
 *                  sr_contrib's weight w and the pixel's value v of channel c.  |q| <= 2^32 when |v| <= 2^(32-s).
 *   saturated      DEVICE [1] (unsigned 64-bit): the number of (pair, channel) terms that were not exact -- a non-finite
 *                  value, which contributes 0, or |fl(w * v) * 2^s| > 2^32, which contributes +-2^32.
 * Two's-complement integer sums: exact, and independent of the order of pairs, frames, calls or ranks.  With v = 1 and
 * s = 32, q is sr_contrib's q(w). */
#define SR_LIFT_MAX_CHANNELS 32
#define SR_LIFT_SCALE_MIN (-64)
#define SR_LIFT_SCALE_MAX 64
typedef struct sr_lift {
    const float* values;
    int32_t C;
    int64_t values_stride;
    int32_t scale_log2;
    int64_t* sums;
    uint64_t* saturated;
} sr_lift;

/* sr_render_forward_contrib, which it is in every argument, output and check, that also ADDS every rendered frame's
 * lifted values into lift->sums and lift->saturated (never cleared here).  contrib's three words and the rendered
 * outputs get exactly the bits sr_render_forward_contrib gives.  An overflowed frame adds nothing.  lift = NULL is
 * sr_render_forward_contrib: the same kernels and bits.  Otherwise contrib must be non-NULL, F must be 0 (a lift is a
 * colour-only walk), C in 1..32, values_stride >= C*H*W, scale_log2 in range and, with P > 0, values non-NULL and 4-byte
 * aligned, sums and saturated non-NULL and 8-byte aligned. */
SR_API int sr_render_forward_lift(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                                  const float* means3D, const float* shs, const float* colors_precomp,
                                  const float* opacities, const float* scales, const float* rotations,
                                  const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
                                  const float* projmatrix, const float* campos, float* out_color, int64_t out_color_stride,
                                  float* out_features, int64_t out_features_stride, float* out_others, int32_t* radii,
                                  void* arena, int64_t capacity, uint32_t* num_rendered_dev, uint32_t* num_rendered_host,
                                  const sr_contrib* contrib, const sr_lift* lift, void* stream);

/* Each pixel's K heaviest contributing pairs, its anchors on the surfels.
 *   K        slots per pixel: 1, 2, 4 or 8
 *   stride   elements between consecutive frames of ids and weights, >= K*H*W; uv's frames are 2*stride apart
 *   ids      DEVICE (frame, K, H, W) int32: the pair's surfel, -1 for an empty slot
 *   weights  DEVICE (frame, K, H, W): the pair's w, sr_contrib's weight, 0 for an empty slot
 *   uv       DEVICE (frame, K, 2, H, W): where the pixel's ray hits the surfel's disc, in its scaled tangent frame: the
 *            surface point is mean + u*s_u*t_u + v*s_v*t_v, t_u and t_v the first two columns of the rotation and
 *            s the scale, as the forward builds its homography.  A pair on the screen-space filter branch (its rho2d
 *            below its rho3d, where the depth is the centre's) stores (0, 0), the centre.  (0, 0) for an empty slot.
 * The slots are sorted by w, descending.  A pair enters only if its w is strictly larger than the last slot's, so among
 * equal weights the earlier pair of the front-to-back walk stays ahead: the result is deterministic. */
#define SR_ANCHORS_MAX 8
typedef struct sr_anchors {
    int32_t K;
    int64_t stride;
    int32_t* ids;
    float* weights;
    float* uv;
} sr_anchors;

/* sr_render_forward, which it is in every argument, output and check, that also WRITES every rendered frame's anchors
 * (overwritten, never added into); the rendered outputs get exactly the bits sr_render_forward gives.  An overflowed
 * frame writes no anchors: the caller re-runs it with a larger capacity.  P = 0 writes empty slots.  anchors must be
 * non-NULL, K in {1, 2, 4, 8}, F must be 0 (anchors are a colour-only walk), stride >= K*H*W, and ids, weights and uv
 * non-NULL and 4-byte aligned. */
SR_API int sr_render_forward_anchors(const sr_frame* f, const sr_batch* b, const float* background, int32_t bg_channels,
                                     const float* means3D, const float* shs, const float* colors_precomp,
                                     const float* opacities, const float* scales, const float* rotations,
                                     const float* features, int32_t F, int64_t features_stride, const float* viewmatrix,
                                     const float* projmatrix, const float* campos, float* out_color,
                                     int64_t out_color_stride, float* out_features, int64_t out_features_stride,
                                     float* out_others, int32_t* radii, void* arena, int64_t capacity,
                                     uint32_t* num_rendered_dev, uint32_t* num_rendered_host, const sr_anchors* anchors,
                                     void* stream);

/* sr_post_forward over M frames in one launch: frame m's allmap (allmap + m*8*H*W) and world_view_transform (+ m*16) give
 * its acc, rend_normal, rend_dist, depth_median, depth_expected, surf_depth, surf_normal (each output packed (M, c, H, W)).
 * cameras: optional DEVICE (M,4) table of surfel_camera.h; with it frame m's rays use its own tangents and principal
 * point offsets (tan_fovx / tan_fovy are not read), as sr_render_loss_batch_cameras does.  Without it every frame uses
 * tan_fovx / tan_fovy and the centred principal point, bit-identical to sr_post_forward frame by frame.
 * learnable_bkgd: optional DEVICE [3]; with it frame m's colour planes color + m*color_stride (color_stride >= 3*H*W
 * floats) become color + (1 - acc) * bkgd, three rounded operations, in place.  Without it color is not read. */
SR_API int sr_post_forward_frames(int32_t M, int32_t W, int32_t H, float tan_fovx, float tan_fovy, const float* cameras,
                                  float depth_ratio, const float* allmap, const float* world_view_transform,
                                  const float* learnable_bkgd, float* color, int64_t color_stride, float* acc,
                                  float* rend_normal, float* rend_dist, float* depth_median, float* depth_expected,
                                  float* surf_depth, float* surf_normal, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_RENDER_H_ */
