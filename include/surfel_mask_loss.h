/*
 * surfel_mask_loss.h -- C ABI of Stage 3's fused silhouette (mask) loss and its gradient.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer; adding the loss here leaves that ABI (and SR_ABI_VERSION) untouched.
 *
 * Computes the reference's mask term as lab4d/engine/model.py weighs it (field_type "fg"):
 *   vd       = vis2d * is_detected[frame]                                            get_mask_balance_wt (:587-611)
 *   pos_wt   = sum(vd) / sum(mask[vd > 0]),   neg_wt = sum(vd) / sum(1 - mask[vd > 0])     fp32 sums, fp32 division
 *   bw       = 0.5 pos_wt mask + 0.5 neg_wt (1 - mask)  if sum(mask) > 0 and sum(1 - mask) > 0,  else 1
 *   v        = (acc - mask)^2 * bw * vis2d * is_detected[frame]                      :648-650, mask_losses :950-967
 *   loss     = w * mean(v[v > 0]) over the whole batch, or w * mean(v) if no v is > 0   apply_loss_weights :1000-1012
 * with acc the rendered alpha.  The degenerate cases are the reference's: an all-zero or all-one mask gives bw = 1; no
 * mask pixel inside vd (or no detected frame) gives pos_wt = inf (NaN), and then a NaN loss and gradient.
 *
 * Layouts (all DEVICE float32): alpha and dL_dalpha: frame m's H x W plane at alpha + m * alpha_stride (floats, >= H*W),
 * e.g. plane 1 of an (M,8,H,W) allmap with alpha_stride = 8*H*W; mask_gt and vis2d [M][H][W] contiguous;
 * is_detected [M]; weight [1] (read at run time, so a captured call follows in-place updates).
 * Limits: 1 <= M <= 65535, 1 <= W, 1 <= H <= 524280.
 *
 * Results are bit-identical from run to run: every sum is a per-CTA partial reduced in a fixed order in float64, with no
 * float atomics.  No call allocates memory or synchronises with the host, so each can be captured in a CUDA graph.
 * Every function returns 0 on success or a negative SR_E* code; bad arguments return SR_EINVAL before any device work.
 */
#ifndef SURFEL_MASK_LOSS_H_
#define SURFEL_MASK_LOSS_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bytes of DEVICE scratch sr_mask_loss_batch needs for M frames of W x H pixels (-1: bad shape); about 5 bytes per
 * pixel plus 40 bytes per 32 x 8 tile */
SR_API int64_t sr_mask_loss_scratch_bytes(int32_t M, int32_t W, int32_t H);

/*
 * vis2d and is_detected may be NULL (all ones).
 * terms [M]: each frame's share of the weighted loss (they sum to the loss); counts [M]: each frame's number of v > 0.
 * balance [3]: pos_wt, neg_wt and 1.0f / 0.0f for the branch (bw = 1 when 0; the weights are written either way).
 * dL_dalpha: scale * dv/dacc is ADDED, with scale = w / C (C = the batch's count of v > 0; only pixels with v > 0
 * receive gradient) or w / (M*H*W) when C = 0.
 * scratch: DEVICE, at least sr_mask_loss_scratch_bytes(M, W, H) bytes, 256-byte aligned.
 */
SR_API int sr_mask_loss_batch(int32_t M, int32_t W, int32_t H, const float* alpha, int64_t alpha_stride,
                              const float* mask_gt, const float* vis2d, const float* is_detected, const float* weight,
                              float* terms, int32_t* counts, float* balance, float* dL_dalpha, void* scratch,
                              int64_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_MASK_LOSS_H_ */
