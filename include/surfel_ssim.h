/*
 * surfel_ssim.h -- C ABI of the fused SSIM (structural similarity) loss and its gradient.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer (RAST); SSIM is a loss on images, not part of that boundary, and adding it here leaves the
 * rasterizer's ABI (and SR_ABI_VERSION) untouched.
 *
 * Computes the reference's  ssim(img1, img2)  (gs/utils/loss_utils.py:33-68): per (image, channel) plane of H x W
 * pixels, the 11x11 Gaussian window (sigma 1.5, built as the reference builds it: float32 exp of the double,
 * normalised by the float32 sum) applied separably with zero padding to x, y, x^2, y^2 and xy;
 *   m = (2 mu1 mu2 + C1)(2 s12 + C2) / ((mu1^2 + mu2^2 + C1)(s11 + s22 + C2) + 1e-10),   C1 = 0.01^2, C2 = 0.03^2,
 * with s11 = E[x^2] - mu1^2, s22 = E[y^2] - mu2^2, s12 = E[xy] - mu1 mu2.  x is img1, y is img2.
 *
 * Layout: img1, img2 are DEVICE float32 [N][C][H][W], contiguous.  Any N, C, H, W >= 1 (also smaller than the window).
 *
 * Compositing option (alpha != NULL): the image x is then  img1 + (1 - alpha) * bkgd[channel],  as csrc/loss.cu
 * composites the learnable background: alpha is one H x W plane per image, image n's at alpha + n * alpha_stride
 * (floats, >= H*W), and bkgd is a DEVICE float[3]; C must be 3.
 *
 * Results are bit-identical from run to run: per-CTA partial sums are reduced in a fixed order, with no float atomics.
 * No call allocates memory or synchronises with the host, so each can be captured in a CUDA graph.
 * Every function returns 0 on success or a negative SR_E* code; bad arguments return SR_EINVAL before any device work.
 */
#ifndef SURFEL_SSIM_H_
#define SURFEL_SSIM_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bytes of DEVICE scratch sr_ssim_forward / sr_ssim_backward need for N images of C x H x W (-1: bad shape) */
SR_API int64_t sr_ssim_scratch_bytes(int32_t N, int32_t C, int32_t H, int32_t W);

/*
 * ssim_img[N]: each image's mean of m over C*H*W; ssim_mean[1]: the mean over N*C*H*W.
 * maps (nullable): DEVICE float [3][N*C][H][W], written when a gradient will be wanted -- per pixel
 *   A = dm/dmu1 - 2 mu1 dm/ds11 - mu2 dm/ds12,   B = dm/ds11,   Cm = dm/ds12.
 * scratch: DEVICE, at least sr_ssim_scratch_bytes(N, C, H, W) bytes.
 */
SR_API int sr_ssim_forward(int32_t N, int32_t C, int32_t H, int32_t W, const float* img1, const float* img2,
                           const float* alpha, int64_t alpha_stride, const float* bkgd, float* ssim_img, float* ssim_mean,
                           float* maps, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * dL/dx(q) = g * [ (w*A)(q) + 2 x(q) (w*B)(q) + y(q) (w*Cm)(q) ], the maps filtered with zero outside the image.
 * dL_dssim: DEVICE; per_image = 0: dL_dssim[0] is dL/d ssim_mean and g = dL_dssim[0] / (N*C*H*W);
 *           per_image = 1: dL_dssim[n] is dL/d ssim_img[n] and g = dL_dssim[n] / (C*H*W).
 * dL_dimg1 [N][C][H][W]: overwritten (accumulate = 0) or added to (accumulate = 1).
 * With alpha: dL_dalpha (plane n at dL_dalpha + n * alpha_stride) gets -sum_ch dL/dx * bkgd[ch] added, and
 * dL_dbkgd [N][3] gets each image's sum over pixels of dL/dx * (1 - alpha) added (both required, both added to).
 */
SR_API int sr_ssim_backward(int32_t N, int32_t C, int32_t H, int32_t W, const float* img1, const float* img2,
                            const float* alpha, int64_t alpha_stride, const float* bkgd, const float* maps,
                            const float* dL_dssim, int32_t per_image, float* dL_dimg1, int32_t accumulate, float* dL_dalpha,
                            float* dL_dbkgd, void* scratch, int64_t scratch_bytes, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_SSIM_H_ */
