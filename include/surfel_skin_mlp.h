/*
 * surfel_skin_mlp.h -- C ABI of the fused delta-skinning MLP and its gradient.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer; adding the MLP here leaves that ABI (and SR_ABI_VERSION) untouched.
 *
 * Computes the reference's delta skinning term (lab4d/nnutils/skinning.py:104-119):
 *   delta = relu(delta_field([xyz_bone | t_embed | inst_code])) * 0.1,
 * delta_field = CondMLP(D = 2, W = 64) (lab4d/nnutils/base.py:65-78,123-150), i.e. Linear -> ReLU -> Linear -> ReLU ->
 * Linear, and xyz_bone (skinning.py:126-142) affine in the point.  The conditioning channels are constant per frame and
 * xyz_bone is affine in x, so the caller folds the first Linear, the bones, the Gaussian scales and the conditioning
 * vector into one (64,4) table per frame:  h1 = relu(F_m [x; 1]).  Per point x of frame m:
 *   h1[j] = relu(F_m[j][3] + F_m[j][0] x0 + F_m[j][1] x1 + F_m[j][2] x2)
 *   h2[j] = relu(b2[j] + sum_k W2[j][k] h1[k])          k ascending
 *   y[b]  =      b3[b] + sum_k W3[b][k] h2[k]
 *   delta[b] = 0.1f * relu(y[b])
 * in FP32 fused multiply-adds (no tensor cores, no TF32).
 *
 * Layouts (all DEVICE float32, contiguous): points [M][N][3]; F [Mt][64][4] with Mt = 1 (one table for every frame) or
 * Mt = M; W2 [64][64], b2 [64], W3 [B][64], b3 [B] (torch.nn.Linear's weight layout); delta, g_delta [M][N][B].
 * Limits: width = 64 hidden units, depth = 2 hidden layers, 1 <= B <= 64, 1 <= M <= 65535, M * N < 2^31.
 *
 * Results are bit-identical from run to run: the weight gradients are per-CTA partial sums reduced in a fixed order,
 * with no float atomics.  No call allocates memory or synchronises with the host, so each can be captured in a CUDA
 * graph.  Every function returns 0 on success or a negative SR_E* code; bad arguments return SR_EINVAL before any
 * device work.
 */
#ifndef SURFEL_SKIN_MLP_H_
#define SURFEL_SKIN_MLP_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bytes of DEVICE scratch sr_delta_skin_backward needs for M frames of N points and B bones, for either Mt
 * (-1: bad shape) */
SR_API int64_t sr_delta_skin_scratch_bytes(int32_t M, int32_t N, int32_t B);

/* delta [M][N][B] is overwritten. */
SR_API int sr_delta_skin_forward(int32_t M, int32_t N, int32_t B, int32_t Mt, int32_t width, int32_t depth,
                                 const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                                 const float* b3, float* delta, void* stream);

/*
 * Recomputes h1, h2 and y from the points (nothing but the inputs is saved), then
 *   g_y  = 0.1f g_delta [y > 0],   g_h2 = W3^T g_y [h2 > 0],   g_h1 = W2^T g_h2 [h1 > 0],
 *   g_points = F_m[:, 0:3]^T g_h1                                                  [M][N][3]
 *   g_W3 = sum g_y (x) h2  [B][64],   g_b3 = sum g_y  [B],   g_W2 = sum g_h2 (x) h1  [64][64],   g_b2 = sum g_h2  [64],
 *   g_F[m] = sum over frame m's points (every point when Mt = 1) of g_h1 (x) [x; 1]  [Mt][64][4].
 * All seven outputs are overwritten.  scratch: DEVICE, at least sr_delta_skin_scratch_bytes(M, N, B) bytes, 16-byte
 * aligned.
 */
SR_API int sr_delta_skin_backward(int32_t M, int32_t N, int32_t B, int32_t Mt, int32_t width, int32_t depth,
                                  const float* points, const float* F, const float* W2, const float* b2, const float* W3,
                                  const float* b3, const float* g_delta, float* g_points, float* g_F, float* g_W2,
                                  float* g_b2, float* g_W3, float* g_b3, void* scratch, int64_t scratch_bytes,
                                  void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_SKIN_MLP_H_ */
