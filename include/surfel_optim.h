/*
 * surfel_optim.h -- C ABI of the optimizer step whose per-step state lives on the device: gradient-norm clipping over
 * the flat surfel gradient buffer, an Adam pass that reads its step count, learning rates and clip coefficient from
 * device memory, and the batched densification statistics.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer; sr_adam_flat there takes its step count and rates as launch arguments, which a CUDA graph
 * freezes at capture.
 *
 * The flat buffer holds n_groups parameter groups back to back: group g is elements [begin[g], begin[g+1]), with
 * begin a HOST int64 array of n_groups + 1 entries, begin[0] = 0, non-decreasing, 1 <= n_groups <= 8.  Groups may start
 * at any element offset; the buffers themselves are 16-byte aligned.
 *
 * Together the two calls do what torch.nn.utils.clip_grad_norm_(params, max_norm) followed by torch.optim.Adam.step()
 * does (lab4d/engine/trainer.py:547, 589-591):
 *   S_g   = sum over group g of (grads * grad_scale)^2, in float64, per CTA and group, then a fixed-order one-CTA sum;
 *   total = (float) sqrt(S_0 + ... + S_{n-1} + n_0^2 + ... + n_{e-1}^2), the n_i the fp32 norms of other gradients;
 *   coef  = min((1 / (total + 1e-6f)) * max_norm, 1) in fp32, NaN passing through, as torch evaluates it;
 *   Adam on (grads * grad_scale) * coef with bias corrections of the device step count.
 * The launch shapes depend on the buffer size only, so equal inputs give equal bits on every device and stream.
 * Neither call allocates memory or synchronises with the host, so both can be captured in a CUDA graph.
 * Every function returns 0 on success or a negative SR_E* code; bad arguments return SR_EINVAL before any device work.
 */
#ifndef SURFEL_OPTIM_H_
#define SURFEL_OPTIM_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* bytes of DEVICE scratch sr_grad_norm_flat needs for n_groups groups, whatever their size (-1: bad n_groups) */
SR_API int64_t sr_grad_norm_scratch_bytes(int32_t n_groups);

/*
 * total_norm[1], clip_coef[1]: DEVICE float, written.  group_sumsq (nullable): DEVICE double [n_groups], gets S_g.
 * extra_norms: DEVICE float [n_extra] (n_extra >= 0; NULL allowed when 0).  scratch: DEVICE, at least
 * sr_grad_norm_scratch_bytes(n_groups) bytes, 8-byte aligned.
 */
SR_API int sr_grad_norm_flat(int32_t n_groups, const int64_t* begin, const float* grads, float grad_scale,
                             const float* extra_norms, int32_t n_extra, float max_norm, float* total_norm, float* clip_coef,
                             double* group_sumsq, void* scratch, int64_t scratch_bytes, void* stream);

/*
 * One Adam step (torch.optim.Adam: amsgrad off, weight_decay 0) over params / exp_avg / exp_avg_sq, DEVICE float.
 * lr: DEVICE float [n_groups].  step: DEVICE int64, incremented first; the step runs with t = the new value, the step
 * size (float)(lr / (1 - pow(beta1, t))) and the bias correction (float)sqrt(1 - pow(beta2, t)) evaluated in double from
 * the double betas, as sr_adam_flat does on the host and torch.optim.Adam does in Python.  clip_coef: DEVICE float, or
 * NULL for 1.  The step count advances also when the buffer is empty.
 */
SR_API int sr_adam_flat_state(int32_t n_groups, const int64_t* begin, const float* lr, double beta1, double beta2, float eps,
                              int64_t* step, float grad_scale, const float* clip_coef, float* params, const float* grads,
                              float* exp_avg, float* exp_avg_sq, void* stream);

/*
 * Densification statistics of a batch of M frames (gaussian_model.py add_densification_stats, trainer.py:553-560).
 * viewspace_grad: DEVICE float (M,P,3), the screen-space proxy gradient of the batched backward.  radii: DEVICE int32
 * (M,P); frame m sees surfel i iff radii[m,i] > 0.  accum, denom, max_radii: DEVICE float [P], updated in place: for
 * m = 0 .. M-1 in order, where frame m sees surfel i,
 *   accum[i] += ||grad_scale * viewspace_grad[m,i]||,  denom[i] += 1,  max_radii[i] = max(max_radii[i], radii[m,i]),
 * each step rounded to float as torch's per-frame update rounds it (the norm: fl(fl(fl(x^2) + fl(z^2)) + fl(y^2)),
 * then a correctly rounded sqrt).  One thread per surfel, no atomics: equal inputs give equal bits.  M = 0 or P = 0
 * launches nothing.  Arrays 4-byte aligned.
 */
SR_API int sr_densify_stats(int32_t M, int32_t P, const float* viewspace_grad, const int32_t* radii, float grad_scale,
                            float* accum, float* denom, float* max_radii, void* stream);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_OPTIM_H_ */
