/*
 * surfel_deterministic.h -- a bit-reproducible rasterizer backward.
 *
 * The same library as surfel_raster.h (libsurfel_raster.so), the same SR_API visibility, SR_E* codes and
 * sr_last_error() message path.  It lives in its own header because surfel_raster.h is the drop-in boundary of the
 * reference rasterizer, whose prototypes stay as they are.
 *
 * By default sr_backward sends each (instance, tile)'s colour-gradient sum and every feature pair's gradient to the
 * per-surfel accumulators with float atomics, so the order of the adds -- and the last bits of every gradient -- depend
 * on scheduling.  With SR_BATCH_DETERMINISTIC no float atomic touches a gradient: each (instance, tile) writes its sum
 * into its own slot of a caller-provided scratch, indexed by the instance's emission index, and one thread per surfel
 * sums its slots in emission order, then the frames in order for inputs the batch shares.  Every sum then has an order
 * fixed by the data (frame, surfel, tile in emission order, pixel), so two calls on the same inputs give the same bits,
 * and each frame of a batch gives the bits a one-frame call on that frame gives.
 */
#ifndef SURFEL_DETERMINISTIC_H_
#define SURFEL_DETERMINISTIC_H_

#include "surfel_raster.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Bit of sr_batch.flags.  When set, the sr_batch passed to sr_backward is the `batch` member of an sr_batch_det, and the
 * backward runs deterministically in `scratch`.  sr_forward ignores the bit (its outputs are deterministic already).
 * A NULL scratch, or scratch_bytes below sr_backward_det_bytes(capacity, F) * frames, is SR_EINVAL before any device
 * work. */
#define SR_BATCH_DETERMINISTIC 2u

typedef struct sr_batch_det {
    sr_batch batch;           /* batch.flags has SR_BATCH_DETERMINISTIC set */
    void* scratch;            /* DEVICE, 16-byte aligned, at least scratch_bytes */
    int64_t scratch_bytes;
} sr_batch_det;

/* Scratch one frame of a deterministic backward needs: one 80-byte slot per instance of `capacity` (the binning
 * buffer's), and F floats per instance for the feature gradients. */
SR_API size_t sr_backward_det_bytes(int64_t capacity, int32_t F);

#ifdef __cplusplus
}
#endif

#endif /* SURFEL_DETERMINISTIC_H_ */
