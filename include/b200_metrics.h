/*
 * b200_metrics.h -- C ABI of the evaluation metric kernels (part of libb200ps.so, csrc/eval_metrics.cu).
 *
 * Replaces the per-update work of tf.keras.metrics.AUC (ROC curve, the default thresholds) that the reference's
 * master runs on the outputs its workers report (elasticdl/python/common/evaluation_utils.py:68-77): Keras
 * compares every prediction with every threshold ([T, n] booleans) and reduces four confusion counts.  Here one
 * launch adds every prediction to a histogram over the threshold buckets; the confusion counts follow from its
 * suffix sums where the result is read (common/evaluation_utils.py):
 *   tp[i] = sum_{k > i} hist[1][k],  fp[i] = sum_{k > i} hist[0][k],  fn[i] = P - tp[i],  tn[i] = N - fp[i].
 *
 * Bucket k of a prediction p is the number of thresholds t with t < p (fp32 comparisons against the exact
 * threshold values), so bucket k > i iff p > thresholds[i], bit for bit Keras' `predictions > thresholds`.
 * A label is positive iff it is non-zero (Keras casts y_true to bool).  A prediction that is NaN, below 0 or above
 * 1 (Keras asserts on these) is not bucketed: it is added to *invalid.
 *
 * State: hist is uint64 [2][T + 1] (row 0 negatives, row 1 positives) and invalid uint64 [1], added to with 64-bit
 * atomics and never reset by the kernel, so several callers (streams, engines) may add to one state.
 *
 * The launch reads nothing back to the host and allocates nothing, so it can be captured in a CUDA graph.
 */
#ifndef B200_METRICS_H_
#define B200_METRICS_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_METRICS_MIN_THRESHOLDS 2
#define B200_METRICS_MAX_THRESHOLDS 16384 /* the thresholds and one histogram copy fit in a CTA's shared memory */
#define B200_METRICS_THREADS 256          /* threads per CTA */
#define B200_METRICS_MIN_PER_CTA 2048     /* the grid has at most ceil(n / 2048) CTAs */

/* Adds predictions probs [n] with labels [n] (fp32, device) to the AUC state hist [2][T + 1] / invalid [1], for the
 * ascending fp32 thresholds [T] (device).  n = 0 launches nothing.
 * Returns 0, or -1 (B200PS_EINVAL) for a null buffer, n outside [0, 2^31) or T outside
 * [B200_METRICS_MIN_THRESHOLDS, B200_METRICS_MAX_THRESHOLDS], -2 for a CUDA error. */
int b200_metrics_auc_update(const float* probs, const float* labels, int64_t n, const float* thresholds, int32_t T,
                            uint64_t* hist, uint64_t* invalid, void* stream);
const char* b200_metrics_last_error(void);
int64_t b200_metrics_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_METRICS_H_ */
