/*
 * b200_census.h -- C ABI of the census wide & deep tower (part of libb200ps.so, csrc/census_tower.cu).
 *
 * Replaces, for the census wide & deep model of BASELINE.json configs[2], what the reference runs in
 * TensorFlow between the pull and the push of one minibatch (paths relative to /root/reference/):
 *   - the pooled Embedding lookups           model_zoo/census_wide_deep_model/wide_deep_functional_api.py:164-195
 *   - wide_deep (Dense 24 -> 16 -> 8 -> 4,   wide_deep_functional_api.py:198-212
 *     no activation, reduce_sum)
 *   - the mean sigmoid cross-entropy         wide_deep_functional_api.py:48-55
 *   - tape.gradient and the per-row sums of  elasticdl/python/worker/ps_trainer.py:391-400,
 *     the IndexedSlices the PS applies        elasticdl/python/common/tensor_utils.py:39-60
 * in one launch, with the touched rows of every table compacted into the segments b200ps_push_rows takes.
 *
 * Inputs: ids int32 [12, B] as census_transform writes them: rows 4g .. 4g+3 are the four ids of group g
 * (g = 0, 1, 2 with 28, 75, 115 rows).  An id outside [0, rows of its group) is added to *error and read
 * as row 0.
 *
 * Flat parameter buffer (floats; Keras layouts: a Dense kernel is [in, out] row-major):
 *   MLP   [ dense/kernel 24x16 @0 | dense/bias 16 @384 | dense_1/kernel 16x8 @400 | dense_1/bias 8 @528 |
 *           dense_2/kernel 8x4 @536 | dense_2/bias 4 @568 ]                                     572 floats
 *   wide  [ embedding [28,1] @572 | embedding_1 [75,1] @600 ]                                   103 floats
 *   deep  [ embedding_2 [28,8] @675 | embedding_3 [75,8] @899 | embedding_4 [115,8] @1499 ]   1744 floats
 * grads [572] is the MLP block's gradient in the same order.
 *
 * Tables t = 0..4 are embedding .. embedding_4 (wide group 1, wide group 2, deep groups 1, 2, 3).  Table t
 * gets the b200ps_push_rows segment (uniq + B200_CENSUS_UNIQ_OFF[t], n_unique + t, gsum + B200_CENSUS_GSUM_OFF[t]):
 * its touched rows in ascending order, their count, and row i's gradient [dim] -- a row that occurs in the
 * batch is listed even when its gradient is zero.  The gsum offsets are the tables' parameter offsets minus 572.
 *
 * reference_reshape = 0: the DNN input of sample b is [e_1(b) | e_2(b) | e_3(b)] (e_g = the sum of group g's
 * four deep rows).  reference_reshape = 1: quirk Q11 -- tf.reshape of the list [e_1, e_2, e_3] stacks it to
 * [3, B, 8], so slot k of row r is e_g(s) with g * B + s = 3r + k (DESIGN.md).  The wide part is per sample
 * in both modes.
 *
 * Summation order is fixed and there are no float atomics: two calls on the same inputs give the same bits.
 */
#ifndef B200_CENSUS_H_
#define B200_CENSUS_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_CENSUS_PARAMS 2419
#define B200_CENSUS_MLP 572
#define B200_CENSUS_UNIQ_ROWS 321   /* 28 + 75 + 28 + 75 + 115 */
#define B200_CENSUS_GSUM_FLOATS 1847 /* 28 + 75 + (28 + 75 + 115) x 8 */
#define B200_CENSUS_TILE 256         /* samples per tile */
/* uniq row offsets of tables 0..4: 0, 28, 103, 131, 206; gsum float offsets: 0, 28, 103, 327, 927 */

typedef struct {
  int32_t B;                 /* batch size, >= 1 */
  int32_t reference_reshape; /* 0 or 1 (see above) */
  const int32_t* ids;        /* [12, B] */
  const float* labels;       /* [B] */
  const float* params;       /* [2419] */
  float* loss;               /* [1] mean sigmoid cross-entropy */
  float* logits;             /* [B] */
  float* grads;              /* [572] */
  int64_t* uniq;             /* [321] */
  int32_t* n_unique;         /* [5] */
  float* gsum;               /* [1847] */
  int32_t* error;            /* [1] out-of-range ids are added to it (never reset by the kernel) */
  void* workspace;           /* b200_census_workspace_bytes(B) bytes, zero before the first call; every call
                              * leaves its arrival counter at zero again, so a captured graph can replay */
  size_t workspace_bytes;
} b200_census_args_t;

/* Workspace bytes for batch B on the current device (one partial per CTA of the persistent grid). */
size_t b200_census_workspace_bytes(int64_t B);
/* One launch: forward, loss, backward, the MLP gradients and the five push_rows segments.
 * Returns 0, or -1 (B200PS_EINVAL) for a bad argument / too small a workspace, -2 for a CUDA error. */
int b200_census_tower(const b200_census_args_t* args, void* stream);
const char* b200_census_last_error(void);
int64_t b200_census_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_CENSUS_H_ */
