/*
 * b200_census_sqlflow.h -- C ABI of the census_model_sqlflow wide & deep tower (part of libb200ps.so,
 * csrc/census_sqlflow_tower.cu).
 *
 * Replaces, for model_zoo/census_model_sqlflow/wide_and_deep/ (paths relative to the ElasticDL tree), what the
 * reference runs in TensorFlow between the pull and the push of one minibatch:
 *   - the mean-pooled sparse lookups        SparseEmbedding(combiner="mean") over the ToSparse-pruned ids
 *                                           (wide_deep_functional_keras.py:207-227, layers/sparse_embedding.py),
 *                                           or embedding_column's mean combiner (wide_deep_functional_fc.py:237-255)
 *   - Dense 24 -> 16 -> 8 -> 4, no          wide_deep_functional_keras.py:60-73
 *     activation, reduce_sum with the wide part
 *   - the mean sigmoid cross-entropy        wide_deep_functional_keras.py:253-260
 *   - tape.gradient and the per-row sums of the IndexedSlices the PS applies
 * in one launch, with the touched rows of every table compacted into the segments b200ps_push_rows takes.
 *
 * Inputs: ids int32 [12, B]: rows 4g .. 4g+3 are the four features of group g (g = 0, 1, 2 with 27, 73, 113
 * rows), -1 = absent (ToSparse dropped the cell, or a feature-column id was pruned).  An id outside [-1, rows of
 * its group) is added to *error and read as absent.
 *
 * Pooling: e_g(b) = the mean of the rows of group g's present ids of sample b (an id present twice counts
 * twice); a group with no present id gives a zero vector and no row gradient.  Wide: w_g(b) likewise, dim 1.
 *
 * Flat parameter buffer (floats; Keras layouts: a Dense kernel is [in, out] row-major):
 *   MLP   [ dense/kernel 24x16 @0 | dense/bias 16 @384 | dense_1/kernel 16x8 @400 | dense_1/bias 8 @528 |
 *           dense_2/kernel 8x4 @536 | dense_2/bias 4 @568 ]                                       572 floats
 *   wide  [ group 1 [27,1] @572 | group 2 [73,1] @599 ]                                            100 floats
 *   deep  [ group 1 [27,8] @672 | group 2 [73,8] @888 | group 3 [113,8] @1472 ]                   1704 floats
 * grads [572] is the MLP block's gradient in the same order.
 *
 * Tables t = 0..4 are wide group 1, wide group 2, deep groups 1, 2, 3.  Table t gets the b200ps_push_rows
 * segment (uniq + UNIQ_OFF[t], n_unique + t, gsum + GSUM_OFF[t]): its touched rows (present in the batch) in
 * ascending order, their count, and row i's gradient [dim] -- a touched row is listed even when its gradient is
 * zero.  UNIQ_OFF = 0, 27, 100, 127, 200; GSUM_OFF = 0, 27, 100, 316, 900 (the parameter offsets minus 572).
 *
 * reference_reshape = 0: the DNN input of sample b is [e_1(b) | e_2(b) | e_3(b)].  reference_reshape = 1: quirk
 * Q11 -- tf.reshape of the list [e_1, e_2, e_3] stacks it to [3, B, 8], so slot k of row r is e_g(s) with
 * g * B + s = 3r + k (DESIGN.md).  The wide part is per sample in both modes.
 *
 * Summation order is fixed and there are no float atomics: two calls on the same inputs give the same bits.
 */
#ifndef B200_CENSUS_SQLFLOW_H_
#define B200_CENSUS_SQLFLOW_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_CSQL_PARAMS 2376
#define B200_CSQL_MLP 572
#define B200_CSQL_UNIQ_ROWS 313    /* 27 + 73 + 27 + 73 + 113 */
#define B200_CSQL_GSUM_FLOATS 1804 /* 27 + 73 + (27 + 73 + 113) x 8 */
#define B200_CSQL_TILE 256         /* samples per tile */

typedef struct {
  int32_t B;                 /* batch size, >= 1 */
  int32_t reference_reshape; /* 0 or 1 (see above) */
  const int32_t* ids;        /* [12, B] */
  const float* labels;       /* [B]; unused by the forward */
  const float* params;       /* [2376] */
  float* loss;               /* [1] mean sigmoid cross-entropy */
  float* logits;             /* [B] */
  float* grads;              /* [572] */
  int64_t* uniq;             /* [313] */
  int32_t* n_unique;         /* [5] */
  float* gsum;               /* [1804] */
  int32_t* error;            /* [1] out-of-range ids are added to it (never reset by the kernel) */
  void* workspace;           /* b200_csql_workspace_bytes(B) bytes, zero before the first call; every call leaves
                              * its arrival counter at zero again, so a captured graph can replay */
  size_t workspace_bytes;
} b200_csql_args_t;

/* Workspace bytes for batch B on the current device (one partial per CTA of the persistent grid). */
size_t b200_csql_workspace_bytes(int64_t B);
/* One launch: forward, loss, backward, the MLP gradients and the five push_rows segments.
 * Returns 0, or -1 for a bad argument / too small a workspace, -2 for a CUDA error. */
int b200_csql_tower(const b200_csql_args_t* args, void* stream);
/* The forward alone: logits (and *error); labels, loss, grads, uniq, n_unique, gsum and the workspace are unused
 * and may be NULL. */
int b200_csql_forward(const b200_csql_args_t* args, void* stream);
const char* b200_csql_last_error(void);
int64_t b200_csql_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_CENSUS_SQLFLOW_H_ */
