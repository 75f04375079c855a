/*
 * b200_deepctr_deepfm.h -- C ABI of the deepctr DeepFM estimator tower (csrc/deepctr_deepfm_tower.cu): deepctr's
 * DeepFMEstimator(linear, dnn, task="binary") of model_zoo/deepctr/deepfm_estimator.py on Criteo-shaped rows, one
 * training step from hashed ids to the loss and the complete dense gradient of all 73 parameters.
 *
 * Inputs: ids [26, B] (categorical_column_with_hash_bucket(C<j>, 1000) of C1..C26, int32; -1 = an empty cell, which
 * the column drops), dense [13, B] (I1..I13, float32, raw), labels [B].
 *   e_j = E_j[id_j], or 0 for an absent id (embedding_column, combiner 'mean' over the ids that remain)
 *   x = [e_1 .. e_26 | I1 .. I13]                               (F = 117: 104 sparse columns, then 13 dense)
 *   h1 = relu(x W0 + b0) [256], h2 = relu(h1 W1 + b1) [128], h3 = relu(h2 W2 + b2) [64]
 *   linear = sum_j L_j[id_j] (present ids) + I w_num + bias_weights, the columns in name order (C1, C10, .., I9)
 *   fm = 1/2 sum_d ((sum_j e_jd)^2 - sum_j e_jd^2)
 *   z = linear + fm + h3 wd
 *   loss = sum_b (max(z, 0) - z y + log1p(exp(-|z|)))
 *          + 1e-5/2 (sum_b sum_j |e_bj|^2 + sum_j |L_j|^2 + |w_num|^2)    (bias_weights unregularised)
 *
 * Flat parameters (201,438 floats; names recalled from TF1, see workloads/deepctr_deepfm.py), the dnn group first:
 *   C<j> embedding [1000, 4] @ 4000 (j - 1)                    j = 1 .. 26
 *   dnn kernel0 [117, 256] @ 104000, bias0 [256] @ 133952, kernel1 [256, 128] @ 134208, bias1 [128] @ 166976,
 *   kernel2 [128, 64] @ 167104, bias2 [64] @ 175296, logit kernel [64, 1] @ 175360,
 *   then the linear group: C<j> weights [1000, 1] @ 175424 + 1000 (j - 1), I<i> weights [1, 1] @ 201424 + (i - 1),
 *   bias_weights [1] @ 201437.
 * grads has the same layout.  An embedding row gets the sum over its occurrences of (dx + 1e-5 e), so a row no
 * sample read gets exactly 0; a linear row gets 1e-5 w + its occurrences' dz; I<i> weights 1e-5 w + sum I dz;
 * bias_weights sum dz.
 *
 * The three hidden layers' forward, data-gradient and weight-gradient contractions run as 3xTF32 on mma.sync
 * (csrc/mma_tf32.cuh) with fp32 accumulation.  No float atomics: every sum is taken in a fixed order, so two
 * launches on one device give the same bits.  No host read; the workspace needs no zeroing between calls, so a
 * captured graph replays.  Every pointer is a device pointer; `stream` is a cudaStream_t passed as void*.
 * Return 0 = ok, -1 = a refused argument, -2 = a CUDA error; message via b200_deepctr_deepfm_last_error().
 */
#ifndef B200_DEEPCTR_DEEPFM_H_
#define B200_DEEPCTR_DEEPFM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_DEEPCTR_DEEPFM_FIELDS 26      /* C1 .. C26 */
#define B200_DEEPCTR_DEEPFM_DENSE 13       /* I1 .. I13 */
#define B200_DEEPCTR_DEEPFM_ROWS 1000      /* hash buckets of every column */
#define B200_DEEPCTR_DEEPFM_DIM 4          /* embedding width */
#define B200_DEEPCTR_DEEPFM_PARAMS 201438  /* floats of the flat parameters */
#define B200_DEEPCTR_DEEPFM_DNN_FLOATS 175424 /* floats of the dnn group, the first part of the flat buffer */
#define B200_DEEPCTR_DEEPFM_TILE 64        /* samples per tile of the tower */
#define B200_DEEPCTR_DEEPFM_MAX_B 4194304  /* largest batch */

typedef struct {
  int64_t B;             /* batch size, in [1, B200_DEEPCTR_DEEPFM_MAX_B] */
  const int32_t* ids;    /* [26, B]; -1 is absent; an id outside [-1, 1000) is read as absent and counted in *error */
  const float* dense;    /* [13, B] */
  const float* labels;   /* [B]; unused by the forward */
  const float* params;   /* [201438], 16-byte aligned */
  float* loss;           /* [1]; unused by the forward */
  float* logits;         /* [B] z, before the sigmoid */
  float* grads;          /* [201438], 16-byte aligned; unused by the forward */
  int32_t* error;        /* [1] count of ids outside [-1, 1000) (added to, never cleared) */
  void* workspace;       /* b200_deepctr_deepfm_workspace_bytes(B) bytes, 256-byte aligned; unused by the forward */
  size_t workspace_bytes;
} b200_deepctr_deepfm_args_t;

/* Workspace bytes of a training call at batch B on the current device; 0 for a refused B. */
size_t b200_deepctr_deepfm_workspace_bytes(int64_t B);
/* One training step: the loss, the logits and the complete gradient (five launches). */
int b200_deepctr_deepfm_tower(const b200_deepctr_deepfm_args_t* args, void* stream);
/* The forward alone: logits and the id error count (one launch). */
int b200_deepctr_deepfm_forward(const b200_deepctr_deepfm_args_t* args, void* stream);
const char* b200_deepctr_deepfm_last_error(void);
int64_t b200_deepctr_deepfm_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_DEEPCTR_DEEPFM_H_ */
