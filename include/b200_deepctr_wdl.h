/*
 * b200_deepctr_wdl.h -- C ABI of the deepctr WDL tower (csrc/deepctr_wdl_tower.cu): deepctr's premade
 * WDL(fixlen, fixlen, task="binary") of model_zoo/deepctr/wdl.py:19-75 on Criteo-shaped rows, one training step
 * from hashed ids to the loss and the complete dense gradient of all 61 parameters.
 *
 * Inputs: ids [26, B] (Hash(10000) of C1..C26, int32), dense [13, B] (I1..I13, float32, raw), labels [B].
 *   x = [E_1[id_1] .. E_26[id_26] | I1 .. I13]                    (F = 117: 104 sparse columns, then 13 dense)
 *   h1 = relu(x W0 + b0) [256], h2 = relu(h1 W1 + b1) [128], h3 = relu(h2 W2 + b2) [64]
 *   z = h3 wd + sum_j L_j[id_j] + I w_lin + global_bias,  p = sigmoid(z)
 *   loss = mean_b Keras-clipped BCE(y, p) + 1e-5 (sum_j |E_j|^2 + sum_j |L_j|^2 + |w_lin|^2) over whole tables
 *
 * Flat parameters (1,371,438 floats; names recalled from deepctr, see workloads/deepctr_wdl.py):
 *   sparse_emb_C<j> [10000, 4] @ 40000 (j - 1)            j = 1 .. 26
 *   linear0sparse_emb_C<j> [10000, 1] @ 1040000 + 10000 (j - 1)
 *   linear/linear_kernel [13, 1] @ 1300000, dnn/kernel0 [117, 256] @ 1300013, dnn/bias0 [256] @ 1329965,
 *   dnn/kernel1 [256, 128] @ 1330221, dnn/bias1 [128] @ 1362989, dnn/kernel2 [128, 64] @ 1363117,
 *   dnn/bias2 [64] @ 1371309, dense/kernel [64, 1] @ 1371373, prediction_layer/global_bias [1] @ 1371437.
 * grads has the same layout.  Every table row gets 2e-5 W + the sum of the batch's occurrences of the row: the
 * regularizer makes each table's gradient dense (DESIGN.md section 4, Q28).
 *
 * The three hidden layers' forward, data-gradient and weight-gradient contractions run as 3xTF32 on mma.sync
 * (csrc/mma_tf32.cuh) with fp32 accumulation.  No float atomics: every sum is taken in a fixed order, so two
 * launches on one device give the same bits.  No host read; the workspace needs no zeroing between calls, so a
 * captured graph replays.  Every pointer is a device pointer; `stream` is a cudaStream_t passed as void*.
 * Return 0 = ok, -1 = a refused argument, -2 = a CUDA error; message via b200_deepctr_wdl_last_error().
 */
#ifndef B200_DEEPCTR_WDL_H_
#define B200_DEEPCTR_WDL_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_DEEPCTR_WDL_FIELDS 26      /* C1 .. C26 */
#define B200_DEEPCTR_WDL_DENSE 13       /* I1 .. I13 */
#define B200_DEEPCTR_WDL_ROWS 10000     /* hash buckets of every table */
#define B200_DEEPCTR_WDL_DIM 4          /* deep embedding width */
#define B200_DEEPCTR_WDL_PARAMS 1371438 /* floats of the flat parameters */
#define B200_DEEPCTR_WDL_TILE 64        /* samples per tile of the tower */
#define B200_DEEPCTR_WDL_MAX_B 4194304  /* largest batch */

typedef struct {
  int64_t B;             /* batch size, in [1, B200_DEEPCTR_WDL_MAX_B] */
  const int32_t* ids;    /* [26, B]; an id outside [0, 10000) is read as row 0 and counted in *error */
  const float* dense;    /* [13, B] */
  const float* labels;   /* [B]; unused by the forward */
  const float* params;   /* [1371438], 16-byte aligned */
  float* loss;           /* [1]; unused by the forward */
  float* logits;         /* [B] z, before the sigmoid */
  float* grads;          /* [1371438]; unused by the forward */
  int32_t* error;        /* [1] count of ids read as row 0 (added to, never cleared) */
  void* workspace;       /* b200_deepctr_wdl_workspace_bytes(B) bytes; unused by the forward */
  size_t workspace_bytes;
} b200_deepctr_wdl_args_t;

/* Workspace bytes of a training call at batch B on the current device; 0 for a refused B. */
size_t b200_deepctr_wdl_workspace_bytes(int64_t B);
/* One training step: the loss, the logits and the complete gradient (five launches). */
int b200_deepctr_wdl_tower(const b200_deepctr_wdl_args_t* args, void* stream);
/* The forward alone: logits and the id error count (one launch). */
int b200_deepctr_wdl_forward(const b200_deepctr_wdl_args_t* args, void* stream);
const char* b200_deepctr_wdl_last_error(void);
int64_t b200_deepctr_wdl_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_DEEPCTR_WDL_H_ */
