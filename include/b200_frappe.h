/*
 * b200_frappe.h -- C ABI of the frappe DeepFM tower (part of libb200ps.so, csrc/frappe_tower.cu).
 *
 * Replaces, for the frappe DeepFM model the reference's own tests train, what the reference runs in TensorFlow
 * between the pull and the push of one minibatch (paths relative to the reference tree):
 *   - the masked Embedding lookups (dim 64 and 1)  model_zoo/deepfm_edl_embedding/deepfm_edl_embedding.py:24-49
 *   - the FM, Flatten, Dense(64) and Dense(1)       deepfm_edl_embedding.py:50-70
 *     (no activation), logit = first + second + deep
 *   - the mean sigmoid cross-entropy                deepfm_edl_embedding.py:76-84
 *   - tape.gradient and the per-row sums of the     elasticdl/python/worker/ps_trainer.py:391-400
 *     IndexedSlices the PS applies
 * (model_zoo/deepfm_functional_api/deepfm_functional_api.py:40-101 is the same model with bounded ids.)
 *
 * Inputs: ids int64 [B, 10] (F = 10 fields, sample-major); id 0 is the pad.  The mask is m_bf = (id_bf != 0):
 * a masked occurrence contributes nothing to the forward and exactly zero to every gradient.  inv int32 [10 B]
 * and n_unique int32 [1] are the dedup's (b200ps_unique over the 10 B ids in sample-major order: position
 * b * 10 + f); bet_deep [U, 64] / bet_wide [U, 1] are the rows of the dedup's unique ids, pulled from
 * embedding/embeddings:0 (dim 64) and embedding_1/embeddings:0 (dim 1).
 *
 * Flat dense buffer (floats; Keras layouts: a Dense kernel is [in, out] row-major), 41089 floats:
 *   [ dense/kernel [640, 64] @0 | dense/bias [64] @40960 | dense_1/kernel [64, 1] @41024 | dense_1/bias [1] @41088 ]
 * grads [41089] is its gradient in the same order.  The Dense(64) input is Flatten(e_b), f-major:
 * x[f * 64 + d] = m_bf E[id_bf][d].
 *
 * Outputs of b200_frappe_tower: loss (the mean), logits [B], grads [41089], and gsum_deep [U, 64] /
 * gsum_wide [U, 1] aligned with the dedup's unique ids -- the two b200ps_push_rows segments.  Rows [0, n_unique)
 * are overwritten; a row that occurs only masked (id 0 always) gets exactly 0.
 *
 * The Dense stack is linear: with v = K w2 [640] and c = b . w2 + b2 the deep term is x . v + c, a row's
 * gradient per occurrence is m_bf g_b (S_b - e_bf + v_f) with g_b = (sigmoid(z_b) - y_b) / B and S_b = sum_f e_bf,
 * and the dense gradients follow from s = sum_b g_b x_b and G = sum_b g_b (DESIGN.md section 7b).
 *
 * Determinism: NOT bit-deterministic.  The per-row sums, s, G and the loss are accumulated with fp32 atomic adds
 * to global memory (after combining equal rows inside a warp), so two calls agree within the fp32 rounding of
 * those sums, not bit for bit.  The logits are computed per sample in a fixed order and are reproducible.
 *
 * Each call is two launches on `stream`: a prologue (v, c, and zeroing the n_unique rows of gsum) and the main
 * pass; the last CTA of the main pass writes the dense gradients and the loss and leaves the workspace's
 * accumulators and arrival counter at zero, so a captured CUDA graph can replay.
 */
#ifndef B200_FRAPPE_H_
#define B200_FRAPPE_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_FRAPPE_FIELDS 10
#define B200_FRAPPE_DIM 64
#define B200_FRAPPE_PARAMS 41089 /* 640 x 64 + 64 + 64 + 1 */
#define B200_FRAPPE_TILE 64      /* samples per CTA tile */

typedef struct {
  int32_t B;                 /* batch size, >= 1 */
  int32_t pad_;
  const int64_t* ids;        /* [B, 10] */
  const int32_t* inv;        /* [10 B] */
  const int32_t* n_unique;   /* [1] */
  const float* bet_deep;     /* [>= n_unique, 64], 16-byte aligned */
  const float* bet_wide;     /* [>= n_unique] */
  const float* labels;       /* [B] (not read by b200_frappe_forward) */
  const float* params;       /* [41089] */
  float* loss;               /* [1] */
  float* logits;             /* [B] */
  float* grads;              /* [41089] */
  float* gsum_deep;          /* [>= n_unique, 64], 16-byte aligned */
  float* gsum_wide;          /* [>= n_unique] */
  void* workspace;           /* b200_frappe_workspace_bytes(B) bytes, zero before the first call */
  size_t workspace_bytes;
} b200_frappe_args_t;

/* Workspace bytes for batch B (accumulators, v, c and the arrival counter). */
size_t b200_frappe_workspace_bytes(int64_t B);
/* Forward, loss, backward, the dense gradients and the two push_rows segments.
 * Returns 0, or -1 (B200PS_EINVAL) for a bad argument / too small a workspace, -2 for a CUDA error. */
int b200_frappe_tower(const b200_frappe_args_t* args, void* stream);
/* Forward only: logits [B] (labels, loss, grads and gsum are not touched). */
int b200_frappe_forward(const b200_frappe_args_t* args, void* stream);
const char* b200_frappe_last_error(void);
int64_t b200_frappe_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_FRAPPE_H_ */
