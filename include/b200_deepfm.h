/*
 * b200_deepfm.h -- C ABI of the fused DeepFM tower (part of libb200ps.so).
 *
 * Replaces, for the dac_ctr DeepFM workload of BASELINE.json configs[1], what the
 * reference runs in TensorFlow between the pull and the push of one minibatch
 * (paths relative to /root/reference/):
 *   - tf.gather(batch_embedding, idx)      elasticdl/python/elasticdl/embedding_delegate.py:95
 *   - model.call                           model_zoo/dac_ctr/deepfm_model.py:61-109 (DNN[16,4], FM, linear)
 *   - tape.gradient(loss, vars + BETs)     elasticdl/python/worker/ps_trainer.py:391-400
 *   - the sum of deduplicate_indexed_slices elasticdl/python/common/tensor_utils.py:39-60
 *     (the per-occurrence embedding gradients are reduced per unique id on the fly)
 * in two launches that read every embedding row twice (L2) and write every
 * per-unique-id gradient once.
 *
 * Fixed architecture (dac_ctr): 13 dense features, deep dim 8, DNN 16 -> 4 -> 1,
 * G id groups (38 for dac_ctr), one id per group per sample.
 * Parameter / gradient layout (floats), all torch.nn.Linear layouts:
 *   [ w_dense 13 (+3 pad) | w1 16 x (13 + 8G) | b1 16 | w2 4 x 16 | b2 4 | w3 4 ]
 */
#ifndef B200_DEEPFM_H_
#define B200_DEEPFM_H_
#include <stddef.h>
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

#define B200_DEEPFM_NDENSE 13
#define B200_DEEPFM_DIM 8
#define B200_DEEPFM_H1 16
#define B200_DEEPFM_H2 4
#define B200_DEEPFM_SCRATCH 44 /* floats of per-sample backward state */
#define B200_DEEPFM_TILE_MAXG 38 /* id groups the tile tower holds */

/* Where the tile tower reads its embedding rows when they are not pulled into bet_wide / bet_deep first:
 * straight from the parameter server's direct-indexed record slabs (b200ps_table_rows_ptr).  The row of
 * sample b in group g is the record of id uniq[g*B + inv[g*B + b]]; the ids are those the dedup wrote, so
 * they are inside their table.  Deep records must be 16-byte aligned (base, stride and param offset). */
typedef struct {
  const int64_t* uniq;                           /* [G][B] unique ids of each group (device) */
  const float* deep_base[B200_DEEPFM_TILE_MAXG]; /* record slab of group g's deep (dim 8) table */
  const float* wide_base[B200_DEEPFM_TILE_MAXG]; /* record slab of group g's wide (dim 1) table */
  int64_t deep_stride, wide_stride;              /* floats between consecutive records, same for every group */
  int64_t deep_param_off, wide_param_off;        /* float offset of the parameter row inside a record */
} b200_deepfm_rows_t;

typedef struct {
  int32_t G;               /* id groups */
  int32_t B;               /* samples in the batch */
  const int32_t* inv;      /* [G][B]  rank of each sample's id among its group's unique ids */
  const int32_t* n_unique; /* [G]     distinct ids per group (device) */
  const float* bet_wide;   /* [G][B]      pulled wide rows (first n_unique[g] valid) */
  const float* bet_deep;   /* [G][B][8]   pulled deep rows */
  const float* dense;      /* [B][13] */
  const float* labels;     /* [B] */
  const float* params;     /* flat parameter buffer, layout above */
  float* grads;            /* flat gradient buffer, same layout (overwritten) */
  float* gsum_wide;        /* [G][B]     d loss / d pulled rows, per unique id (overwritten) */
  float* gsum_deep;        /* [G][B][8] */
  float* loss;             /* [1] mean binary cross entropy with logits */
  float* logits;           /* [B] or NULL */
  float* scratch;          /* B*B200_DEEPFM_SCRATCH + 16*(13+8G) floats: per-sample backward state, then W1^T */
  const b200_deepfm_rows_t* rows; /* host struct or NULL.  Set: the tile tower's training entry points read the
                                     rows from the tables and bet_wide / bet_deep are not used; the other
                                     towers and the forward-only entry points refuse it (-1). */
} b200_deepfm_args_t;

size_t b200_deepfm_param_count(int G);
/* forward + backward of one batch; asynchronous on `stream` (cudaStream_t). */
int b200_deepfm_fwd_bwd(const b200_deepfm_args_t* args, void* stream);
/* Same contract as b200_deepfm_fwd_bwd, computed by the tensor-core tower (csrc/deepfm_tower_mma.cu): the
 * rows of a chunk of samples are gathered once into a shared-memory tile and the three first-layer
 * contractions run as 3xTF32 mma.sync.  `scratch` is not used. */
int b200_deepfm_fwd_bwd_mma(const b200_deepfm_args_t* args, void* stream);
int64_t b200_deepfm_mma_launch_count(void);
/* Same contract, computed by the TILE tower (csrc/deepfm_tower2.cu, round 2, the default): a CTA gathers the
 * rows of 32 samples once into shared memory (cp.async) and runs forward, backward and the
 * parameter-gradient contraction from that tile -- two launches (prep + tile kernel).  `scratch` needs
 * 320*16 + 16 floats (W1 in tile column order, then the dynamic tile counter); at most 38 id groups. */
int b200_deepfm_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_forward_tile(const b200_deepfm_args_t* args, void* stream);
/* b200_deepfm_fwd_bwd_tile in its two halves, so that a caller can put the prologue on another stream, beside
 * the row pull: the prologue (W1 into tile order; zero the gradient buffers, the loss and the live rows of the
 * per-unique-id sums) reads only `params` and `n_unique`; the main kernel needs the prologue and the pulled rows. */
/* The step's loss to the host without a copy-engine operation: ring_host_mapped is pinned host memory as the
 * device sees it (cudaHostAlloc / UVA); entry cursor % ring_len receives *loss_dev, then the cursor advances. */
int b200_deepfm_publish_loss(const float* loss_dev, float* ring_host_mapped, int ring_len, unsigned* cursor_dev, void* stream);
int b200_deepfm_tile_prologue(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_tile_main(const b200_deepfm_args_t* args, void* stream);
int64_t b200_deepfm_tile_launch_count(void);

/* The dac_ctr Deep & Cross Network (model_zoo/dac_ctr/dcn_model.py:53-95) on the same tile design
 * (csrc/dcn_tower.cu): the DNN 16 -> 4 over x0 = [dense 13 | deep 8G] as above, a two-layer CrossNet over x0
 * ("vector" parameterization: x_{l+1} = x0 (x_l . w_l) + b_l + x_l), and
 *   logit = sum(wide) + w_dense . dense + w_out . [dnn_out 4 | x_2],
 *   loss  = mean BCE with logits + 1e-5 (|w_0|^2 + |w_1|^2)   (the gradients include 2e-5 w_l).
 * Parameter / gradient layout (floats), in = 13 + 8G:
 *   [ w_dense 13 (+3 pad) | w1 16 x in | b1 16 | w2 4 x 16 | b2 4 | w_out 4 + in | w_0 in | w_1 in | b_0 in | b_1 in ]
 * Same arguments and outputs as the DeepFM tile entry points (`loss` includes the L2 term); `scratch` needs
 * B200_DEEPFM_DCN_SCRATCH floats; at most 38 id groups, a larger G is refused (-1, b200_deepfm_last_error). */
#define B200_DEEPFM_DCN_SCRATCH (320 * 20 + 16) /* W1 and the cross weights in tile column order, counters */
size_t b200_deepfm_dcn_param_count(int G);
int b200_deepfm_dcn_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_dcn_tile_prologue(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_dcn_tile_main(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_dcn_forward_tile(const b200_deepfm_args_t* args, void* stream);
int64_t b200_deepfm_dcn_launch_count(void);
/* The dac_ctr Wide & Deep model (model_zoo/dac_ctr/wide_deep_model.py:62-107): DeepFM without its FM term,
 *   logit = sum(wide) + w_dense . dense + w3 . relu(W2 relu(W1 [dense | deep] + b1) + b2),
 *   loss  = mean BCE with logits   (no regularization term).
 * It has DeepFM's parameters: the DeepFM flat layout above and b200_deepfm_param_count.  Computed by the tile
 * tower's kernel without the FM term (csrc/deepfm_tower2.cu), with the same arguments, outputs, `scratch` and
 * refusals as the DeepFM tile entry points (at most 38 id groups; -1 and b200_deepfm_last_error); its launches
 * are counted by b200_deepfm_tile_launch_count. */
int b200_deepfm_wide_deep_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_wide_deep_tile_prologue(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_wide_deep_tile_main(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_wide_deep_forward_tile(const b200_deepfm_args_t* args, void* stream);
/* The dac_ctr xDeepFM model (model_zoo/dac_ctr/xdeepfm_model.py:55-107): Wide & Deep plus a Compressed Interaction
 * Network over the deep rows X0 = [G fields x 8] (layer_size (128, 128), relu, split_half, l2_reg 1e-5):
 *   Z_k[b, d, i H_k + j] = X0[b, i, d] X_k[b, j, d]   (H_0 = G, H_1 = 64),
 *   C_k[b, h, d] = relu(sum_K W_k[h, K] Z_k[b, d, K] + b_k[h]),  X_1 = C_0 channels 0..63,
 *   p = sum_d [C_0 channels 64..127 | C_1]  (192),
 *   logit = (the Wide & Deep logit) + w_ex . p + b_ex,
 *   loss  = mean BCE with logits + 1e-5 (|W_0|^2 + |W_1|^2)   (the gradients include 2e-5 W_k).
 * Parameter / gradient layout (floats): the DeepFM / Wide & Deep layout above, then
 *   [ W_0 128 x G^2 | b_0 128 | W_1 128 x 64G | b_1 128 | w_ex 192 | b_ex 1 ]
 * filter row h contiguous over K = i H_k + j (501,753 floats at G = 38, 496,577 of them the CIN's).
 * Computed by csrc/xdeepfm_cin.cu (the CIN, 3xTF32 mma.sync) and the Wide & Deep tile kernel with the CIN logit
 * (csrc/deepfm_tower2.cu), with the DeepFM tile entry points' arguments and outputs; `scratch` needs
 * b200_deepfm_xdeepfm_scratch_floats(G, B) floats (about 170 MB at G = 38, B = 32768).  The prologue reads only
 * `params` and `n_unique`.  Refused (-1, b200_deepfm_last_error, nothing launched): G < 2 (with one field the
 * model has no CIN), G > 38, a row source on the forward-only entry, a null scratch.  Its launches, the tile
 * kernel's included, are counted by b200_deepfm_xdeepfm_launch_count. */
size_t b200_deepfm_xdeepfm_param_count(int G);
size_t b200_deepfm_xdeepfm_scratch_floats(int G, int B);
int b200_deepfm_xdeepfm_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_xdeepfm_tile_prologue(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_xdeepfm_tile_main(const b200_deepfm_args_t* args, void* stream);
int b200_deepfm_xdeepfm_forward_tile(const b200_deepfm_args_t* args, void* stream);
int64_t b200_deepfm_xdeepfm_launch_count(void);
/* Why the last call of any tower entry point (publish_loss included) that returned -1 (refused) or -2 (launch
 * error) failed; on the calling thread. */
const char* b200_deepfm_last_error(void);
/* forward only (logits), for evaluation. */
int b200_deepfm_forward(const b200_deepfm_args_t* args, void* stream);
/* kernels launched by the two calls above so far */
int64_t b200_deepfm_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif
