/*
 * b200_fc_dnn.h -- C ABI of the feature-column DNN tower (csrc/fc_dnn_tower.cu): the model zoo's
 * DenseFeatures -> Dense(16, relu) -> Dense(16, relu) -> Dense(1, sigmoid) models
 * (model_zoo/census_dnn_model/census_functional_api.py:19-30, model_zoo/heart_functional_api/
 * heart_functional_api.py:45-57), forward, Keras binary cross-entropy on the probability, backward, the MLP
 * gradients and the gradient sum of every unique row of every embedding-column table, in one launch.
 *
 * The DenseFeatures input x [F] of a sample is described by a layout of column blocks, each at `offset` in x:
 *   NUMERIC    x[offset] = numeric[src][b]                                (numeric_column, pass-through)
 *   BUCKET     x[offset + i] = (ids[src][b] == i), i < width              (bucketized_column, one-hot)
 *   EMBEDDING  x[offset + d] = table src's row of the sample, d < dim     (EDL embedding_column, combiner over
 *              one id per sample; a sample whose string is empty has no id and gets a zero row)
 * Table k's rows are the step's pulled unique rows, rows[row_off(k) + inv[k][b] * dim_k + d], where row_off(k) =
 * sum over j < k of table_rows[j] * table_dim[j]; gsum has the same layout.  A table's ids are hash buckets, so
 * it has at most table_rows[k] unique rows.
 *
 * Flat MLP parameters, Keras [in, out] kernels (16 F + 305 floats):
 *   dense/kernel:0 [F, 16] @0, dense/bias:0 [16] @16F, dense_1/kernel:0 [16, 16] @16F+16,
 *   dense_1/bias:0 [16] @16F+272, dense_2/kernel:0 [16, 1] @16F+288, dense_2/bias:0 [1] @16F+304.
 *
 * Loss (DESIGN.md section 4, Q19): p = sigmoid(z) clipped to [1e-7, 1 - 1e-7], l = -(y log(p + 1e-7) + (1 - y)
 * log(1 - p + 1e-7)); no gradient flows where the clip is active.  loss_mean = 1: the loss and the gradients are
 * batch means; 0: batch sums (Q16).
 *
 * Every sum over samples is taken in a fixed order (per-CTA partials added by the last CTA in CTA order, no
 * float atomics), so two launches on one device give the same bits.
 * No torch types; every pointer except the layout is a device pointer; `stream` is a cudaStream_t passed as
 * void*.  Return 0 = ok, -1 = a refused argument, -2 = a CUDA error; message via b200_fc_dnn_last_error().
 */
#ifndef B200_FC_DNN_H_
#define B200_FC_DNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_FC_DNN_HIDDEN 16
#define B200_FC_DNN_TILE 64        /* samples per tile */
#define B200_FC_DNN_MAX_F 160      /* DenseFeatures width */
#define B200_FC_DNN_MAX_BLOCKS 16
#define B200_FC_DNN_MAX_TABLES 8
#define B200_FC_DNN_MAX_SLOTS 512  /* sum of table_rows */

enum { B200_FC_NUMERIC = 0, B200_FC_BUCKET = 1, B200_FC_EMBEDDING = 2 };

typedef struct {
  int32_t kind;   /* B200_FC_* */
  int32_t src;    /* NUMERIC: numeric row; BUCKET: ids row; EMBEDDING: table */
  int32_t width;  /* NUMERIC: 1; BUCKET: buckets (len(boundaries) + 1); EMBEDDING: the table's dim */
  int32_t offset; /* first column in x */
} b200_fc_block_t;

typedef struct {
  int32_t F;          /* columns of x; the blocks cover [0, F) exactly once */
  int32_t n_blocks;
  int32_t n_tables;
  int32_t loss_mean;  /* 1 = batch mean, 0 = batch sum */
  int32_t table_rows[B200_FC_DNN_MAX_TABLES];   /* hash buckets */
  int32_t table_dim[B200_FC_DNN_MAX_TABLES];
  int32_t table_string[B200_FC_DNN_MAX_TABLES]; /* the string column whose emptiness drops the table's id */
  b200_fc_block_t blocks[B200_FC_DNN_MAX_BLOCKS];
} b200_fc_layout_t;

typedef struct {
  int64_t B;               /* batch size, >= 1 */
  int32_t n_numeric;       /* rows of numeric */
  int32_t n_ids;           /* rows of ids */
  int32_t n_strings;       /* string columns */
  int32_t W;               /* string width in bytes */
  const float* numeric;    /* [n_numeric, B] */
  const int32_t* ids;      /* [n_ids, B] (BUCKET blocks read row src) */
  const uint8_t* strings;  /* [n_strings, B, W], zero-padded: a string is empty iff its first byte is 0 */
  const int32_t* inv;      /* [n_tables, B] the dedup's inverse index of each table's ids */
  const int32_t* n_unique; /* [n_tables] */
  const float* rows;       /* the pulled unique rows (layout above) */
  const float* labels;     /* [B]; unused by the forward */
  const float* params;     /* [16 F + 305] */
  float* loss;             /* [1] */
  float* logits;           /* [B] z, before the sigmoid */
  float* grads;            /* [16 F + 305] */
  float* gsum;             /* like rows: the gradient sum of unique row u of table k for u < n_unique[k] */
  void* workspace;         /* b200_fc_dnn_workspace_bytes bytes, zero before the first call; every call leaves
                            * its arrival counter at zero again, so a captured graph can replay */
  size_t workspace_bytes;
} b200_fc_dnn_args_t;

/* Floats of the flat MLP (16 F + 305); 0 for a refused layout. */
int64_t b200_fc_dnn_params(const b200_fc_layout_t* layout);
/* Workspace bytes for batch B on the current device (one partial per CTA of the persistent grid). */
size_t b200_fc_dnn_workspace_bytes(const b200_fc_layout_t* layout, int64_t B);
/* ids[k][b] = 0 for every table k (rows 0 .. n_tables - 1 of ids) whose string strings[table_string[k]][b] is
 * empty: the fill id that safe_embedding_lookup_sparse looks up for an empty row.  One launch. */
int b200_fc_dnn_fill_empty(const b200_fc_layout_t* layout, int32_t* ids, const uint8_t* strings, int64_t B, int W,
                           void* stream);
/* One launch: forward, loss, backward, MLP gradients and the per-table unique-row gradient sums. */
int b200_fc_dnn_tower(const b200_fc_layout_t* layout, const b200_fc_dnn_args_t* args, void* stream);
/* The forward alone: logits only (labels, loss, grads, gsum, n_unique and workspace unused). */
int b200_fc_dnn_forward(const b200_fc_layout_t* layout, const b200_fc_dnn_args_t* args, void* stream);
const char* b200_fc_dnn_last_error(void);
int64_t b200_fc_dnn_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_FC_DNN_H_ */
