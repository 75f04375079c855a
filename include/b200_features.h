/*
 * b200_features.h -- C ABI of the feature-id generation kernels (SURVEY.md section 8f-3): the
 * preprocessing layers ElasticDL's model zoo runs in front of the embedding lookups, on the GPU,
 * fused into one launch in front of b200ps_unique.
 *
 * What it replaces (paths relative to /root/reference/):
 *   - elasticdl_preprocessing/layers/hashing.py:61-92        Hashing = tf.strings.to_hash_bucket_fast
 *         (FarmHash Fingerprint64 of the string, mod num_bins; integers go through tf.as_string first)
 *   - elasticdl_preprocessing/layers/discretization.py:60-78  Discretization = math_ops._bucketize
 *         (left-closed bins: id = number of boundaries <= x)
 *   - elasticdl_preprocessing/layers/concatenate_with_offset.py:50-87  id + offsets[i], concatenated
 *   - elasticdl_preprocessing/layers/normalizer.py            (x - subtractor) / divisor
 *   as composed by model_zoo/dac_ctr/feature_transform.py:36-118 (transform_feature / transform_group).
 *
 * Inputs are FEATURE-MAJOR device arrays, like the reference's one-Keras-input-per-feature tensors:
 *   numeric  [n_numeric][B]      int64 (dac_ctr: tf.io.FixedLenFeature((1,), tf.int64)) or float32
 *   strings  [n_string][B][W]    zero-padded byte strings of at most W <= 64 bytes (a string ends at its
 *                                first NUL, so a string holding a NUL byte cannot be carried)
 * Outputs: ids [G][B] (int64 or int32), the layout b200ps_unique takes; dense [B][n_dense] float32.
 *
 * Parity: Fingerprint64 is third-party arithmetic (TensorFlow / FarmHash, not under /root/reference).
 * It is restated from the published farmhashna::Hash64 (lengths 0..64) and pinned by the reference's
 * only vector (hashing.py:35-39: 'A'..'E', 3 bins -> [1,0,1,1,2]); longer strings are rejected.
 * No torch types; every *_dev pointer is a device pointer; `stream` is a cudaStream_t passed as void*.
 * Return 0 = ok, negative = error, message via b200feat_last_error().
 */
#ifndef B200_FEATURES_H_
#define B200_FEATURES_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  B200FEAT_DISCRETIZE = 0,  /* Discretization(bins) of numeric column `column` */
  B200FEAT_HASH_STRING = 1, /* Hashing(num_bins) of string column `column` */
  B200FEAT_HASH_INT = 2     /* Hashing(num_bins) of numeric column `column`: tf.as_string, then hash (int64 columns only) */
};

/* One output id group = one feature transformed + its ConcatenateWithOffset offset
 * (feature_transform.py:80-118; dac_ctr's FEATURE_GROUPS hold one feature per group). */
typedef struct {
  int32_t kind;
  int32_t column;
  int32_t n_boundaries; /* DISCRETIZE: boundaries[boundary_off .. boundary_off + n_boundaries), ascending, no NaN */
  int32_t boundary_off;
  int64_t num_bins;     /* HASH_*: > 0 */
  int64_t offset;       /* added to the id (ConcatenateWithOffset) */
} b200feat_group_t;

/* Normalizer of numeric column `column` -> dense_out[:, j]. */
typedef struct {
  int32_t column;
  int32_t pad;
  double subtractor;
  double divisor;
} b200feat_dense_t;

const char* b200feat_last_error(void);

/* One fused launch: ids_out_dev[g*B + b] for every group, dense_out_dev[b*n_dense + j] for every
 * normalised column.  groups / dense descriptors and boundaries are HOST arrays (copied by value into
 * the launch, G <= 64, n_dense <= 32, total boundaries <= 256).  numeric_is_float: 0 = int64 columns,
 * 1 = float32 columns (Discretization compares them in float, like int64 columns; HASH_INT refuses them).
 * ids32: 0 = int64 ids, 1 = int32 ids (narrow transport into b200ps_unique_bounded_i32); a group whose
 * ids [offset, offset + num_bins) or [offset, offset + n_boundaries] leave int32 is refused.
 * Any of the two outputs may be NULL. */
int b200feat_transform(const b200feat_group_t* groups, int G, const float* boundaries, int n_boundaries,
                       const b200feat_dense_t* dense, int n_dense, const void* numeric_dev, int n_numeric,
                       int numeric_is_float, const uint8_t* strings_dev, int n_string, int W, int64_t B,
                       void* ids_out_dev, int ids32, float* dense_out_dev, void* stream);

/* The layers one by one (thin wrappers over the same device code). */
int b200feat_hash_strings(const uint8_t* strings_dev, int W, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream);
int b200feat_hash_ints(const int64_t* values_dev, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream);
int b200feat_bucketize(const float* x_dev, int64_t n, const float* boundaries, int n_boundaries, int64_t* out_dev,
                       void* stream);
/* raw FarmHash Fingerprint64 of zero-padded strings (tests / tools) */
int b200feat_fingerprint64(const uint8_t* strings_dev, int W, int64_t n, uint64_t* out_dev, void* stream);
int64_t b200feat_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_FEATURES_H_ */
