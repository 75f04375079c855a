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
 *   as composed by model_zoo/dac_ctr/feature_transform.py:36-118 (transform_feature / transform_group), and
 *   - elasticdl_preprocessing/layers/index_lookup.py:57-128   IndexLookup = index_table_from_tensor with
 *         num_oov_buckets (term at vocabulary position i -> i; any other string -> V + Fingerprint64 % n_oov,
 *         or -1 with n_oov = 0); also census_wide_deep_model/keras_process_layer.py:55-65 (CategoryLookup)
 *   - elasticdl_preprocessing/layers/log_round.py:53-98        LogRound = rint(log(x) [/ log(base)]) in float64
 *   - elasticdl_preprocessing/layers/round_identity.py:44-86   RoundIdentity = rint(x) in float32
 *         (both: an id outside [0, num_bins) -- NaN, +-inf and >= 2^63 included -- becomes default_value)
 *   as composed by model_zoo/census_wide_deep_model/wide_deep_functional_api.py:120-161 (transform_group).
 *
 * Vocabulary table (LOOKUP): open addressing with linear probing over n_slots = a power of two >= 2V slots
 * (load <= 0.5).  Slot = b200feat_vocab_slot_t {Fingerprint64(term), index (-1 = empty), length}; a term's
 * home slot is fingerprint & (n_slots - 1).  Beside it sit the terms, a zero-padded uint8 [V][Wv] matrix
 * (Wv <= 64).  b200feat_vocab_build fills both on the HOST, inserting in vocabulary order (so the bytes are
 * a function of the vocabulary alone); the kernels probe at most n_slots slots, so a malformed table cannot
 * hang a launch.  The table holds indices and fingerprints, no addresses: it can be copied between devices.
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
  B200FEAT_HASH_INT = 2,    /* Hashing(num_bins) of numeric column `column`: tf.as_string, then hash (int64 columns only) */
  B200FEAT_LOOKUP = 3,      /* IndexLookup of string column `column`; num_bins = num_oov_tokens (>= 0); table in ext */
  B200FEAT_LOG_ROUND = 4,   /* LogRound of numeric column `column`; num_bins = num_bins; default / base in ext */
  B200FEAT_ROUND_IDENTITY = 5 /* RoundIdentity of numeric column `column`; num_bins = num_buckets; default in ext */
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

/* One slot of a vocabulary table (16 bytes, read with one 16-byte load). */
typedef struct {
  uint64_t fingerprint; /* Fingerprint64 of the term */
  int32_t index;        /* vocabulary position, -1 = empty slot */
  int32_t length;       /* the term's length in bytes */
} b200feat_vocab_slot_t;

/* Per-group extension of b200feat_group_t, parallel to the groups array (b200feat_transform_ext). */
typedef struct {
  const b200feat_vocab_slot_t* slots_dev; /* LOOKUP: n_slots slots (device) */
  const uint8_t* terms_dev;               /* LOOKUP: [V][Wv] zero-padded terms (device) */
  int64_t n_slots;                        /* LOOKUP: a power of two >= 2V */
  int32_t V;                              /* LOOKUP: vocabulary size, >= 1 */
  int32_t Wv;                             /* LOOKUP: term row width, 1..64 */
  int64_t default_value;                  /* LOG_ROUND, ROUND_IDENTITY: the id of a value outside [0, num_bins) */
  int32_t has_base;                       /* LOG_ROUND: 0 = natural log (base None), 1 = log(x) / log(base) */
  int32_t absent;                         /* any kind: 0 = every cell gets an id; 1 = a cell ToSparse drops with
                                           * its default ignore_value (to_sparse.py:55-63) -- an empty string, a
                                           * float32 0.0 (-0.0 too) or an int64 -1 -- is absent: its id is -1,
                                           * without the offset.  (A LOOKUP without OOV tokens still writes
                                           * -1 + offset for an unknown string.) */
  double base;                            /* LOG_ROUND with has_base */
} b200feat_group_ext_t;

const char* b200feat_last_error(void);

/* Slot count of a V-term table: the least power of two >= 2V; -1 for V < 1 or V >= 2^31. */
int64_t b200feat_vocab_slots(int64_t V);
/* Builds a vocabulary table on the HOST: terms is a host [V][Wv] zero-padded matrix (a term ends at its first
 * NUL and the row must be zero after it), slots_out a host array of n_slots slots.  A term seen before is refused:
 * the return is -1 and *dup_pos (if not NULL) is the position of its second occurrence.  Refuses V < 1,
 * V >= 2^31, Wv outside 1..64 and an n_slots that is not a power of two >= 2V. */
int b200feat_vocab_build(const uint8_t* terms, int64_t V, int Wv, int64_t n_slots, b200feat_vocab_slot_t* slots_out,
                         int64_t* dup_pos);

/* One fused launch: ids_out_dev[g*B + b] for every group, dense_out_dev[b*n_dense + j] for every
 * normalised column.  groups / dense descriptors and boundaries are HOST arrays (copied by value into
 * the launch, G <= 64, n_dense <= 32, total boundaries <= 256).  numeric_is_float: 0 = int64 columns,
 * 1 = float32 columns (Discretization compares them in float, like int64 columns; HASH_INT refuses them).
 * ids32: 0 = int64 ids, 1 = int32 ids (narrow transport into b200ps_unique_bounded_i32); a group whose
 * ids [offset, offset + num_bins) or [offset, offset + n_boundaries] leave int32 is refused.
 * Any of the two outputs may be NULL.  Takes the kinds 0..2 only (b200feat_transform_ext with ext = NULL). */
int b200feat_transform(const b200feat_group_t* groups, int G, const float* boundaries, int n_boundaries,
                       const b200feat_dense_t* dense, int n_dense, const void* numeric_dev, int n_numeric,
                       int numeric_is_float, const uint8_t* strings_dev, int n_string, int W, int64_t B,
                       void* ids_out_dev, int ids32, float* dense_out_dev, void* stream);
/* The same launch with every group kind: ext (HOST array of G, or NULL) carries what LOOKUP / LOG_ROUND /
 * ROUND_IDENTITY need beyond b200feat_group_t; with ext = NULL those kinds are refused as unknown.
 * LOOKUP reads string column `column` (any W: an input longer than Wv is out of vocabulary); LOG_ROUND and
 * ROUND_IDENTITY read numeric column `column` (int64 columns: LogRound casts to float64, RoundIdentity passes
 * them through; float32 columns: rounded in float64 / in float32).  ids32 also refuses a group whose id set
 * plus its offset leaves int32: [0, V + n_oov) or {-1} u [0, V) for LOOKUP, [0, num_bins) u {default_value}
 * for the other two. */
int b200feat_transform_ext(const b200feat_group_t* groups, const b200feat_group_ext_t* ext, int G,
                           const float* boundaries, int n_boundaries, const b200feat_dense_t* dense, int n_dense,
                           const void* numeric_dev, int n_numeric, int numeric_is_float, const uint8_t* strings_dev,
                           int n_string, int W, int64_t B, void* ids_out_dev, int ids32, float* dense_out_dev,
                           void* stream);

/* The layers one by one (thin wrappers over the same device code). */
int b200feat_hash_strings(const uint8_t* strings_dev, int W, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream);
int b200feat_hash_ints(const int64_t* values_dev, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream);
int b200feat_bucketize(const float* x_dev, int64_t n, const float* boundaries, int n_boundaries, int64_t* out_dev,
                       void* stream);
/* IndexLookup (index_lookup.py:78-96) of n zero-padded strings of width W through a table of b200feat_vocab_build */
int b200feat_index_lookup(const uint8_t* strings_dev, int W, int64_t n, const b200feat_vocab_slot_t* slots_dev,
                          const uint8_t* terms_dev, int64_t n_slots, int32_t V, int32_t Wv, int64_t num_oov_tokens,
                          int64_t* out_dev, void* stream);
/* LogRound (log_round.py:75-86) / RoundIdentity (round_identity.py:70-81) of n values: int64 (x_is_float = 0)
 * or float32 (x_is_float = 1) */
int b200feat_log_round(const void* x_dev, int x_is_float, int64_t n, int64_t num_bins, int64_t default_value,
                       int has_base, double base, int64_t* out_dev, void* stream);
int b200feat_round_identity(const void* x_dev, int x_is_float, int64_t n, int64_t num_buckets, int64_t default_value,
                            int64_t* out_dev, void* stream);
/* raw FarmHash Fingerprint64 of zero-padded strings (tests / tools) */
int b200feat_fingerprint64(const uint8_t* strings_dev, int W, int64_t n, uint64_t* out_dev, void* stream);
int64_t b200feat_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* B200_FEATURES_H_ */
