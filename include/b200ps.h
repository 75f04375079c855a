/*
 * b200ps.h -- C ABI of libb200ps.so: the GPU-native replacement for the
 * ElasticDL parameter-server data path.
 *
 * What it replaces (paths relative to /root/reference/elasticdl/):
 *   - the cgo C ABI go/pkg/kernel/capi/kernel_api.h:10-37 (SGD/Momentum/Adam/
 *     Adagrad on raw float*), and the per-row Sparse and Indexed loops of
 *     go/pkg/kernel/kernel.go:27-199 that call it;
 *   - the state those kernels run on: go/pkg/common/embedding_table.go:22-88
 *     and go/pkg/ps/model.go:25-107;
 *   - the RPC surface of go/pkg/ps/server.go:144-230 (proto/elasticdl.proto:78-86)
 *     that python/worker/ps_client.py:87-301 fans out to.
 *
 * Model: a *PS group* of N shards.  A shard's memory (row slabs, dense
 * parameters, control block) lives in the HBM of one GPU.  A client process
 * creates the group view, creates the shards it owns, and imports the shards
 * owned by peer processes (CUDA IPC); every kernel then dereferences the owning
 * shard's memory directly (local HBM or NVLink peer access) -- there is no
 * serialisation and no host hop.  Rows are placed as shard = id % N,
 * slot = id / N (python/common/hash_utils.py:22-23); dense parameters live on
 * the shard the caller names (string_to_id, hash_utils.py:17-19).
 *
 * Conventions: every pointer named *_dev is a DEVICE pointer valid on the
 * client device; `stream` is a cudaStream_t of the client device passed as
 * void*; calls are asynchronous on that stream unless noted.  Return value:
 * 0 = ok, negative = error (B200PS_E*), message via b200ps_last_error().
 * No torch types, no C++ types.
 */
#ifndef B200PS_H_
#define B200PS_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200PS_ABI_VERSION 2
#define B200PS_MAX_SHARDS 16
#define B200PS_MAX_SEGS 96 /* segments per batched launch (DeepFM: 76 tables in one) */

enum {
  B200PS_OK = 0,
  B200PS_EINVAL = -1,    /* bad argument / optimizer-arg grammar (optimizer.go:304-326) */
  B200PS_ECUDA = -2,     /* CUDA runtime error (no device, OOM, launch failure) */
  B200PS_ENOTFOUND = -3, /* unknown table / parameter ("grad %s not in Parameter", optimizer.go:49,59) */
  B200PS_EWIDTH = -4,    /* "grad width is not equal to embedding dim" (kernel.go:36-38) */
  B200PS_ERANGE = -5,    /* id outside the table (embedding_delegate.py:254-264) */
  B200PS_ESTATE = -6     /* call out of order / shard not attached */
};

typedef struct b200ps b200ps_t;

/* One (table, ids, rows) segment of a batched pull / push / set.
 * n_dev (optional) points at a device int32 holding the live row count
 * (<= n), so that callers never have to read a unique-count back to the host. */
typedef struct {
  int32_t table;        /* id from b200ps_table_register / b200ps_dense_register */
  int32_t n;            /* rows in this segment (upper bound when n_dev != NULL) */
  const int64_t* ids_dev;
  const int32_t* n_dev;
  float* rows_dev;      /* [n, dim] row-major: pull output / gradient input / values to set */
} b200ps_seg_t;

const char* b200ps_last_error(void);
int b200ps_abi_version(void);

/* ---- lifecycle ------------------------------------------------------- */

/* ≙ NewServer(optType, optArgs, ..., lrStalenessModulation), server.go:89-120,
 * one call for the whole group.  opt_args uses the exact "k=v;k=v;" grammar of
 * optimizer.go:304-390 ("SGD" | "Adam" | "Adagrad" as in Go; "Ftrl" added, see
 * DESIGN.md).  flags: bit0 = reproduce quirk Q1 (dense AMSGrad applied twice,
 * optimizer.go:186-192), bit1 = do not track created rows. */
int b200ps_create(int n_shards, int client_device, const char* opt_type, const char* opt_args,
                  int lr_staleness_modulation, unsigned flags, b200ps_t** out);
int b200ps_destroy(b200ps_t* ps);

/* A second client view of the SAME shards inside one process (one view per worker thread /
 * stream: each view has its own per-push scratch, error word and directory copy).  The
 * reference's tests drive several workers as threads against shared PS instances
 * (python/tests/worker_ps_interaction_test.py:136-151).  `src` keeps ownership of the memory
 * and must outlive the view; register tables on `src` first.  Call b200ps_commit on the view. */
int b200ps_clone_view(b200ps_t* src, int client_device, b200ps_t** out);

/* This process owns shard `shard_id`; its memory is allocated on `device`. */
int b200ps_shard_create_local(b200ps_t* ps, int shard_id, int device);
/* Serialise the CUDA-IPC handles of everything allocated so far on a local
 * shard; a peer process passes the blob to b200ps_shard_import (idempotent:
 * already-imported allocations are skipped, new ones are mapped). */
int b200ps_shard_export(b200ps_t* ps, int shard_id, void* blob, size_t cap, size_t* size);
int b200ps_shard_import(b200ps_t* ps, int shard_id, const void* blob, size_t size);

/* ---- model definition (every process, same order) -------------------- */

/* ≙ PushEmbeddingTableInfos -> Model.SetEmbeddingTableInfo + Opt.InitOptimizer
 * (server.go:224-230, model.go:57-63, optimizer.go:145-154).  Idempotent per
 * name.  capacity = number of ids (input_dim); rows are direct-indexed.
 * initializer: only the literal "uniform" randomises (embedding_table.go:51),
 * anything else zero-fills.  Returns the table id (>= 0) or an error. */
int b200ps_table_register(b200ps_t* ps, const char* name, int dim, const char* initializer,
                          int64_t capacity, uint64_t seed);
/* Two tables that are always addressed with the same ids -- a dim-8 table A and a dim-1 table B
 * (DeepFM's deep and wide embeddings of one id group) -- stored as ONE record per id so that one
 * memory request per id serves both (see ps_kernels.cuh "Paired tables").  Both names stay
 * individually addressable by every other call; b200ps_pull_rows_pair / b200ps_push_rows_pair
 * serve both at once.  Zero initializer only.  Returns A's id; B's id is b200ps_lookup(name_b). */
int b200ps_table_register_pair(b200ps_t* ps, const char* name_a, const char* name_b, const char* initializer,
                               int64_t capacity, uint64_t seed);
/* Same, for UNBOUNDED ids (an ElasticDL Embedding used without input_dim, e.g.
 * model_zoo/deepfm_edl_embedding): the shard keeps an open-addressing key array in HBM and a
 * row is created on first pull or push, like the Go map (embedding_table.go:41-58).
 * expected_rows sizes the slot pool (load factor <= 0.5); running out of slots raises
 * B200PS_ERANGE at the next b200ps_check.  "uniform" rows get slot-keyed draws (insertion-order
 * dependent, as the reference's seed = len(map) is). */
int b200ps_table_register_hashed(b200ps_t* ps, const char* name, int dim, const char* initializer,
                                 int64_t expected_rows, uint64_t seed);
/* ≙ PushModel's dense part: Model.InitFromModelPB + InitOptimizer slots
 * (model.go:70-72, optimizer.go:146-150).  A dense parameter is a [rows, dim]
 * matrix on one shard (1-D: rows = numel, dim = 1) so that IndexedSlices
 * gradients can address its rows (kernel.go:48-55).  Returns its id, which
 * shares the table id space. */
int b200ps_dense_register(b200ps_t* ps, const char* name, int shard, int64_t rows, int dim);
int b200ps_lookup(b200ps_t* ps, const char* name); /* id or B200PS_ENOTFOUND */
/* Upload the table directory to the client device; call after registering /
 * importing and before the first data call (cheap, idempotent). */
int b200ps_commit(b200ps_t* ps);

/* ---- data path ------------------------------------------------------- */

/* ≙ PullEmbeddingVectors / EmbeddingTable.GetEmbeddingVectors
 * (server.go:163-173, embedding_table.go:61-68) for up to B200PS_MAX_SEGS
 * (table, ids) requests in ONE launch: rows_dev[i] = row(ids_dev[i]). */
int b200ps_pull_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);
/* ≙ EmbeddingTable.SetEmbeddingVectors / dense push_model rows
 * (embedding_table.go:71-77). */
int b200ps_set_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);

/* Paired pull / push: segs_a[i] addresses table A of a pair (ids, n_dev, A rows [n,8]);
 * rows_b[i] / grads_b[i] are the dim-1 rows of table B for the same ids.  At most
 * B200PS_MAX_SEGS / 2 segments per call.  push_rows_pair belongs between push_begin and push_end. */
int b200ps_pull_rows_pair(b200ps_t* ps, const b200ps_seg_t* segs_a, float* const* rows_b, int nseg, void* stream);
int b200ps_push_rows_pair(b200ps_t* ps, const b200ps_seg_t* segs_a, float* const* grads_b, int nseg, void* stream);

/* Owner-computes exchange for rank-per-GPU groups (csrc/ps_exchange.cuh): instead of touching peer
 * rows one by one, each rank publishes its unique-id lists; every owner streams them over NVLink,
 * serves the ids it owns (id % N) from its own shard and returns the rows contiguously; gradient
 * rows travel back in the same order and the owner applies the optimizer to its own shard.  Every
 * rank must issue the same xchg calls in the same order (bulk-synchronous step).  Tables come in
 * (dim-8, dim-1) pairs addressed by the same ids; uniq / n_unique / bet / gsum are the [G][B]
 * buffers of b200ps_unique.  create: collective, then re-export / import the shards (the exchange
 * buffer is a peer-mapped allocation).  push belongs between b200ps_push_begin and b200ps_push_end
 * and updates the rows of the b200ps_xchg_pull that precedes it (gsum indexed like that pull's
 * bet rows); a push without its pull returns B200PS_ESTATE.  A row that several ranks push in one
 * step receives every rank's update, applied in rank order (rank 0's first), as if the ranks had
 * pushed one after the other.  An id outside the table (negative, or >= the table's rows per shard
 * x N) comes back as a zero row and makes the requesting rank's next b200ps_check fail with
 * B200PS_ERANGE; a push leaves such a row alone.
 * create accepts 1 <= G <= B200PS_MAX_SEGS / 2 pairs of direct-indexed tables striped over every
 * shard (b200ps_table_register or b200ps_table_register_pair), with one slot layout among the
 * deep tables and one among the wide tables, and a process that owns exactly one shard.  It
 * returns B200PS_EINVAL for G out of range, a hashed table, a dense parameter, a table pinned to
 * one shard, a raw buffer or differing slot layouts; B200PS_EWIDTH for dims other than 8 / 1;
 * B200PS_ENOTFOUND for an unknown table id; B200PS_ESTATE for a second create, a process without
 * exactly one local shard or a table not allocated on it.  A refused create changes nothing. */
int b200ps_xchg_create(b200ps_t* ps, int G, int B, const int32_t* deep_tables, const int32_t* wide_tables);
int b200ps_xchg_pull(b200ps_t* ps, const int64_t* uniq_dev, const int32_t* n_unique_dev, float* bet_deep_dev,
                     float* bet_wide_dev, void* stream);
int b200ps_xchg_push(b200ps_t* ps, const float* gsum_deep_dev, const float* gsum_wide_dev, void* stream);
/* Profiling aid: one pull + one push (after a b200ps_push_begin), a CUDA event after every kernel,
 * synchronous; ms_out[6] = post, serve, unscatter, send_upd, apply, wait_applied. */
int b200ps_xchg_profile(b200ps_t* ps, const int64_t* uniq_dev, const int32_t* n_unique_dev, float* bet_deep_dev,
                        float* bet_wide_dev, const float* gsum_deep_dev, const float* gsum_wide_dev, float* ms_out,
                        void* stream);

/* ≙ PullDenseParameters payload (server.go:144-160): copy whole dense
 * parameters owner-shard -> dst (segs[i].rows_dev; ids_dev/n ignored). */
int b200ps_pull_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);
/* ≙ PushModel dense payload (server.go:209-221): dst <- values. */
int b200ps_set_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);

/* Optimizer-slot access (slot 0 = the parameter itself, 1.. = the optimizer's
 * slot rows in the order m/v/max_square, velocity, accumulator/linear): read
 * (write = 0) or write (write = 1) slot rows / whole slot arrays.  The Go PS
 * never ships slots (they are not even checkpointed, quirk Q9); this exists for
 * the parity tests and for restoring state. */
int b200ps_slot_rows(b200ps_t* ps, int slot, int write, const b200ps_seg_t* segs, int nseg, void* stream);
int b200ps_slot_dense(b200ps_t* ps, int slot, int write, const b200ps_seg_t* segs, int nseg, void* stream);

/* ≙ PushGradients (server.go:176-206) = one ApplyGradients on EVERY shard
 * (ps_client.py:271-277, quirk Q7):
 *   begin : per shard step++ (optimizer.go:44), effective lr with staleness
 *           modulation against model_versions[s] (server.go:178-187);
 *   push_dense / push_rows : the Dense / Sparse / Indexed kernels fused with the
 *           optimizer update (kernel.go:27-199, kernel_api.cc:6-96);
 *   end   : per shard Version++ (server.go:196-199); versions_out (host, may be
 *           pinned) receives the N new versions after the stream reaches it.
 * push_rows expects ids unique within a segment (PSClient dedups first,
 * ps_client.py:255-257) -- use b200ps_unique + b200ps_segment_sum. */
int b200ps_push_begin(b200ps_t* ps, float learning_rate, const int32_t* model_versions, void* stream);

/* A learning-rate schedule of tf.keras.optimizers.schedules (TF 2.5), evaluated by push_begin on the device
 * (elasticdl/python/elasticdl/callbacks.py:69-109 runs it on the worker; server.go:178-187 applies its lr).
 * Argument x = max(max_s version_s - 1, 0), the shard versions push_begin reads; in double, rounded once to
 * float:
 *   PIECEWISE     values[0] for x <= boundaries[0], values[i] for boundaries[i-1] < x <= boundaries[i],
 *                 values[n_boundaries] past the last (boundaries strictly increasing, at most 32);
 *   EXPONENTIAL   initial * decay_rate^p, p = x / decay_steps (floored if staircase);
 *   INVERSE_TIME  initial / (1 + decay_rate * p), p as EXPONENTIAL;
 *   POLYNOMIAL    (initial - end) * (1 - s / D)^power + end; s = min(x, decay_steps), D = decay_steps, or with
 *                 cycle s = x, D = decay_steps * max(1, ceil(x / decay_steps)).
 * The value takes the place of push_begin's learning_rate, which is ignored while a schedule is installed;
 * staleness modulation still divides it and a value <= 0 falls back to the optimizer's lr. */
#define B200PS_LR_MAX_BOUNDARIES 32
enum {
  B200PS_LR_PIECEWISE = 1,
  B200PS_LR_EXPONENTIAL = 2,
  B200PS_LR_INVERSE_TIME = 3,
  B200PS_LR_POLYNOMIAL = 4
};
typedef struct {
  int32_t kind;         /* B200PS_LR_* */
  int32_t n_boundaries; /* PIECEWISE */
  int32_t staircase;    /* EXPONENTIAL, INVERSE_TIME */
  int32_t cycle;        /* POLYNOMIAL */
  double initial_learning_rate, decay_steps, decay_rate, end_learning_rate, power;
  double boundaries[B200PS_LR_MAX_BOUNDARIES];
  float values[B200PS_LR_MAX_BOUNDARIES + 1];
} b200ps_lr_schedule_t;
/* Install `s` on this client view (copied; NULL clears it).  Other views of the group, b200ps_clone_view's
 * included, keep their own.  B200PS_EINVAL, changing nothing, for an unknown kind, decay_steps <= 0 (the
 * decaying kinds), a non-finite parameter, or n_boundaries outside [0, 32] or boundaries not strictly
 * increasing (PIECEWISE). */
int b200ps_set_lr_schedule(b200ps_t* ps, const b200ps_lr_schedule_t* s);
int b200ps_push_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);
/* Dense gradients: rows_dev = gradient [numel]. */
int b200ps_push_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream);
/* Dense gradient REDUCE fused with the update: s = sum_r grads_dev[r] in fp32, left to right
 * (r = 0..n_replicas-1, pointers may be peer memory), then g = s / scale when divide != 0 (sync-SGD
 * averaging, python/ps/servicer.py:205-212: grad / grads_to_wait) or g = s * scale when divide == 0
 * (Horovod's postscale_factor, elasticai_api/pytorch/optimizer.py:141-157), then the optimizer update
 * in place (kernel_api.cc:6-96).  s / w and s * fl(1/w) differ in the last bit for most w that are not
 * powers of two.  divide with scale 0 is B200PS_EINVAL. */
int b200ps_push_dense_reduce(b200ps_t* ps, int dense_id, const float* const* grads_dev,
                             int n_replicas, float scale, int divide, void* stream);
int b200ps_push_end(b200ps_t* ps, int32_t* versions_out_host, void* stream);
/* begin / end that reach ONE shard only: the owner-side ApplyGradients of the allreduce controller's fused
 * reduce + update (every rank updates the slice it owns exactly once per step), and of the per-shard gRPC
 * facade (ps/grpc_server.py: one Pserver = one shard, server.go:176-206). */
int b200ps_push_begin_shard(b200ps_t* ps, int shard, float learning_rate, const int32_t* model_versions /* [n_shards] or NULL */,
                            void* stream);
int b200ps_push_end_shard(b200ps_t* ps, int shard, void* stream);

/* ---- the dense allreduce controller's data path (rank-per-GPU groups) ----------------------------
 * Replaces the Horovod collectives of elasticai_api/pytorch/optimizer.py:141-168 + the wrapped optimizer's
 * step: every rank keeps its flat gradient bucket in a RAW buffer that the peers map (CUDA IPC); the owner
 * of parameter slice s runs b200ps_push_dense_allreduce with the N peer pointers -- the reduce-scatter, the
 * averaging and the in-place optimizer update are ONE kernel that reads the peers' gradients over NVLink --
 * and every rank then reads the updated slices back with b200ps_pull_dense (the all-gather).  b200ps_barrier
 * orders the phases on the device (flags in the peer-mapped shard control blocks; no host round trip, no NCCL).
 * raw_register: a zero-filled allocation of `bytes` on every local shard, exported with the shard; returns its
 * id (shares the table id space).  raw_ptr: its address on `shard` as mapped on the client device.
 * push_dense_allreduce: b200ps_push_dense_reduce with divide = 0 and torch.optim's semantics, for SGD / momentum
 * / Adam / AMSGrad groups (B200PS_EINVAL otherwise): the parameter is read from param_dev (the caller's copy, so
 * its edits between steps count) and the updated value written to the PS copy.  Adam takes this step's
 * coefficients from the caller, evaluated in double from the double hyper-parameters as torch.optim.Adam
 * does: m = beta1 m + one_minus_beta1 g, v = beta2 v + one_minus_beta2 g^2, p -= alpha m / (sqrt(v) + epsilon)
 * with alpha = lr sqrt(1 - beta2^t) / (1 - beta1^t) and epsilon = eps sqrt(1 - beta2^t) -- torch adds eps to
 * sqrt(v) / sqrt(1 - beta2^t).  (kernel_api.cc adds eps to sqrt(v) and evaluates 1 - beta from the fp32
 * betas, 1.3e-5 off for beta2 = 0.999.)  SGD ignores the four; its lr is b200ps_push_begin_shard's. */
int b200ps_push_dense_allreduce(b200ps_t* ps, int dense_id, const float* param_dev, const float* const* grads_dev,
                                int n_replicas, float scale, float alpha, float epsilon, float one_minus_beta1,
                                float one_minus_beta2, void* stream);
int b200ps_raw_register(b200ps_t* ps, const char* name, size_t bytes);
int b200ps_raw_ptr(b200ps_t* ps, int table, int shard, void** ptr, size_t* bytes);
/* The record slab of a direct-indexed embedding table on `shard`, as mapped on the client device: slot s of
 * the shard's records is at base + s * row_stride floats, its parameter row param_off floats further; rows =
 * records on the shard.  For readers that gather rows themselves (b200_deepfm_rows_t).  Such a read does not
 * mark a row as created; a push of the row does.  B200PS_EINVAL for hashed tables, dense parameters and raw
 * buffers. */
int b200ps_table_rows_ptr(b200ps_t* ps, int table, int shard, float** base, int64_t* row_stride, int64_t* param_off,
                          int64_t* rows);
int b200ps_barrier(b200ps_t* ps, void* stream);
/* step++ only (a failed ApplyGradients still bumps it, quirk Q2). */
int b200ps_bump_step(b200ps_t* ps, void* stream);

/* ---- the reference's native C ABI, on device arrays -------------------
 * One-to-one with go/pkg/kernel/capi/kernel_api.h:10-37 (same argument order and meaning, a
 * stream appended): in-place dense optimizer kernels on raw float arrays, same arithmetic
 * (kernel_api.cc:6-96).  max_square == NULL selects plain Adam, else AMSGrad. */
int b200ps_kernel_sgd(const float* grad, float* param, float lr, long long size, void* stream);
int b200ps_kernel_momentum(const float* grad, float* param, float* velocity, float mu, int nesterov, float lr,
                           long long size, void* stream);
int b200ps_kernel_adam(const float* grad, float* param, float* m, float* v, float lr, long long size, long long step,
                       float beta1, float beta2, float epsilon, float* max_square, void* stream);
int b200ps_kernel_adagrad(const float* grad, float* param, float* m, float lr, long long size, float epsilon,
                          void* stream);

/* ---- id dedup (client side of the exchange) -------------------------- */

/* These three take `ps` only for the device and the launch counter; ps may be
 * NULL (current device).
 * tf.unique (embedding_delegate.py:85) for T equal-length id segments in one
 * launch (one persistent kernel, csrc/ps_unique.cuh): uniq_dev[t*k + r] = r-th distinct id of
 * segment t in FIRST-OCCURRENCE order, inv_dev[t*k + i] = rank of ids[t*k + i],
 * n_unique_dev[t] = number of distinct ids.  Workspace from b200ps_unique_workspace(T, k) bytes;
 * its content may be arbitrary on first use (a magic word detects a fresh / foreign workspace),
 * but one workspace must not be used by two streams at once. */
size_t b200ps_unique_workspace(int T, int64_t k);
/* Same with host-side knowledge of the id range of each segment (bounds[t] = table capacity, 0 =
 * unknown): small-range segments use a direct-address position array instead of the hash table.
 * An id outside [0, bounds[t]) is counted as id 0 and sets the range bit of the group's error word, so the
 * next b200ps_check() fails with B200PS_ERANGE (the reference raises for it, embedding_delegate.py:254-264). */
size_t b200ps_unique_bounded_workspace(int T, int64_t k, const int64_t* bounds);
int b200ps_unique_bounded(b200ps_t* ps, const int64_t* ids_dev, int T, int64_t k, const int64_t* bounds,
                          int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                          size_t workspace_bytes, void* stream);
int b200ps_unique(b200ps_t* ps, const int64_t* ids_dev, int T, int64_t k, int64_t* uniq_dev,
                  int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev, size_t workspace_bytes,
                  void* stream);
/* Narrow id transport: the same dedup over int32 ids (every table capacity < 2^31, e.g. ids that crossed
 * PCIe as 4-byte words); the widening to int64 happens at the kernel's first read, the outputs
 * (uniq_dev int64, inv_dev, n_unique_dev) are identical to b200ps_unique_bounded on the widened ids. */
int b200ps_unique_bounded_i32(b200ps_t* ps, const int32_t* ids32_dev, int T, int64_t k, const int64_t* bounds,
                              int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                              size_t workspace_bytes, void* stream);
/* The general form: ids int64 or int32; blocks_per_sm > 0 caps the persistent grid (a caller that overlaps
 * the dedup with other kernels on a second stream asks for a thin grid, 1 block per SM: the blocks keep
 * their registers for the whole call); 0 = as many as fit. */
int b200ps_unique_bounded_ex(b200ps_t* ps, const void* ids_dev, int ids_are_int32, int T, int64_t k, const int64_t* bounds,
                             int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                             size_t workspace_bytes, int blocks_per_sm, void* stream);
/* Narrowest id transport: segment t of the ids buffer holds k UNSIGNED ids of widths[t] bytes (1, 2 or 4; 8 =
 * int64), the segments back to back, each padded to 16 bytes (b200ps_packed_ids_bytes gives the total).  A
 * table with fewer than 256 / 65536 rows needs one / two bytes per id on PCIe and in HBM; the widening to
 * int64 happens at the dedup kernel's first read, the outputs are those of b200ps_unique_bounded. */
int b200ps_unique_packed(b200ps_t* ps, const void* ids_dev, const int32_t* widths, int T, int64_t k, const int64_t* bounds,
                         int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                         size_t workspace_bytes, int blocks_per_sm, void* stream);
size_t b200ps_packed_ids_bytes(const int32_t* widths, int T, int64_t k);
/* Profiling aid: a device buffer (>= 64 B per resident block) that the persistent kernels fill with
 * %globaltimer stamps per block and phase; NULL switches it off. */
int b200ps_debug_buffer(void* dev_ptr, size_t bytes);
/* deduplicate_indexed_slices' sum (tensor_utils.py:39-60) / gather backward:
 * out[t][inv[t][i], :] += values[t][i, :] with warp-level id dedup; out is
 * zeroed first for rows < k.  Refuses k * (dim / W) > INT32_MAX work items per
 * segment (W = 8 / 4 floats for 16 B aligned pointers and dim % 8 / % 4 == 0,
 * else 1). */
int b200ps_segment_sum(b200ps_t* ps, const float* values_dev, const int32_t* inv_dev, int T, int64_t k,
                       int dim, float* out_dev, void* stream);
/* forward of the layer's gather: out[t][i,:] = bet[t][inv[t][i], :]. */
int b200ps_gather_rows(b200ps_t* ps, const float* bet_dev, const int32_t* inv_dev, int T, int64_t k,
                       int dim, float* out_dev, void* stream);

/* ---- pooled lookup of a sparse [B, L] input (safe_embedding_lookup_sparse without weights,
 * embedding_delegate.py:108-230): prune ids < 0, give each empty row the id 0, sum each row's BET rows, scale
 * (combiner 0 = sum, 1 = mean: / cnt, 2 = sqrtn: / sqrtf(cnt)), write 0 for the rows that were empty.
 * The input is a coalesced COO: rows_dev int64 [nnz] in row-major order, vals_dev int64 or int32 [nnz].  All three
 * take the same (B, nnz, dim) and one workspace of b200ps_sparse_workspace(B, nnz, dim) bytes (16 B aligned), which
 * prep fills and combine / combine_grad use; either may run any number of times after one prep.  Each refuses a
 * workspace_bytes smaller than b200ps_sparse_workspace(B, nnz, dim), nnz + B above INT32_MAX.  ps may be NULL, as for
 * b200ps_unique. */
size_t b200ps_sparse_workspace(int64_t B, int64_t nnz, int dim);
/* Three launches, no host read.  ids_dev int64 [nnz + B] receives the filled id stream: row-major, the kept ids in
 * input order and one id 0 in the slot of each empty row, then copies of the last filled id up to nnz + B (a repeat
 * changes neither tf.unique's set nor its first-occurrence order, so b200ps_unique can take all nnz + B entries).
 * An entry whose row lies outside [0, B) is dropped and counted in the workspace's first int32 word. */
int b200ps_sparse_prep(b200ps_t* ps, const int64_t* rows_dev, const void* vals_dev, int vals_are_int32, int64_t B,
                       int64_t nnz, int dim, int64_t* ids_dev, void* workspace_dev, size_t workspace_bytes,
                       void* stream);
/* The same filled id stream and workspace from nn.EmbeddingBag input, in one launch with no host read: offsets_dev NULL
 * = a 2-D [B, width] id tensor (nnz = B * width); else 1-D ids [nnz] with int64 offsets [B] (offsets [B + 1] when
 * include_last_offset; ids past the last offset are not read).  Entries equal to padding_idx (-1 = none) are dropped and
 * counted by no bag; a bag with no kept entry is empty (the fill id 0, a zero output).  A negative id is dropped and
 * sets the group's range error; offsets that do not start at 0, decrease, or end past nnz make every bag empty and set
 * the group's offsets error: b200ps_check raises on either.  ps is required (its error word). */
int b200ps_bag_prep(b200ps_t* ps, const void* ids_dev, int ids_are_int32, const int64_t* offsets_dev, int64_t width,
                    int include_last_offset, int64_t padding_idx, int64_t B, int64_t nnz, int dim, int64_t* out_ids_dev,
                    void* workspace_dev, size_t workspace_bytes, void* stream);
/* out_dev[b, :] = s_b * sum of bet_dev[inv_dev[j], :] over row b's filled entries j; bet_dev is [U, dim] (the
 * unique rows), inv_dev is b200ps_unique's inverse of ids_dev.  One launch.  Rows of any length are split into
 * pieces of 256 entries across warps.  The sum is NOT in strict entry order: within a piece each lane sums a
 * lane-strided subset of the entries in order, the lanes are added through a fixed xor butterfly, and the pieces of a
 * row in piece order.  Every order is fixed, so two calls give the same bits, and the result lies within
 * (m - 1) 2^-24 sum|x| of the exact sum of m entries, as any order does. */
int b200ps_sparse_combine(b200ps_t* ps, const float* bet_dev, const int32_t* inv_dev, void* workspace_dev,
                          size_t workspace_bytes, int64_t B, int64_t nnz, int dim, int combiner, float* out_dev,
                          void* stream);
/* Its backward: gbet_dev [n_unique, dim] = 0, then gbet[inv[j], :] += s_row(j) * gout[row(j), :] for every entry j of
 * a non-empty row (b200ps_segment_sum's warp-dedup reduction, with its INT32_MAX work-item refusal: (nnz + B) *
 * (dim / W)). */
int b200ps_sparse_combine_grad(b200ps_t* ps, const float* gout_dev, const int32_t* inv_dev, const void* workspace_dev,
                               size_t workspace_bytes, int64_t B, int64_t nnz, int dim, int combiner, int64_t n_unique,
                               float* gbet_dev, void* stream);
/* The weighted lookup (safe_embedding_lookup_sparse with sparse_weights, nn.EmbeddingBag's per_sample_weights):
 * weights_dev float32 [nnz] in input-entry order (the coalesced COO's, or the bag input's), read through the entry
 * order prep records, so one prep serves weighted and unweighted combines.  out[b, :] = sum w_j bet[inv[j], :] over
 * row b's kept entries, divided by sum w_j (mean) or sqrtf(sum w_j^2) (sqrtn); each divisor is summed in the row's
 * order, so two calls give the same bits; an empty row gives 0, a non-empty row whose divisor is 0 divides by 0 in IEEE
 * arithmetic.  Unit weights give the bits of b200ps_sparse_combine.  The combine stores each row's divisor in the
 * workspace, and the grad of mean / sqrtn reads it: run the grad after the weighted combine of the same weights. */
int b200ps_sparse_combine_weighted(b200ps_t* ps, const float* bet_dev, const int32_t* inv_dev,
                                   const float* weights_dev, void* workspace_dev, size_t workspace_bytes, int64_t B,
                                   int64_t nnz, int dim, int combiner, float* out_dev, void* stream);
/* Its backward: gbet[inv[j], :] += gout[row(j), :] * w_j / d_row (no division for sum).  gweights_dev (nullable,
 * float32 [nnz], sum combiner only; refused otherwise) receives dot(bet[inv[j], :], gout[row(j), :]) for each kept
 * input entry and 0 for every dropped one; bet_dev is needed with it. */
int b200ps_sparse_combine_weighted_grad(b200ps_t* ps, const float* gout_dev, const int32_t* inv_dev,
                                        const float* weights_dev, const float* bet_dev, const void* workspace_dev,
                                        size_t workspace_bytes, int64_t B, int64_t nnz, int dim, int combiner,
                                        int64_t n_unique, float* gbet_dev, float* gweights_dev, void* stream);

/* ---- state queries (synchronous on the client device) ---------------- */
int b200ps_shard_state(b200ps_t* ps, int shard, int32_t* version, int64_t* step, int32_t* initialized);
int b200ps_set_shard_state(b200ps_t* ps, int shard, int32_t version, int64_t step, int32_t initialized);
/* Asynchronous snapshot of every shard's control block: out_host[3*s + {0,1,2}] =
 * {version, step, initialized} once `stream` reaches the copy (out_host should be
 * pinned).  ≙ the version / initialized fields of PullDenseParametersResponse. */
int b200ps_snapshot_state(b200ps_t* ps, int64_t* out_host, void* stream);
/* PushModel's first-writer-wins handshake (server.go:209-221, `s.lock` +
 * `!s.Model.Initialized`): try_init atomically claims an uninitialised shard
 * (*won = 1 for exactly one caller, synchronous); the winner writes the dense
 * parameters (b200ps_set_dense) and calls finish_init, which publishes
 * Initialized = true and adopts `version` if >= 1 (model.go:84-86). */
int b200ps_try_init(b200ps_t* ps, int shard, int* won);
int b200ps_finish_init(b200ps_t* ps, int shard, int32_t version, void* stream);
/* number of created rows of a table on a shard (len(EmbeddingVectors)) */
int b200ps_table_size(b200ps_t* ps, int table, int shard, int64_t* rows);
/* ids of created rows of a table on a shard (ToIndexedSlices, embedding_table.go:80-88);
 * ids_dev capacity cap; *n receives the count. */
int b200ps_table_ids(b200ps_t* ps, int table, int shard, int64_t* ids_dev, int64_t cap, int64_t* n);
/* Raise and clear the sticky device-side error word (out-of-range ids ...). */
int b200ps_check(b200ps_t* ps);
/* Kernels launched so far by this group (bench.py gpu_launches); ps == NULL:
 * launches of the group-less primitives. */
int64_t b200ps_launch_count(b200ps_t* ps);

#ifdef __cplusplus
}
#endif
#endif /* B200PS_H_ */
