// Device-visible data layout of a PS group (see DESIGN.md "HBM layout").
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200ps.h"

namespace b200ps_impl {

constexpr int kMaxShards = B200PS_MAX_SHARDS;
constexpr int kMaxSegs = B200PS_MAX_SEGS;
constexpr int kMaxSlots = 3;

// Optimizer kinds.  Slot counts: go/pkg/ps/optimizer.go:145-154 (Momentum v),
// :222-237 (Adam m, v[, maxSquare]), :273-282 (Adagrad m); FTRL accumulator +
// linear and the Keras optimizers of the Python PS (python/ps/optimizer_wrapper.py:116-149,
// slot names :200-210): RMSprop rms[, momentum][, mg], Adadelta accum_grad, accum_var,
// Adamax / Nadam m, v.  RMSprop is four kinds ({plain, momentum} x {not centered, centered}):
// the slot count and the arithmetic differ (DESIGN.md section 4, Q13).
enum OptKind : int {
  kSGD = 0, kMomentum = 1, kAdam = 2, kAMSGrad = 3, kAdagrad = 4, kFTRL = 5,
  kRMSprop = 6, kRMSpropMomentum = 7, kRMSpropCentered = 8, kRMSpropCenteredMomentum = 9,
  kAdadelta = 10, kAdamax = 11, kNadam = 12,
};
constexpr int kNumOptKinds = 13;

__host__ __device__ constexpr int opt_slots(int kind) {
  return kind == kSGD ? 0 : kind == kMomentum ? 1 : kind == kAdam ? 2 : kind == kAMSGrad ? 3
       : kind == kAdagrad ? 1 : kind == kFTRL ? 2 : kind == kRMSprop ? 1
       : kind == kRMSpropMomentum || kind == kRMSpropCentered ? 2 : kind == kRMSpropCenteredMomentum ? 3
       : 2;  // Adadelta, Adamax, Nadam
}

// Nadam's momentum schedule S_t = u_1 * ... * u_t (Keras' float32 `m_cache`) as a table indexed by the
// step, built on the host once per group: concurrent pushers draw their steps with an atomic, so a
// running product could not be advanced in step order.  The table ends where S_t stops changing
// (it reaches 0, or a subnormal that u_t < 1 no longer moves).  The first factors are near beta_1 / 2,
// so every beta_1 in [0, 1] settles within 160 steps; a beta_1 whose schedule has not settled after
// kNadamMaxSteps steps (beta_1 > 1 drives S_t to infinity) is refused.
constexpr int kNadamMaxSteps = 1 << 16;

struct OptParams {
  int kind;
  int nesterov;
  float lr;  // opt.lr, the fallback when the request carries learning_rate <= 0 (server.go:183-187)
  float mu;
  float beta1, beta2, epsilon;
  float c1, c2;  // (float)(1.0 - beta): kernel_api.cc:63,65 evaluate (1.0 - beta) in double
  float l1, l2, l2s, beta, init_accum;  // FTRL
  // RMSprop / Adadelta keep rho in beta1 and (float)(1.0 - rho) in c1, RMSprop's momentum in mu; Adamax and
  // Nadam use beta1, beta2, c1, c2, epsilon as Adam does.  (No new fields: every row kernel takes this struct.)
};

// One table (embedding table or dense parameter) as the kernels see it.
//   embedding table: rows striped over shards, shard = id % N, slot = id / N;
//     a row RECORD holds the parameter row and its optimizer slot rows
//     back to back ([p(dim) | s0(dim) | s1(dim) ...], record stride padded to
//     16 B) so one push touches one contiguous span of HBM;
//   dense parameter: all rows on `owner`; param and slots are separate
//     contiguous arrays (structure of arrays) so the whole-tensor update
//     streams at full width.
struct TableView {
  float* base[kMaxShards];        // record slab / param array on each shard (peer-mapped)
  uint32_t* present[kMaxShards];  // created-row bitmap (nullptr: untracked)
  long long* keys[kMaxShards];    // hashed tables (unbounded ids): open-addressing key array, else nullptr
  int64_t rows;                   // rows per shard (striped) / total rows (dense)
  int64_t row_stride;             // floats between consecutive rows
  int64_t slot_off[kMaxSlots + 1];  // float offset of [param, slot0, slot1, slot2] from the row start
  int32_t dim;
  int32_t n_slots;
  int32_t owner;  // -1: striped by id % N; >= 0: dense parameter on this shard
  int32_t is_dense;
};

// Per-shard control block, resident on the owning shard, peer-mapped everywhere:
// Model.Version / Model.Initialized (model.go:25-31) and BaseOptimizer.step
// (optimizer.go:33-35).
struct ShardCtl {
  long long step;
  int version;
  int initialized;
  unsigned err;
  int bar_count;  // b200ps_barrier: arrivals (every rank adds 1 to every shard's counter per barrier)
  int bar_epoch;  // b200ps_barrier: barriers this shard's owner has entered
  int pad[9];
};

// Per-push values produced by k_push_begin, consumed by the update kernels.  Every row kernel hands
// these three words to opt_update<OPT> and the exchange header carries them verbatim, so a kind that
// needs other per-push scalars folds them into these three (nadam_coefs).
struct PushRt {
  float lr[kMaxShards];     // effective lr (server.go:176-187); Nadam: coefficient of g (nadam_coefs)
  float alpha[kMaxShards];  // Adam lr_t = lr*sqrt(1-b2^t)/(1-b1^t), double math (kernel_api.cc:67);
                            // Adamax lr/(1-b1^t); Nadam: coefficient of m
  float l2adj[kMaxShards];  // FTRL l2 + beta/(2*lr); Nadam: epsilon*sqrt(1-b2^t)
  long long step[kMaxShards];
  int version[kMaxShards];
};

struct GroupView {
  const TableView* tables;
  ShardCtl* ctl[kMaxShards];
  PushRt* rt;
  unsigned* err;  // client-local sticky error word
  int n_shards;
  int shard_shift;  // log2(n_shards) if power of two, else -1
};

struct SegBatch {
  b200ps_seg_t seg[kMaxSegs];
  int nseg;
};

enum ErrBits : unsigned { kErrRange = 1u, kErrWidth = 2u, kErrFull = 4u };
constexpr long long kEmptySlot = (long long)0x8000000000000000ULL;

}  // namespace b200ps_impl
