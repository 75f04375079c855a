// libb200ps.so -- host side of the C ABI declared in include/b200ps.h.
// State a Go PS keeps in maps (go/pkg/ps/model.go:25-31) lives here as HBM
// allocations on the owning shard's GPU plus a small directory (TableView[])
// mirrored to the client device.
#include <cuda_runtime.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include "ps_kernels.cuh"
#include "ps_flat.cuh"
#include "ps_unique.cuh"
#include "ps_exchange.cuh"

using namespace b200ps_impl;

namespace {

thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define CUDA_OK(expr)                                                                 \
  do {                                                                                \
    cudaError_t e_ = (expr);                                                          \
    if (e_ != cudaSuccess)                                                            \
      return fail(B200PS_ECUDA, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) {
    cudaGetDevice(&prev);
    if (prev != dev) cudaSetDevice(dev);
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

struct Alloc {  // one cudaMalloc on a shard, exported / imported as a CUDA-IPC handle
  void* ptr = nullptr;
  size_t bytes = 0;
  bool imported = false;  // mapped from a peer process (cudaIpcOpenMemHandle)
  bool borrowed = false;  // owned by another b200ps_t of this process (b200ps_clone_view)
};

struct Table {
  std::string name;
  int dim = 0;
  int n_slots = 0;
  bool is_dense = false;
  int owner = -1;
  int64_t rows = 0;  // per shard (striped) or total (dense)
  int64_t row_stride = 0;
  int64_t slot_off[kMaxSlots + 1] = {0, 0, 0, 0};
  size_t present_off = 0;  // byte offset of the bitmap inside the allocation
  size_t keys_off = 0;     // byte offset of the key array (hashed tables), 0 = direct-indexed
  bool hashed = false;
  bool raw = false;        // plain zero-filled bytes (the exchange buffer), no rows
  int pair_of = -1;        // >= 0: this table shares the record slab of table `pair_of` (b200ps_table_register_pair)
  int pair_b = -1;         // table A of a pair: id of its partner
  size_t base_off = 0;     // byte offset of this table's first float inside the shared allocation
  size_t bytes = 0;
  bool uniform = false;
  uint64_t seed = 0;
  Alloc alloc[kMaxShards];
};

struct Shard {
  bool local = false;
  bool attached = false;
  int device = -1;
  Alloc ctl;
};

// Blob layout for export / import.
struct BlobHeader {
  uint32_t magic;
  int32_t shard;
  int32_t n_entries;
  int32_t pad;
};
struct BlobEntry {
  int32_t table;  // -1: control block
  int32_t pad;
  uint64_t bytes;
  cudaIpcMemHandle_t handle;
};
constexpr uint32_t kBlobMagic = 0xB200F5A1u;

}  // namespace

struct b200ps {
  int n_shards = 0;
  int client_device = 0;
  OptParams opt{};
  int staleness = 0;
  unsigned flags = 0;
  Shard shard[kMaxShards];
  std::vector<Table> tables;
  std::unordered_map<std::string, int> by_name;
  TableView* d_tables = nullptr;
  int d_tables_cap = 0;
  bool dirty = true;
  PushRt* d_rt = nullptr;
  std::vector<float> nadam_sched;  // Nadam: S_t, t = 0..last (nadam_schedule); uploaded to d_nadam
  float* d_nadam = nullptr;
  unsigned* d_err = nullptr;
  int* d_versions = nullptr;
  unsigned long long* d_count = nullptr;
  long long* d_state = nullptr;
  long long launches = 0;
  int n_sm = 132;
  // owner-computes exchange (b200ps_xchg_*)
  int x_table = -1, x_G = 0, x_B = 0, x_me = -1;
  long long x_cap = 0, x_off_ids = 0, x_off_resp = 0, x_off_upd = 0, x_off_served = 0;
  bool x_pulled = false;
  XTabs x_tabs{};
  // the dedup's two kernels (small segments / large segments) run side by side: a second stream + fork / join events
  cudaStream_t u_side = nullptr;
  cudaEvent_t u_fork = nullptr, u_join = nullptr;
  std::mutex mu;
};

namespace {

// ---- optimizer argument grammar: go/pkg/ps/optimizer.go:284-390 -------------
int parse_bool(const std::string& s, bool* out) {  // strconv.ParseBool
  static const char* t[] = {"1", "t", "T", "TRUE", "true", "True"};
  static const char* f[] = {"0", "f", "F", "FALSE", "false", "False"};
  for (auto x : t) if (s == x) { *out = true; return 0; }
  for (auto x : f) if (s == x) { *out = false; return 0; }
  return -1;
}

int parse_float(const std::string& s, float* out) {
  char* end = nullptr;
  double v = strtod(s.c_str(), &end);
  if (end == s.c_str() || *end != '\0') return -1;
  *out = (float)v;  // strconv.ParseFloat(s, 32) then float32()
  return 0;
}

int parse_optimizer(const char* type_c, const char* args_c, OptParams* o) {
  std::string type = type_c ? type_c : "", args = args_c ? args_c : "";
  static const std::map<std::string, std::vector<std::string>> want = {
      {"SGD", {"learning_rate", "momentum", "nesterov"}},
      {"Adam", {"learning_rate", "beta_1", "beta_2", "epsilon", "amsgrad"}},
      {"Adagrad", {"learning_rate", "epsilon"}},
      {"Ftrl", {"learning_rate", "initial_accumulator_value", "l1_regularization_strength",
                "l2_regularization_strength", "l2_shrinkage_regularization_strength", "beta"}},
      // the Keras optimizers of the Python PS (optimizer_wrapper.py:116-149), get_config() key names
      {"RMSprop", {"learning_rate", "rho", "momentum", "epsilon", "centered"}},
      {"Adadelta", {"learning_rate", "rho", "epsilon"}},
      {"Adamax", {"learning_rate", "beta_1", "beta_2", "epsilon"}},
      {"Nadam", {"learning_rate", "beta_1", "beta_2", "epsilon"}},
  };
  auto it = want.find(type);
  if (it == want.end()) return fail(B200PS_EINVAL, "Unknown optimizer type " + type);
  std::map<std::string, std::string> kv;
  size_t pos = 0;
  while (pos <= args.size()) {  // strings.Split(optArgs, ";")
    size_t semi = args.find(';', pos);
    std::string item = args.substr(pos, semi == std::string::npos ? std::string::npos : semi - pos);
    if (!item.empty()) {
      size_t eq = item.find('=');
      if (eq == std::string::npos) return fail(B200PS_EINVAL, "malformed optimizer argument " + item);
      kv[item.substr(0, eq)] = item.substr(eq + 1);
    }
    if (semi == std::string::npos) break;
    pos = semi + 1;
  }
  for (auto& k : it->second)
    if (!kv.count(k)) return fail(B200PS_EINVAL, "Args passed to ps should contain " + k);
  if (kv.size() != it->second.size()) return fail(B200PS_EINVAL, "Args passed to ps contain redundant items");
  memset(o, 0, sizeof(*o));
  if (parse_float(kv["learning_rate"], &o->lr)) return fail(B200PS_EINVAL, "Having error converting learning rate to number");
  if (type == "SGD") {
    bool nes;
    if (parse_float(kv["momentum"], &o->mu) || parse_bool(kv["nesterov"], &nes)) return fail(B200PS_EINVAL, "bad SGD argument");
    o->nesterov = nes;
    o->kind = o->mu > 0.0f ? kMomentum : kSGD;  // optimizer.go:353-356
  } else if (type == "Adam") {
    bool ams;
    if (parse_float(kv["beta_1"], &o->beta1) || parse_float(kv["beta_2"], &o->beta2) ||
        parse_float(kv["epsilon"], &o->epsilon) || parse_bool(kv["amsgrad"], &ams))
      return fail(B200PS_EINVAL, "bad Adam argument");
    o->kind = ams ? kAMSGrad : kAdam;
    o->c1 = (float)(1.0 - (double)o->beta1);
    o->c2 = (float)(1.0 - (double)o->beta2);
  } else if (type == "Adagrad") {
    if (parse_float(kv["epsilon"], &o->epsilon)) return fail(B200PS_EINVAL, "bad Adagrad argument");
    o->kind = kAdagrad;
  } else if (type == "RMSprop") {
    bool centered;
    if (parse_float(kv["rho"], &o->beta1) || parse_float(kv["momentum"], &o->mu) ||
        parse_float(kv["epsilon"], &o->epsilon) || parse_bool(kv["centered"], &centered))
      return fail(B200PS_EINVAL, "bad RMSprop argument");
    const bool mom = o->mu > 0.0f;  // Keras: self._momentum = momentum > 0 (the momentum slot exists only then)
    o->kind = centered ? (mom ? kRMSpropCenteredMomentum : kRMSpropCentered) : (mom ? kRMSpropMomentum : kRMSprop);
    o->c1 = (float)(1.0 - (double)o->beta1);  // rho, 1 - rho (OptParams)
  } else if (type == "Adadelta") {
    if (parse_float(kv["rho"], &o->beta1) || parse_float(kv["epsilon"], &o->epsilon))
      return fail(B200PS_EINVAL, "bad Adadelta argument");
    o->kind = kAdadelta;
    o->c1 = (float)(1.0 - (double)o->beta1);  // rho, 1 - rho (OptParams)
  } else if (type == "Adamax" || type == "Nadam") {
    if (parse_float(kv["beta_1"], &o->beta1) || parse_float(kv["beta_2"], &o->beta2) ||
        parse_float(kv["epsilon"], &o->epsilon))
      return fail(B200PS_EINVAL, "bad " + type + " argument");
    o->kind = type == "Adamax" ? kAdamax : kNadam;
    o->c1 = (float)(1.0 - (double)o->beta1);
    o->c2 = (float)(1.0 - (double)o->beta2);
  } else {
    if (parse_float(kv["initial_accumulator_value"], &o->init_accum) ||
        parse_float(kv["l1_regularization_strength"], &o->l1) ||
        parse_float(kv["l2_regularization_strength"], &o->l2) ||
        parse_float(kv["l2_shrinkage_regularization_strength"], &o->l2s) || parse_float(kv["beta"], &o->beta))
      return fail(B200PS_EINVAL, "bad Ftrl argument");
    o->kind = kFTRL;
  }
  return B200PS_OK;
}

// Nadam's schedule S_0 = 1, S_t = S_{t-1} * u_t, multiplied in float32 in Keras' order, up to the first t
// where it stops changing (ps_types.cuh, kNadamMaxSteps).  From there on it never changes again: once 0 it
// stays 0, and for 0 <= beta_1 <= 1 the factors u_t grow with t and stay below 1, so S * u keeps rounding to S.
int nadam_schedule(float beta1, std::vector<float>* s) {
  s->assign(1, 1.0f);
  for (long long t = 1; t <= kNadamMaxSteps; ++t) {
    const float prev = s->back(), cur = prev * nadam_u(beta1, t);
    s->push_back(cur);
    if (cur == prev && (cur == 0.0f || (beta1 >= 0.0f && beta1 <= 1.0f))) return B200PS_OK;
  }
  s->clear();
  return fail(B200PS_EINVAL, "Nadam: the momentum schedule of beta_1 = " + std::to_string(beta1) +
                                 " does not settle within " + std::to_string(kNadamMaxSteps) + " steps");
}

// Copies the host schedule to the client device, where k_push_begin reads it.
cudaError_t upload_nadam(b200ps_t* ps) {
  if (ps->opt.kind != kNadam) return cudaSuccess;
  const size_t bytes = ps->nadam_sched.size() * sizeof(float);
  cudaError_t e = cudaMalloc(&ps->d_nadam, bytes);
  if (e == cudaSuccess) e = cudaMemcpy(ps->d_nadam, ps->nadam_sched.data(), bytes, cudaMemcpyHostToDevice);
  return e;
}

GroupView group_view(b200ps_t* ps) {
  GroupView gv{};
  gv.tables = ps->d_tables;
  for (int s = 0; s < ps->n_shards; ++s) gv.ctl[s] = (ShardCtl*)ps->shard[s].ctl.ptr;
  gv.rt = ps->d_rt;
  gv.err = ps->d_err;
  gv.n_shards = ps->n_shards;
  gv.shard_shift = -1;
  if ((ps->n_shards & (ps->n_shards - 1)) == 0) {
    int sh = 0;
    while ((1 << sh) < ps->n_shards) ++sh;
    gv.shard_shift = sh;
  }
  return gv;
}

long long g_free_launches = 0;  // launches of the group-less primitives (ps == NULL)

int client_dev(b200ps_t* ps) {
  if (ps) return ps->client_device;
  int d = 0;
  cudaGetDevice(&d);
  return d;
}

void count_launch(b200ps_t* ps, int n) {
  if (ps) ps->launches += n; else g_free_launches += n;
}

int grid_for(b200ps_t* ps, long long work_items, int per_block = 256) {
  long long blocks = (work_items + per_block - 1) / per_block;
  long long cap = (long long)(ps ? ps->n_sm : 132) * 16;  // 16 CTAs of 256 threads per SM keep ~2 waves resident
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

int ready(b200ps_t* ps) {
  if (!ps) return fail(B200PS_EINVAL, "null group");
  for (int s = 0; s < ps->n_shards; ++s)
    if (!ps->shard[s].attached) return fail(B200PS_ESTATE, "shard " + std::to_string(s) + " is not attached");
  if (ps->dirty) return fail(B200PS_ESTATE, "b200ps_commit() not called after the last registration/import");
  if (ps->opt.kind < 0 || ps->opt.kind >= kNumOptKinds)  // parse_optimizer sets every kind; DISPATCH_OPT relies on it
    return fail(B200PS_EINVAL, "unknown optimizer kind " + std::to_string(ps->opt.kind));
  return B200PS_OK;
}

void fill_view(b200ps_t* ps, const Table& t, TableView* v) {
  memset(v, 0, sizeof(*v));
  for (int s = 0; s < ps->n_shards; ++s) {
    v->base[s] = t.alloc[s].ptr ? (float*)((char*)t.alloc[s].ptr + t.base_off) : nullptr;
    v->present[s] = (t.present_off && t.alloc[s].ptr) ? (uint32_t*)((char*)t.alloc[s].ptr + t.present_off) : nullptr;
    v->keys[s] = (t.hashed && t.alloc[s].ptr) ? (long long*)((char*)t.alloc[s].ptr + t.keys_off) : nullptr;
  }
  v->rows = t.rows;
  v->row_stride = t.row_stride;
  for (int k = 0; k <= kMaxSlots; ++k) v->slot_off[k] = t.slot_off[k];
  v->dim = t.dim;
  v->n_slots = t.n_slots;
  v->owner = t.owner;
  v->is_dense = t.is_dense;
}

int alloc_table_on_shard(b200ps_t* ps, Table& t, int s, int table_id) {
  Shard& sh = ps->shard[s];
  DeviceGuard g(sh.device);
  void* p = nullptr;
  CUDA_OK(cudaMalloc(&p, t.bytes));
  t.alloc[s].ptr = p;
  t.alloc[s].bytes = t.bytes;
  InitArgs a{};
  a.base = (float*)p;
  a.rows = t.rows;
  a.row_stride = t.row_stride;
  for (int k = 0; k <= kMaxSlots; ++k) { a.slot_off[k] = t.slot_off[k]; a.slot_init[k] = 0.f; }
  if (ps->opt.kind == kFTRL) a.slot_init[1] = ps->opt.init_accum;  // "accumulator" slot
  a.dim = t.dim;
  a.n_slots = t.n_slots;
  a.uniform = t.uniform;
  a.shard = s;
  a.n_shards = ps->n_shards;
  a.is_dense = t.is_dense;
  a.seed = t.seed;
  if (t.hashed) {
    // slot-keyed initial values: which id gets which draw depends on insertion order, exactly like the
    // reference's RandomUniform(seed = len(map)) (embedding_table.go:51-54) -- excluded from parity
    a.is_dense = 1;
    a.seed = t.seed ^ (0x9E3779B97F4A7C15ULL * (uint64_t)(s + 1));
  }
  // a pair's record section is [A(8) | B(1) | pad(3)]: A's and B's columns are initialised together as 9
  // columns, the pads are zeroed with the rest of the slab
  const bool pair = t.pair_b >= 0;
  if (pair) a.dim = 9;
  bool need_kernel = !t.raw && (t.uniform || (ps->opt.kind == kFTRL && ps->opt.init_accum != 0.0f));
  if (need_kernel) {
    if (pair) CUDA_OK(cudaMemsetAsync(p, 0, t.bytes, 0));
    else if (t.bytes > t.present_off && t.present_off) CUDA_OK(cudaMemsetAsync((char*)p + t.present_off, 0, t.bytes - t.present_off, 0));
    long long work = t.rows * (long long)a.dim * (t.n_slots + 1);
    k_init_rows<<<grid_for(ps, work), 256>>>(a);
    ps->launches++;
    CUDA_OK(cudaGetLastError());
  } else {
    CUDA_OK(cudaMemsetAsync(p, 0, t.bytes, 0));
  }
  if (t.hashed) {  // after the slab fill: every slot starts unclaimed
    k_fill_keys<<<grid_for(ps, t.rows), 256>>>((long long*)((char*)p + t.keys_off), t.rows);
    ps->launches++;
    CUDA_OK(cudaGetLastError());
  }
  CUDA_OK(cudaDeviceSynchronize());
  (void)table_id;
  return B200PS_OK;
}

// Direct-indexed tables and dense-parameter row views go through the flat kernels (ps_flat.cuh): one
// launch for all their segments whatever the dims.  Hashed tables (a probe per row) keep the
// per-segment kernels, split by vector class so that each launch is homogeneous:
// class 2: dim % 8 == 0 (32 B sector per thread), 1: dim % 4 == 0, 0: scalar.
bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

int legacy_class(const Table& t, const void* rows) {
  if (!aligned16(rows) || t.row_stride % 4 != 0) return 0;
  if (t.dim % 8 == 0) return 2;
  if (t.dim % 4 == 0) return 1;
  return 0;
}

constexpr int kClasses = 3;
struct Split {
  SegBatch b[kClasses];  // hashed tables / whole dense parameters
  long long max_work[kClasses] = {0, 0, 0};
  b200ps_seg_t flat[kMaxSegs];  // direct-indexed tables and dense row views: one flat launch
  unsigned char flat_vec[kMaxSegs];
  int flat_n = 0;
  long long flat_items = 0;  // upper bound of lane-items (device-side counts can only lower it)
};

int split_segs(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, bool want_dense, Split* out, bool push = false) {
  if (nseg < 0 || nseg > kMaxSegs) return fail(B200PS_EINVAL, "nseg out of range (max " + std::to_string(kMaxSegs) + ")");
  for (int c = 0; c < kClasses; ++c) out->b[c].nseg = 0;
  out->flat_n = 0;
  const bool flat_ok = ps->n_shards <= 8;  // the flat kernels carry <= 8 per-shard pointers per segment in their parameters
  for (int i = 0; i < nseg; ++i) {
    const b200ps_seg_t& sg = segs[i];
    if (sg.table < 0 || sg.table >= (int)ps->tables.size()) return fail(B200PS_ENOTFOUND, "unknown table id " + std::to_string(sg.table));
    const Table& t = ps->tables[sg.table];
    if (want_dense && !t.is_dense) return fail(B200PS_EINVAL, t.name + " is not a dense parameter");
    if (sg.n < 0) return fail(B200PS_EINVAL, "negative segment length");
    if (sg.n == 0 && !want_dense) continue;
    if (!want_dense && !t.hashed && flat_ok && t.row_stride < (1LL << 31)) {
      const int k = out->flat_n++;
      out->flat[k] = sg;
      const bool vec = !push && t.dim % 4 == 0 && t.row_stride % 4 == 0 && t.base_off % 16 == 0 && aligned16(sg.rows_dev);
      out->flat_vec[k] = vec ? 1 : 0;
      // a segment cannot hold more distinct rows than its table has
      const long long cap = t.is_dense ? t.rows : t.rows * ps->n_shards;
      out->flat_items += (sg.n < cap ? (long long)sg.n : cap) * (push ? t.dim : (vec ? t.dim / 4 : t.dim));
      continue;
    }
    int c;
    long long work;
    if (want_dense) {  // one launch for all of them: the kernels pick the 128-bit path per segment
      long long numel = t.rows * t.dim;
      c = 1;
      work = (numel % 4 == 0 && aligned16(sg.rows_dev)) ? numel / 4 : numel;
    } else {
      c = legacy_class(t, sg.rows_dev);
      int W = c == 0 ? 1 : 4 * c;
      work = (long long)sg.n * (t.dim / W);
    }
    SegBatch& b = out->b[c];
    b.seg[b.nseg++] = sg;
    if (work > out->max_work[c]) out->max_work[c] = work;
  }
  return B200PS_OK;
}

// Resolve the flat segments on the host: everything a row access needs travels in the kernel parameters.
template <int NSMAX>
void fill_flat(b200ps_t* ps, const Split& sp, bool push, int slot, FlatArgs<NSMAX>* a) {
  a->nseg = sp.flat_n;
  a->ns = ps->n_shards;
  a->shard_shift = -1;
  if ((ps->n_shards & (ps->n_shards - 1)) == 0) {
    int sh = 0;
    while ((1 << sh) < ps->n_shards) ++sh;
    a->shard_shift = sh;
  }
  a->slot = slot;
  a->rt = ps->d_rt;
  a->err = ps->d_err;
  for (int k = 0; k < sp.flat_n; ++k) {
    const b200ps_seg_t& sg = sp.flat[k];
    const Table& t = ps->tables[sg.table];
    FlatSegP& f = a->seg[k];
    f.ids = sg.ids_dev;
    f.n_dev = sg.n_dev;
    f.rows = sg.rows_dev;
    f.rows_cap = t.rows;
    for (int j = 0; j <= kMaxSlots; ++j) f.soff[j] = t.slot_off[j];
    f.n = sg.n;
    f.stride = (int)t.row_stride;
    f.dim = t.dim;
    f.vec = sp.flat_vec[k];
    f.lpr = push ? t.dim : (f.vec ? t.dim / 4 : t.dim);
    f.shift = (f.lpr & (f.lpr - 1)) == 0 ? (int)__builtin_ctz((unsigned)f.lpr) : -1;
    f.owner = t.owner;
    f.pad = 0;
    const int ns = NSMAX == 1 ? 1 : ps->n_shards;
    for (int s = 0; s < ns; ++s) {
      const Alloc& al = t.alloc[s];
      a->base[k * ns + s] = al.ptr ? (float*)((char*)al.ptr + t.base_off) : nullptr;
      a->present[k * ns + s] = (t.present_off && al.ptr) ? (uint32_t*)((char*)al.ptr + t.present_off) : nullptr;
    }
  }
}

template <typename F>
int for_each_class(b200ps_t* ps, Split& sp, F&& launch) {
  for (int c = 0; c < kClasses; ++c) {
    if (sp.b[c].nseg == 0) continue;
    // the cap on resident work applies to the whole launch, not to each segment: a segment's
    // blocks loop (grid-stride) instead of launching thousands of blocks that exit at once
    int gx = grid_for(ps, sp.max_work[c]);
    const int per_seg_cap = (ps->n_sm * 16 + sp.b[c].nseg - 1) / sp.b[c].nseg;
    if (gx > per_seg_cap) gx = per_seg_cap < 4 ? 4 : per_seg_cap;
    dim3 grid(gx, sp.b[c].nseg);
    launch(c, grid, sp.b[c]);
    ps->launches++;
    CUDA_OK(cudaGetLastError());
  }
  return B200PS_OK;
}

// Persistent grid of the flat kernels.  The grid must not exceed what is RESIDENT at once: a block that waits for
// a free slot starts after the first wave has finished and pays the block prologue (76 device-side counts ->
// scan -> barrier) and the launch ramp again.  Sized for 8 blocks per SM the 48-register kernels (5 resident)
// would run 1.6 waves, so the grid follows cudaOccupancyMaxActiveBlocksPerMultiprocessor of the kernel actually
// launched.
// U rows in flight per thread only once the work is several times what the resident threads cover.  (U = 4
// measured slower: its 80 registers cost more resident warps than the unroll adds.)
int flat_u(b200ps_t* ps, long long items) {
  const long long resident1 = (long long)ps->n_sm * 6 * 256;  // about what the U = 1 kernels keep resident
  return items >= resident1 * 8 ? 2 : 1;
}

// blocks of `kern` (256 threads, no dynamic shared memory) resident on the whole device
template <typename K>
int flat_grid(b200ps_t* ps, K kern, long long items, int U) {
  static std::mutex mu;
  static std::unordered_map<const void*, int> occ;
  std::lock_guard<std::mutex> lk(mu);
  auto it = occ.find((const void*)kern);
  if (it == occ.end()) {
    int v = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v, kern, 256, 0) != cudaSuccess || v < 1) v = 4;
    it = occ.emplace((const void*)kern, v).first;
  }
  const long long cap = (long long)ps->n_sm * it->second;
  long long blocks = (items + 256LL * U - 1) / (256LL * U);
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return (int)blocks;
}

#define DISPATCH_U(UVAL, ...)                          \
  switch (UVAL) {                                       \
    case 2: { constexpr int U = 2; __VA_ARGS__; } break; \
    default: { constexpr int U = 1; __VA_ARGS__; } break; \
  }

}  // namespace

// =============================================================================
extern "C" {

const char* b200ps_last_error(void) { return g_err.c_str(); }
int b200ps_abi_version(void) { return B200PS_ABI_VERSION; }

int b200ps_create(int n_shards, int client_device, const char* opt_type, const char* opt_args,
                  int lr_staleness_modulation, unsigned flags, b200ps_t** out) {
  if (!out) return fail(B200PS_EINVAL, "out is null");
  if (n_shards < 1 || n_shards > kMaxShards) return fail(B200PS_EINVAL, "n_shards must be in [1, 16]");
  OptParams o;
  int rc = parse_optimizer(opt_type, opt_args, &o);
  if (rc) return rc;
  std::vector<float> sched;
  if (o.kind == kNadam && (rc = nadam_schedule(o.beta1, &sched))) return rc;
  int ndev = 0;
  CUDA_OK(cudaGetDeviceCount(&ndev));
  if (client_device < 0 || client_device >= ndev) return fail(B200PS_ECUDA, "client device " + std::to_string(client_device) + " not present");
  b200ps_t* ps = new b200ps();
  ps->n_shards = n_shards;
  ps->client_device = client_device;
  ps->opt = o;
  ps->nadam_sched = std::move(sched);
  ps->staleness = lr_staleness_modulation;
  ps->flags = flags;
  DeviceGuard g(client_device);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, client_device) == cudaSuccess) ps->n_sm = prop.multiProcessorCount;
  // rows are 32 B sectors scattered over GBs: ask L2 not to over-fetch 64 B per miss (a hint)
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  cudaGetLastError();
  cudaError_t e = cudaMalloc(&ps->d_rt, sizeof(PushRt));
  if (e == cudaSuccess) e = cudaMemset(ps->d_rt, 0, sizeof(PushRt));
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_err, 64);
  if (e == cudaSuccess) e = cudaMemset(ps->d_err, 0, 64);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_versions, sizeof(int) * kMaxShards);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_count, 64);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_state, sizeof(long long) * 3 * kMaxShards);
  if (e == cudaSuccess) e = upload_nadam(ps);
  if (e != cudaSuccess) {
    delete ps;
    return fail(B200PS_ECUDA, std::string("b200ps_create: ") + cudaGetErrorString(e));
  }
  *out = ps;
  return B200PS_OK;
}

int b200ps_destroy(b200ps_t* ps) {
  if (!ps) return B200PS_OK;
  cudaSetDevice(ps->client_device);
  cudaDeviceSynchronize();
  for (auto& t : ps->tables)
    for (int s = 0; s < ps->n_shards; ++s) {
      if (!t.alloc[s].ptr || t.alloc[s].borrowed) continue;
      if (t.alloc[s].imported) cudaIpcCloseMemHandle(t.alloc[s].ptr);
      else { DeviceGuard g(ps->shard[s].device); cudaFree(t.alloc[s].ptr); }
    }
  for (int s = 0; s < ps->n_shards; ++s) {
    Alloc& a = ps->shard[s].ctl;
    if (!a.ptr || a.borrowed) continue;
    if (a.imported) cudaIpcCloseMemHandle(a.ptr);
    else { DeviceGuard g(ps->shard[s].device); cudaFree(a.ptr); }
  }
  cudaFree(ps->d_tables);
  cudaFree(ps->d_rt);
  cudaFree(ps->d_nadam);
  cudaFree(ps->d_err);
  cudaFree(ps->d_versions);
  cudaFree(ps->d_count);
  cudaFree(ps->d_state);
  if (ps->u_side) cudaStreamDestroy(ps->u_side);
  if (ps->u_fork) cudaEventDestroy(ps->u_fork);
  if (ps->u_join) cudaEventDestroy(ps->u_join);
  delete ps;
  return B200PS_OK;
}

int b200ps_clone_view(b200ps_t* src, int client_device, b200ps_t** out) {
  if (!src || !out) return fail(B200PS_EINVAL, "bad argument");
  for (int s = 0; s < src->n_shards; ++s)
    if (!src->shard[s].attached) return fail(B200PS_ESTATE, "source group has unattached shards");
  std::lock_guard<std::mutex> lk(src->mu);
  b200ps_t* ps = new b200ps();
  ps->n_shards = src->n_shards;
  ps->client_device = client_device;
  ps->opt = src->opt;
  ps->nadam_sched = src->nadam_sched;
  ps->staleness = src->staleness;
  ps->flags = src->flags;
  ps->n_sm = src->n_sm;
  for (int s = 0; s < src->n_shards; ++s) {
    ps->shard[s] = src->shard[s];
    ps->shard[s].local = false;  // memory stays owned by `src`
    ps->shard[s].ctl.borrowed = true;
  }
  ps->tables = src->tables;
  for (auto& t : ps->tables)
    for (int s = 0; s < src->n_shards; ++s) t.alloc[s].borrowed = true;
  ps->by_name = src->by_name;
  DeviceGuard g(client_device);
  if (client_device != src->client_device) {
    for (int s = 0; s < src->n_shards; ++s) {
      if (src->shard[s].device == client_device) continue;
      cudaError_t e = cudaDeviceEnablePeerAccess(src->shard[s].device, 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { delete ps; return fail(B200PS_ECUDA, cudaGetErrorString(e)); }
      cudaGetLastError();
    }
  }
  cudaError_t e = cudaMalloc(&ps->d_rt, sizeof(PushRt));
  if (e == cudaSuccess) e = cudaMemset(ps->d_rt, 0, sizeof(PushRt));
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_err, 64);
  if (e == cudaSuccess) e = cudaMemset(ps->d_err, 0, 64);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_versions, sizeof(int) * kMaxShards);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_count, 64);
  if (e == cudaSuccess) e = cudaMalloc(&ps->d_state, sizeof(long long) * 3 * kMaxShards);
  if (e == cudaSuccess) e = upload_nadam(ps);
  if (e != cudaSuccess) {
    delete ps;
    return fail(B200PS_ECUDA, std::string("b200ps_clone_view: ") + cudaGetErrorString(e));
  }
  ps->dirty = true;
  *out = ps;
  return B200PS_OK;
}

int b200ps_shard_create_local(b200ps_t* ps, int shard_id, int device) {
  if (!ps || shard_id < 0 || shard_id >= ps->n_shards) return fail(B200PS_EINVAL, "bad shard id");
  Shard& sh = ps->shard[shard_id];
  if (sh.attached) return fail(B200PS_ESTATE, "shard already attached");
  int ndev = 0;
  CUDA_OK(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(B200PS_ECUDA, "shard device not present");
  if (device != ps->client_device) {
    int can = 0;
    CUDA_OK(cudaDeviceCanAccessPeer(&can, ps->client_device, device));
    if (!can) return fail(B200PS_ECUDA, "no peer access from client device to shard device");
    DeviceGuard g(ps->client_device);
    cudaError_t e = cudaDeviceEnablePeerAccess(device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) CUDA_OK(e);
    cudaGetLastError();
  }
  DeviceGuard g(device);
  // a whole 2 MiB block: an IPC export then never exposes unrelated small allocations
  constexpr size_t kCtlBytes = 2u << 20;
  CUDA_OK(cudaMalloc(&sh.ctl.ptr, kCtlBytes));
  CUDA_OK(cudaMemset(sh.ctl.ptr, 0, kCtlBytes));
  sh.ctl.bytes = kCtlBytes;
  sh.local = true;
  sh.attached = true;
  sh.device = device;
  // tables registered before this shard existed
  for (size_t i = 0; i < ps->tables.size(); ++i) {
    Table& t = ps->tables[i];
    if (t.pair_of < 0 && (t.owner < 0 || t.owner == shard_id) && !t.alloc[shard_id].ptr) {
      int rc = alloc_table_on_shard(ps, t, shard_id, (int)i);
      if (rc) return rc;
    }
  }
  for (auto& t : ps->tables)
    if (t.pair_of >= 0 && !t.alloc[shard_id].ptr && ps->tables[t.pair_of].alloc[shard_id].ptr) {
      t.alloc[shard_id] = ps->tables[t.pair_of].alloc[shard_id];
      t.alloc[shard_id].borrowed = true;
    }
  ps->dirty = true;
  return B200PS_OK;
}

int b200ps_shard_export(b200ps_t* ps, int shard_id, void* blob, size_t cap, size_t* size) {
  if (!ps || shard_id < 0 || shard_id >= ps->n_shards || !size) return fail(B200PS_EINVAL, "bad argument");
  Shard& sh = ps->shard[shard_id];
  if (!sh.local) return fail(B200PS_ESTATE, "only a local shard can be exported");
  std::vector<BlobEntry> entries;
  DeviceGuard g(sh.device);
  BlobEntry ce{};
  ce.table = -1;
  ce.bytes = sh.ctl.bytes;
  CUDA_OK(cudaIpcGetMemHandle(&ce.handle, sh.ctl.ptr));
  entries.push_back(ce);
  for (size_t i = 0; i < ps->tables.size(); ++i) {
    Table& t = ps->tables[i];
    if (!t.alloc[shard_id].ptr || t.pair_of >= 0) continue;
    BlobEntry e{};
    e.table = (int)i;
    e.bytes = t.alloc[shard_id].bytes;
    CUDA_OK(cudaIpcGetMemHandle(&e.handle, t.alloc[shard_id].ptr));
    entries.push_back(e);
  }
  size_t need = sizeof(BlobHeader) + entries.size() * sizeof(BlobEntry);
  *size = need;
  if (!blob || cap < need) return blob ? fail(B200PS_EINVAL, "blob buffer too small") : B200PS_OK;
  BlobHeader h{kBlobMagic, shard_id, (int)entries.size(), 0};
  memcpy(blob, &h, sizeof(h));
  memcpy((char*)blob + sizeof(h), entries.data(), entries.size() * sizeof(BlobEntry));
  return B200PS_OK;
}

int b200ps_shard_import(b200ps_t* ps, int shard_id, const void* blob, size_t size) {
  if (!ps || shard_id < 0 || shard_id >= ps->n_shards || !blob || size < sizeof(BlobHeader)) return fail(B200PS_EINVAL, "bad argument");
  Shard& sh = ps->shard[shard_id];
  if (sh.local) return fail(B200PS_ESTATE, "shard is local to this process");
  BlobHeader h;
  memcpy(&h, blob, sizeof(h));
  if (h.magic != kBlobMagic || h.shard != shard_id) return fail(B200PS_EINVAL, "blob does not describe this shard");
  if (size < sizeof(h) + (size_t)h.n_entries * sizeof(BlobEntry)) return fail(B200PS_EINVAL, "truncated blob");
  DeviceGuard g(ps->client_device);
  const BlobEntry* e = (const BlobEntry*)((const char*)blob + sizeof(h));
  for (int i = 0; i < h.n_entries; ++i) {
    Alloc* a = nullptr;
    if (e[i].table < 0) a = &sh.ctl;
    else {
      if (e[i].table >= (int)ps->tables.size()) return fail(B200PS_ESTATE, "peer registered a table this process has not (register on every process first)");
      a = &ps->tables[e[i].table].alloc[shard_id];
    }
    if (a->ptr) continue;  // already mapped
    void* p = nullptr;
    CUDA_OK(cudaIpcOpenMemHandle(&p, e[i].handle, cudaIpcMemLazyEnablePeerAccess));
    a->ptr = p;
    a->bytes = e[i].bytes;
    a->imported = true;
  }
  for (auto& t : ps->tables)  // a pair's second table aliases the first one's mapping
    if (t.pair_of >= 0 && !t.alloc[shard_id].ptr && ps->tables[t.pair_of].alloc[shard_id].ptr) {
      t.alloc[shard_id] = ps->tables[t.pair_of].alloc[shard_id];
      t.alloc[shard_id].borrowed = true;
    }
  sh.attached = true;
  ps->dirty = true;
  return B200PS_OK;
}

int b200ps_lookup(b200ps_t* ps, const char* name) {
  if (!ps || !name) return fail(B200PS_EINVAL, "bad argument");
  auto it = ps->by_name.find(name);
  if (it == ps->by_name.end()) return fail(B200PS_ENOTFOUND, std::string(name) + " not in Parameter");
  return it->second;
}

static bool is_borrowed_view(b200ps_t* ps) {
  for (int s = 0; s < ps->n_shards; ++s)
    if (ps->shard[s].ctl.borrowed) return true;
  return false;
}

static int register_common(b200ps_t* ps, Table&& t) {
  if (is_borrowed_view(ps)) return fail(B200PS_ESTATE, "tables are registered on the owning group, then b200ps_clone_view again");
  t.n_slots = opt_slots(ps->opt.kind);
  int id = (int)ps->tables.size();
  ps->tables.push_back(std::move(t));
  Table& tt = ps->tables.back();
  ps->by_name[tt.name] = id;
  for (int s = 0; s < ps->n_shards; ++s) {
    if (!ps->shard[s].local) continue;
    if (tt.owner >= 0 && tt.owner != s) continue;
    int rc = alloc_table_on_shard(ps, tt, s, id);
    if (rc) return rc;
  }
  ps->dirty = true;
  return id;
}

int b200ps_table_register(b200ps_t* ps, const char* name, int dim, const char* initializer, int64_t capacity,
                          uint64_t seed) {
  if (!ps || !name || dim < 1 || capacity < 1) return fail(B200PS_EINVAL, "bad table definition");
  std::lock_guard<std::mutex> lk(ps->mu);
  auto it = ps->by_name.find(name);
  if (it != ps->by_name.end()) return it->second;  // model.go:57-63 idempotent
  Table t;
  t.name = name;
  t.dim = dim;
  t.owner = -1;
  t.is_dense = false;
  t.rows = (capacity + ps->n_shards - 1) / ps->n_shards;
  int slots = opt_slots(ps->opt.kind);
  int64_t rec = (int64_t)dim * (slots + 1);
  rec = (rec + 3) / 4 * 4;  // 16 B aligned records
  t.row_stride = rec;
  for (int k = 0; k <= kMaxSlots; ++k) t.slot_off[k] = (int64_t)k * dim;
  size_t rec_bytes = (size_t)t.rows * rec * sizeof(float);
  rec_bytes = (rec_bytes + 255) / 256 * 256;
  size_t bitmap = (ps->flags & 2u) ? 0 : (((size_t)t.rows + 31) / 32 * 4 + 255) / 256 * 256;
  t.present_off = bitmap ? rec_bytes : 0;
  t.bytes = (rec_bytes + bitmap + (2u << 20) - 1) / (2u << 20) * (2u << 20);  // IPC-exportable whole blocks
  t.uniform = initializer && strcmp(initializer, "uniform") == 0;  // embedding_table.go:51 (quirk Q6)
  t.seed = seed;
  return register_common(ps, std::move(t));
}

int b200ps_table_register_pair(b200ps_t* ps, const char* name_a, const char* name_b, const char* initializer,
                               int64_t capacity, uint64_t seed) {
  if (!ps || !name_a || !name_b || capacity < 1) return fail(B200PS_EINVAL, "bad table definition");
  std::lock_guard<std::mutex> lk(ps->mu);
  auto ia = ps->by_name.find(name_a), ib = ps->by_name.find(name_b);
  if (ia != ps->by_name.end() && ib != ps->by_name.end()) return ia->second;
  if (ia != ps->by_name.end() || ib != ps->by_name.end()) return fail(B200PS_ESTATE, "one table of the pair is already registered");
  const int slots = opt_slots(ps->opt.kind);
  const int64_t sec = 12;  // [A(8) | B(1) | pad(3)] floats
  Table a;
  a.name = name_a;
  a.dim = 8;
  a.owner = -1;
  a.rows = (capacity + ps->n_shards - 1) / ps->n_shards;
  a.row_stride = sec * (slots + 1);
  for (int k = 0; k <= kMaxSlots; ++k) a.slot_off[k] = (int64_t)k * sec;
  size_t rec_bytes = ((size_t)a.rows * a.row_stride * sizeof(float) + 255) / 256 * 256;
  size_t bitmap = (ps->flags & 2u) ? 0 : (((size_t)a.rows + 31) / 32 * 4 + 255) / 256 * 256;
  a.present_off = bitmap ? rec_bytes : 0;
  a.bytes = (rec_bytes + 2 * bitmap + (2u << 20) - 1) / (2u << 20) * (2u << 20);
  a.uniform = initializer && strcmp(initializer, "uniform") == 0;
  a.seed = seed;
  a.pair_b = (int)ps->tables.size() + 1;
  if (a.uniform) return fail(B200PS_EINVAL, "paired tables support the zero initializer only (set rows explicitly)");
  int id_a = register_common(ps, std::move(a));
  if (id_a < 0) return id_a;
  Table b;
  b.name = name_b;
  b.dim = 1;
  b.owner = -1;
  const Table& ra = ps->tables[id_a];
  b.rows = ra.rows;
  b.row_stride = ra.row_stride;
  for (int k = 0; k <= kMaxSlots; ++k) b.slot_off[k] = (int64_t)k * sec;
  b.base_off = 8 * sizeof(float);
  b.present_off = bitmap ? rec_bytes + bitmap : 0;
  b.bytes = ra.bytes;
  b.n_slots = ra.n_slots;
  b.pair_of = id_a;
  for (int s = 0; s < ps->n_shards; ++s) {  // shares A's allocation
    b.alloc[s] = ra.alloc[s];
    b.alloc[s].borrowed = true;
  }
  int id_b = (int)ps->tables.size();
  ps->tables.push_back(std::move(b));
  ps->by_name[name_b] = id_b;
  ps->dirty = true;
  return id_a;
}

int b200ps_table_register_hashed(b200ps_t* ps, const char* name, int dim, const char* initializer,
                                 int64_t expected_rows, uint64_t seed) {
  if (!ps || !name || dim < 1 || expected_rows < 1) return fail(B200PS_EINVAL, "bad table definition");
  std::lock_guard<std::mutex> lk(ps->mu);
  auto it = ps->by_name.find(name);
  if (it != ps->by_name.end()) return it->second;
  Table t;
  t.name = name;
  t.dim = dim;
  t.owner = -1;
  t.is_dense = false;
  t.hashed = true;
  int64_t per_shard = (expected_rows + ps->n_shards - 1) / ps->n_shards;
  int64_t slots = 1024;
  while (slots < 2 * per_shard) slots <<= 1;  // load factor <= 0.5
  t.rows = slots;
  int slots_n = opt_slots(ps->opt.kind);
  int64_t rec = (int64_t)dim * (slots_n + 1);
  rec = (rec + 3) / 4 * 4;
  t.row_stride = rec;
  for (int k = 0; k <= kMaxSlots; ++k) t.slot_off[k] = (int64_t)k * dim;
  size_t rec_bytes = ((size_t)t.rows * rec * sizeof(float) + 255) / 256 * 256;
  t.present_off = 0;  // the key array is the created-row record
  t.keys_off = rec_bytes;
  t.bytes = (rec_bytes + (size_t)t.rows * sizeof(long long) + (2u << 20) - 1) / (2u << 20) * (2u << 20);
  t.uniform = initializer && strcmp(initializer, "uniform") == 0;
  t.seed = seed;
  return register_common(ps, std::move(t));
}

int b200ps_dense_register(b200ps_t* ps, const char* name, int shard, int64_t rows, int dim) {
  if (!ps || !name || dim < 1 || rows < 1 || shard < 0 || shard >= ps->n_shards) return fail(B200PS_EINVAL, "bad dense parameter definition");
  std::lock_guard<std::mutex> lk(ps->mu);
  auto it = ps->by_name.find(name);
  if (it != ps->by_name.end()) return it->second;
  Table t;
  t.name = name;
  t.dim = dim;
  t.owner = shard;
  t.is_dense = true;
  t.rows = rows;
  t.row_stride = dim;
  int64_t numel = rows * dim;
  int64_t padded = (numel + 63) / 64 * 64;  // every slot array starts 256 B aligned
  for (int k = 0; k <= kMaxSlots; ++k) t.slot_off[k] = (int64_t)k * padded;
  int slots = opt_slots(ps->opt.kind);
  t.present_off = 0;
  t.bytes = ((size_t)padded * (slots + 1) * sizeof(float) + (2u << 20) - 1) / (2u << 20) * (2u << 20);
  t.uniform = false;
  return register_common(ps, std::move(t));
}

int b200ps_commit(b200ps_t* ps) {
  if (!ps) return fail(B200PS_EINVAL, "null group");
  std::lock_guard<std::mutex> lk(ps->mu);
  DeviceGuard g(ps->client_device);
  int n = (int)ps->tables.size();
  if (n > ps->d_tables_cap) {
    // the old directory may still be read by in-flight kernels
    CUDA_OK(cudaDeviceSynchronize());
    cudaFree(ps->d_tables);
    int cap = n < 64 ? 64 : n * 2;
    CUDA_OK(cudaMalloc(&ps->d_tables, sizeof(TableView) * cap));
    ps->d_tables_cap = cap;
  }
  if (n) {
    std::vector<TableView> host(n);
    for (int i = 0; i < n; ++i) fill_view(ps, ps->tables[i], &host[i]);
    CUDA_OK(cudaMemcpy(ps->d_tables, host.data(), sizeof(TableView) * n, cudaMemcpyHostToDevice));
  }
  ps->dirty = false;
  return B200PS_OK;
}

// ---- data path ---------------------------------------------------------------

static int rows_copy(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream, bool write, int slot = 0) {
  int rc = ready(ps);
  if (rc) return rc;
  if (slot < 0 || slot > opt_slots(ps->opt.kind)) return fail(B200PS_EINVAL, "optimizer has no such slot");
  DeviceGuard g(ps->client_device);
  Split sp;
  rc = split_segs(ps, segs, nseg, false, &sp);
  if (rc) return rc;
  GroupView gv = group_view(ps);
  cudaStream_t st = (cudaStream_t)stream;
  if (sp.flat_n) {
    const int u_rt = flat_u(ps, sp.flat_items);
    int grid;
    if (ps->n_shards == 1) {
      FlatArgs<1> fa;
      fill_flat(ps, sp, false, slot, &fa);
      DISPATCH_U(u_rt, {
        if (write) { grid = flat_grid(ps, k_copy_flat<true, U, 1>, sp.flat_items, U); k_copy_flat<true, U, 1><<<grid, 256, 0, st>>>(fa); }
        else { grid = flat_grid(ps, k_copy_flat<false, U, 1>, sp.flat_items, U); k_copy_flat<false, U, 1><<<grid, 256, 0, st>>>(fa); }
      });
    } else {
      FlatArgs<8> fa;
      fill_flat(ps, sp, false, slot, &fa);
      DISPATCH_U(u_rt, {
        if (write) { grid = flat_grid(ps, k_copy_flat<true, U, 8>, sp.flat_items, U); k_copy_flat<true, U, 8><<<grid, 256, 0, st>>>(fa); }
        else { grid = flat_grid(ps, k_copy_flat<false, U, 8>, sp.flat_items, U); k_copy_flat<false, U, 8><<<grid, 256, 0, st>>>(fa); }
      });
    }
    ps->launches++;
    CUDA_OK(cudaGetLastError());
  }
  return for_each_class(ps, sp, [&](int c, dim3 grid, const SegBatch& b) {
    if (write) {
      if (c == 2) k_rows_copy<2, true><<<grid, 256, 0, st>>>(gv, b, slot);
      else if (c == 1) k_rows_copy<1, true><<<grid, 256, 0, st>>>(gv, b, slot);
      else k_rows_copy<0, true><<<grid, 256, 0, st>>>(gv, b, slot);
    } else {
      if (c == 2) k_rows_copy<2, false><<<grid, 256, 0, st>>>(gv, b, slot);
      else if (c == 1) k_rows_copy<1, false><<<grid, 256, 0, st>>>(gv, b, slot);
      else k_rows_copy<0, false><<<grid, 256, 0, st>>>(gv, b, slot);
    }
  });
}

int b200ps_pull_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  return rows_copy(ps, segs, nseg, stream, false);
}
int b200ps_set_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  return rows_copy(ps, segs, nseg, stream, true);
}

static int dense_copy(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream, bool write, int slot = 0) {
  int rc = ready(ps);
  if (rc) return rc;
  if (slot < 0 || slot > opt_slots(ps->opt.kind)) return fail(B200PS_EINVAL, "optimizer has no such slot");
  DeviceGuard g(ps->client_device);
  Split sp;
  rc = split_segs(ps, segs, nseg, true, &sp);
  if (rc) return rc;
  GroupView gv = group_view(ps);
  cudaStream_t st = (cudaStream_t)stream;
  return for_each_class(ps, sp, [&](int, dim3 grid, const SegBatch& b) {
    if (write) k_dense_copy<true><<<grid, 256, 0, st>>>(gv, b, slot);
    else k_dense_copy<false><<<grid, 256, 0, st>>>(gv, b, slot);
  });
}

int b200ps_pull_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  return dense_copy(ps, segs, nseg, stream, false);
}
int b200ps_set_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  return dense_copy(ps, segs, nseg, stream, true);
}

int b200ps_slot_rows(b200ps_t* ps, int slot, int write, const b200ps_seg_t* segs, int nseg, void* stream) {
  return rows_copy(ps, segs, nseg, stream, write != 0, slot);
}
int b200ps_slot_dense(b200ps_t* ps, int slot, int write, const b200ps_seg_t* segs, int nseg, void* stream) {
  return dense_copy(ps, segs, nseg, stream, write != 0, slot);
}

static int push_begin_impl(b200ps_t* ps, float lr, const int32_t* mv, void* stream, int bump_only, int only_shard = -1) {
  int rc = ready(ps);
  if (rc) return rc;
  if (only_shard >= ps->n_shards) return fail(B200PS_EINVAL, "bad shard id");
  DeviceGuard g(ps->client_device);
  VersionsIn v{};
  for (int s = 0; s < ps->n_shards; ++s) v.v[s] = mv ? mv[s] : 0;
  k_push_begin<<<1, 32, 0, (cudaStream_t)stream>>>(group_view(ps), ps->opt, lr, v, ps->staleness, bump_only, only_shard,
                                                    ps->d_nadam, (long long)ps->nadam_sched.size() - 1);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_push_begin(b200ps_t* ps, float learning_rate, const int32_t* model_versions, void* stream) {
  return push_begin_impl(ps, learning_rate, model_versions, stream, 0);
}
int b200ps_bump_step(b200ps_t* ps, void* stream) { return push_begin_impl(ps, 0.f, nullptr, stream, 1); }
int b200ps_push_begin_shard(b200ps_t* ps, int shard, float learning_rate, const int32_t* model_versions, void* stream) {
  if (shard < 0) return fail(B200PS_EINVAL, "bad shard id");
  return push_begin_impl(ps, learning_rate, model_versions, stream, 0, shard);
}

#define DISPATCH_OPT(KIND, ...)                        \
  switch (KIND) {                                       \
    case kSGD: { constexpr int OPT = kSGD; __VA_ARGS__; } break;           \
    case kMomentum: { constexpr int OPT = kMomentum; __VA_ARGS__; } break; \
    case kAdam: { constexpr int OPT = kAdam; __VA_ARGS__; } break;         \
    case kAMSGrad: { constexpr int OPT = kAMSGrad; __VA_ARGS__; } break;   \
    case kAdagrad: { constexpr int OPT = kAdagrad; __VA_ARGS__; } break;   \
    case kFTRL: { constexpr int OPT = kFTRL; __VA_ARGS__; } break;         \
    case kRMSprop: { constexpr int OPT = kRMSprop; __VA_ARGS__; } break;   \
    case kRMSpropMomentum: { constexpr int OPT = kRMSpropMomentum; __VA_ARGS__; } break;                 \
    case kRMSpropCentered: { constexpr int OPT = kRMSpropCentered; __VA_ARGS__; } break;                 \
    case kRMSpropCenteredMomentum: { constexpr int OPT = kRMSpropCenteredMomentum; __VA_ARGS__; } break; \
    case kAdadelta: { constexpr int OPT = kAdadelta; __VA_ARGS__; } break; \
    case kAdamax: { constexpr int OPT = kAdamax; __VA_ARGS__; } break;     \
    case kNadam: { constexpr int OPT = kNadam; __VA_ARGS__; } break;       \
    default: break;  /* unreachable: ready() refuses any other kind before a push dispatches */         \
  }
static_assert(kNumOptKinds == 13, "DISPATCH_OPT has one case per OptKind");

int b200ps_push_rows(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  Split sp;
  rc = split_segs(ps, segs, nseg, false, &sp, true);
  if (rc) return rc;
  GroupView gv = group_view(ps);
  cudaStream_t st = (cudaStream_t)stream;
  OptParams o = ps->opt;
  if (sp.flat_n) {
    const int u_rt = flat_u(ps, sp.flat_items);
    int grid;
    if (ps->n_shards == 1) {
      FlatArgs<1> fa;
      fill_flat(ps, sp, true, 0, &fa);
      DISPATCH_OPT(o.kind, DISPATCH_U(u_rt, {
        grid = flat_grid(ps, k_push_flat<OPT, U, 1>, sp.flat_items, U);
        k_push_flat<OPT, U, 1><<<grid, 256, 0, st>>>(fa, o);
      }));
    } else {
      FlatArgs<8> fa;
      fill_flat(ps, sp, true, 0, &fa);
      DISPATCH_OPT(o.kind, DISPATCH_U(u_rt, {
        grid = flat_grid(ps, k_push_flat<OPT, U, 8>, sp.flat_items, U);
        k_push_flat<OPT, U, 8><<<grid, 256, 0, st>>>(fa, o);
      }));
    }
    ps->launches++;
    CUDA_OK(cudaGetLastError());
  }
  return for_each_class(ps, sp, [&](int c, dim3 grid, const SegBatch& b) {
    DISPATCH_OPT(o.kind, {
      if (c == 2) k_push_rows<OPT, 2><<<grid, 256, 0, st>>>(gv, b, o);
      else if (c == 1) k_push_rows<OPT, 1><<<grid, 256, 0, st>>>(gv, b, o);
      else k_push_rows<OPT, 0><<<grid, 256, 0, st>>>(gv, b, o);
    });
  });
}

static int pair_batch(b200ps_t* ps, const b200ps_seg_t* segs_a, float* const* rows_b, int nseg, PairBatch* pb,
                      long long* max_n) {
  if (nseg < 1 || nseg > kMaxSegs / 2) return fail(B200PS_EINVAL, "pair launches take 1.." + std::to_string(kMaxSegs / 2) + " segments");
  *max_n = 0;
  for (int i = 0; i < nseg; ++i) {
    const b200ps_seg_t& sg = segs_a[i];
    if (sg.table < 0 || sg.table >= (int)ps->tables.size() || ps->tables[sg.table].pair_b < 0)
      return fail(B200PS_EINVAL, "segment table is not the first table of a registered pair");
    if (!aligned16(sg.rows_dev) || !rows_b[i]) return fail(B200PS_EINVAL, "pair rows must be 16 B aligned / non-null");
    pb->a[i] = sg;
    pb->rows_b[i] = rows_b[i];
    pb->table_b[i] = ps->tables[sg.table].pair_b;
    if (sg.n > *max_n) *max_n = sg.n;
  }
  pb->nseg = nseg;
  return B200PS_OK;
}

static dim3 pair_grid(b200ps_t* ps, long long threads, int nseg) {
  int gx = grid_for(ps, threads);
  const int per_seg_cap = (ps->n_sm * 16 + nseg - 1) / nseg;
  if (gx > per_seg_cap) gx = per_seg_cap < 4 ? 4 : per_seg_cap;
  return dim3(gx, nseg);
}

int b200ps_pull_rows_pair(b200ps_t* ps, const b200ps_seg_t* segs_a, float* const* rows_b, int nseg, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  PairBatch pb;
  long long max_n;
  rc = pair_batch(ps, segs_a, rows_b, nseg, &pb, &max_n);
  if (rc) return rc;
  k_pair_pull<<<pair_grid(ps, max_n * 4, nseg), 256, 0, (cudaStream_t)stream>>>(group_view(ps), pb);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_push_rows_pair(b200ps_t* ps, const b200ps_seg_t* segs_a, float* const* grads_b, int nseg, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  PairBatch pb;
  long long max_n;
  rc = pair_batch(ps, segs_a, grads_b, nseg, &pb, &max_n);
  if (rc) return rc;
  GroupView gv = group_view(ps);
  OptParams o = ps->opt;
  const int S = opt_slots(o.kind);
  const int lpr = 3 * (1 + S) <= 4 ? 4 : 3 * (1 + S) <= 8 ? 8 : 16;
  dim3 grid = pair_grid(ps, max_n * lpr, nseg);
  cudaStream_t st = (cudaStream_t)stream;
  DISPATCH_OPT(o.kind, k_pair_push<OPT><<<grid, 256, 0, st>>>(gv, pb, o));
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

// ---- owner-computes exchange (ps_exchange.cuh) ----------------------------------
int b200ps_xchg_create(b200ps_t* ps, int G, int B, const int32_t* deep_tables, const int32_t* wide_tables) {
  if (!ps || B < 1 || !deep_tables || !wide_tables) return fail(B200PS_EINVAL, "bad exchange definition");
  if (G < 1 || G > kXMaxG) return fail(B200PS_EINVAL, "the exchange moves 1 to " + std::to_string(kXMaxG) + " table pairs");
  if (ps->x_table >= 0) return fail(B200PS_ESTATE, "exchange already created");
  int me = -1, n_local = 0;
  for (int s = 0; s < ps->n_shards; ++s)
    if (ps->shard[s].local) { me = s; ++n_local; }
  if (n_local != 1) return fail(B200PS_ESTATE, "the exchange needs exactly one local shard per process (rank-per-GPU)");
  // the owner-side constants of every pair on my shard: the exchange kernels take them instead of the table directory
  XTabs xt{};
  xt.shard_shift = group_view(ps).shard_shift;
  for (int g = 0; g < G; ++g) {
    if (deep_tables[g] < 0 || deep_tables[g] >= (int)ps->tables.size() || wide_tables[g] < 0 ||
        wide_tables[g] >= (int)ps->tables.size())
      return fail(B200PS_ENOTFOUND, "unknown table id in exchange definition");
    const Table& d = ps->tables[deep_tables[g]];
    const Table& w = ps->tables[wide_tables[g]];
    if (d.dim != 8 || w.dim != 1) return fail(B200PS_EWIDTH, "the exchange moves dim-8 / dim-1 table pairs");
    if (d.hashed || w.hashed || d.is_dense || w.is_dense || d.owner >= 0 || w.owner >= 0 || d.raw || w.raw)
      return fail(B200PS_EINVAL, "the exchange moves direct-indexed tables striped over every shard "
                                 "(not hashed, dense, pinned to one shard or raw)");
    for (int j = 0; j <= kMaxSlots; ++j) {
      if (g == 0) {
        xt.deep_soff[j] = (int)d.slot_off[j];
        xt.wide_soff[j] = (int)w.slot_off[j];
      } else if (xt.deep_soff[j] != (int)d.slot_off[j] || xt.wide_soff[j] != (int)w.slot_off[j]) {
        return fail(B200PS_EINVAL, "the exchanged deep tables, and the wide tables, need one slot layout each");
      }
    }
    if (!d.alloc[me].ptr || !w.alloc[me].ptr) return fail(B200PS_ESTATE, "an exchanged table is not allocated on the local shard");
    xt.deep[g] = (float*)((char*)d.alloc[me].ptr + d.base_off);
    xt.wide[g] = (float*)((char*)w.alloc[me].ptr + w.base_off);
    xt.deep_pres[g] = d.present_off ? (uint32_t*)((char*)d.alloc[me].ptr + d.present_off) : nullptr;
    xt.wide_pres[g] = w.present_off ? (uint32_t*)((char*)w.alloc[me].ptr + w.present_off) : nullptr;
    xt.deep_rows[g] = d.rows;
    xt.wide_rows[g] = w.rows;
    xt.deep_stride[g] = (int)d.row_stride;
    xt.wide_stride[g] = (int)w.row_stride;
  }
  ps->x_G = G;
  ps->x_B = B;
  ps->x_me = me;
  ps->x_cap = (long long)G * B;
  const long long n = ps->n_shards;
  ps->x_off_ids = 4096;
  ps->x_off_resp = ps->x_off_ids + n * ps->x_cap * kXIdEntry;  // one id bucket per owner
  ps->x_off_upd = ps->x_off_resp + n * ps->x_cap * kXResp;
  ps->x_off_served = ps->x_off_upd + n * ps->x_cap * kXUpd;
  const long long bytes = ps->x_off_served + n * ps->x_cap * kXServed;
  static_assert(sizeof(XHeader) <= 4096, "exchange header must fit its page");
  {
    std::lock_guard<std::mutex> lk(ps->mu);
    Table t;
    t.name = "__xchg__";
    t.dim = 1;
    t.owner = -1;
    t.raw = true;
    t.rows = bytes / 4;
    t.row_stride = 1;
    t.bytes = ((size_t)bytes + (2u << 20) - 1) / (2u << 20) * (2u << 20);
    int id = register_common(ps, std::move(t));
    if (id < 0) return id;
    ps->x_table = id;
  }
  ps->x_tabs = xt;  // stays valid: a table's allocation on its shard lives as long as the group
  return B200PS_OK;
}

static int xview(b200ps_t* ps, XView* x) {
  int rc = ready(ps);
  if (rc) return rc;
  if (ps->x_table < 0) return fail(B200PS_ESTATE, "b200ps_xchg_create not called");
  const Table& t = ps->tables[ps->x_table];
  for (int s = 0; s < ps->n_shards; ++s) {
    if (!t.alloc[s].ptr) return fail(B200PS_ESTATE, "exchange buffer of shard " + std::to_string(s) + " is not mapped (sync peers)");
    x->buf[s] = (char*)t.alloc[s].ptr;
  }
  x->off_ids = ps->x_off_ids;
  x->off_resp = ps->x_off_resp;
  x->off_upd = ps->x_off_upd;
  x->off_served = ps->x_off_served;
  x->cap = ps->x_cap;
  x->n = ps->n_shards;
  x->me = ps->x_me;
  x->G = ps->x_G;
  x->B = ps->x_B;
  return B200PS_OK;
}

// grid.x per peer: 4 blocks per SM over all peers
static int xchg_per_peer(b200ps_t* ps) {
  const int v = ps->n_sm * 4 / ps->n_shards;
  return v < 2 ? 2 : v;
}

// The pull's three kernels (post, serve, unscatter) and the push's three (send_upd, apply, wait_applied) on `st`;
// with `ev`, ev[i] is recorded after the i-th kernel.
static void xchg_pull_kernels(b200ps_t* ps, const XView& x, const int64_t* uniq_dev, const int32_t* n_unique_dev,
                              float* bet_deep_dev, float* bet_wide_dev, cudaStream_t st, cudaEvent_t* ev = nullptr) {
  dim3 grid(xchg_per_peer(ps), ps->n_shards);
  k_x_post<<<ps->n_sm, 256, 0, st>>>(x, uniq_dev, n_unique_dev);
  if (ev) cudaEventRecord(ev[0], st);
  k_x_serve<4><<<grid, 256, 0, st>>>(x, ps->x_tabs, ps->d_err);
  if (ev) cudaEventRecord(ev[1], st);
  k_x_unscatter<4><<<grid, 256, 0, st>>>(x, ps->d_err, bet_deep_dev, bet_wide_dev);
  if (ev) cudaEventRecord(ev[2], st);
  ps->launches += 3;
}

static void xchg_push_kernels(b200ps_t* ps, const XView& x, const float* gsum_deep_dev, const float* gsum_wide_dev,
                              cudaStream_t st, cudaEvent_t* ev = nullptr) {
  const OptParams o = ps->opt;
  dim3 grid(xchg_per_peer(ps), ps->n_shards);
  k_x_send_upd<4><<<grid, 256, 0, st>>>(x, ps->d_rt, gsum_deep_dev, gsum_wide_dev);
  if (ev) cudaEventRecord(ev[0], st);
  // one apply launch per source, in rank order: a row that several ranks pushed this step gets every rank's
  // update, as if the ranks had pushed one after the other (concurrent sources would race on the record's
  // read-modify-write and lose updates or tear the record).
  // The apply kernel holds 80 registers: 3 blocks per SM are resident, a 4th would wait for a second wave
  const unsigned grid_apply = (unsigned)ps->n_sm * 3;
  for (int src = 0; src < ps->n_shards; ++src)
    DISPATCH_OPT(o.kind, k_x_apply<OPT, 2><<<grid_apply, 256, 0, st>>>(x, ps->x_tabs, ps->d_err, o, src));
  if (ev) cudaEventRecord(ev[1], st);
  k_x_wait_applied<<<1, 32, 0, st>>>(x, ps->d_err);
  if (ev) cudaEventRecord(ev[2], st);
  ps->launches += 2 + ps->n_shards;
}

int b200ps_xchg_pull(b200ps_t* ps, const int64_t* uniq_dev, const int32_t* n_unique_dev, float* bet_deep_dev,
                     float* bet_wide_dev, void* stream) {
  XView x;
  int rc = xview(ps, &x);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  xchg_pull_kernels(ps, x, uniq_dev, n_unique_dev, bet_deep_dev, bet_wide_dev, (cudaStream_t)stream);
  ps->x_pulled = true;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_xchg_push(b200ps_t* ps, const float* gsum_deep_dev, const float* gsum_wide_dev, void* stream) {
  XView x;
  int rc = xview(ps, &x);
  if (rc) return rc;
  if (!ps->x_pulled) return fail(B200PS_ESTATE, "b200ps_xchg_push follows the b200ps_xchg_pull of the same id lists");
  ps->x_pulled = false;
  DeviceGuard g(ps->client_device);
  xchg_push_kernels(ps, x, gsum_deep_dev, gsum_wide_dev, (cudaStream_t)stream);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

// Debug / profiling: one pull + one push with a CUDA event after every kernel; synchronous.
// ms_out[0..5] = post, serve, unscatter | send_upd, apply, wait_applied.
int b200ps_xchg_profile(b200ps_t* ps, const int64_t* uniq_dev, const int32_t* n_unique_dev, float* bet_deep_dev,
                        float* bet_wide_dev, const float* gsum_deep_dev, const float* gsum_wide_dev, float* ms_out,
                        void* stream) {
  XView x;
  int rc = xview(ps, &x);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  cudaStream_t st = (cudaStream_t)stream;
  cudaEvent_t ev[7];
  for (auto& e : ev) CUDA_OK(cudaEventCreate(&e));
  cudaEventRecord(ev[0], st);
  xchg_pull_kernels(ps, x, uniq_dev, n_unique_dev, bet_deep_dev, bet_wide_dev, st, ev + 1);
  xchg_push_kernels(ps, x, gsum_deep_dev, gsum_wide_dev, st, ev + 4);
  CUDA_OK(cudaStreamSynchronize(st));
  for (int i = 0; i < 6; ++i) cudaEventElapsedTime(&ms_out[i], ev[i], ev[i + 1]);
  for (auto& e : ev) cudaEventDestroy(e);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

// ---- raw peer-visible buffers + device-side barrier (the allreduce controller's data path) ----
int b200ps_raw_register(b200ps_t* ps, const char* name, size_t bytes) {
  if (!ps || !name || bytes < 1) return fail(B200PS_EINVAL, "bad raw buffer definition");
  std::lock_guard<std::mutex> lk(ps->mu);
  auto it = ps->by_name.find(name);
  if (it != ps->by_name.end()) return it->second;
  Table t;
  t.name = name;
  t.dim = 1;
  t.owner = -1;
  t.raw = true;
  t.rows = (int64_t)((bytes + 3) / 4);
  t.row_stride = 1;
  t.bytes = (bytes + (2u << 20) - 1) / (2u << 20) * (2u << 20);  // IPC-exportable whole blocks
  return register_common(ps, std::move(t));
}

int b200ps_raw_ptr(b200ps_t* ps, int table, int shard, void** ptr, size_t* bytes) {
  if (!ps || table < 0 || table >= (int)ps->tables.size() || shard < 0 || shard >= ps->n_shards || !ptr)
    return fail(B200PS_EINVAL, "bad argument");
  const Table& t = ps->tables[table];
  if (!t.raw) return fail(B200PS_EINVAL, t.name + " is not a raw buffer");
  if (!t.alloc[shard].ptr) return fail(B200PS_ESTATE, "shard not attached (sync peers after registering)");
  *ptr = t.alloc[shard].ptr;
  if (bytes) *bytes = t.alloc[shard].bytes;
  return B200PS_OK;
}

int b200ps_table_rows_ptr(b200ps_t* ps, int table, int shard, float** base, int64_t* row_stride, int64_t* param_off,
                          int64_t* rows) {
  if (!ps || table < 0 || table >= (int)ps->tables.size() || shard < 0 || shard >= ps->n_shards || !base ||
      !row_stride || !param_off || !rows)
    return fail(B200PS_EINVAL, "bad argument");
  const Table& t = ps->tables[table];
  if (t.raw || t.is_dense || t.hashed) return fail(B200PS_EINVAL, t.name + " is not a direct-indexed embedding table");
  if (!t.alloc[shard].ptr) return fail(B200PS_ESTATE, "shard not attached (sync peers after registering)");
  *base = (float*)((char*)t.alloc[shard].ptr + t.base_off);
  *row_stride = t.row_stride;
  *param_off = t.slot_off[0];
  *rows = t.rows;
  return B200PS_OK;
}

int b200ps_barrier(b200ps_t* ps, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  int me = -1, n_local = 0;
  for (int s = 0; s < ps->n_shards; ++s)
    if (ps->shard[s].local) { me = s; ++n_local; }
  if (n_local != 1) return fail(B200PS_ESTATE, "b200ps_barrier needs exactly one local shard per process (rank-per-GPU)");
  DeviceGuard g(ps->client_device);
  k_group_barrier<<<1, 32, 0, (cudaStream_t)stream>>>(group_view(ps), me, ps->d_err);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_push_dense(b200ps_t* ps, const b200ps_seg_t* segs, int nseg, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  Split sp;
  rc = split_segs(ps, segs, nseg, true, &sp);
  if (rc) return rc;
  GroupView gv = group_view(ps);
  cudaStream_t st = (cudaStream_t)stream;
  OptParams o = ps->opt;
  const bool twice = (ps->flags & 1u) && o.kind == kAMSGrad;
  return for_each_class(ps, sp, [&](int, dim3 grid, const SegBatch& b) {
    if (twice) {
      k_push_dense<kAMSGrad, true><<<grid, 256, 0, st>>>(gv, b, o);
      return;
    }
    DISPATCH_OPT(o.kind, k_push_dense<OPT, false><<<grid, 256, 0, st>>>(gv, b, o));
  });
}

static int push_dense_reduce_impl(b200ps_t* ps, int dense_id, const float* const* grads_dev, int n_replicas,
                                  float scale, int divide, const float* param_dev, const float* adam, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  if (dense_id < 0 || dense_id >= (int)ps->tables.size() || !ps->tables[dense_id].is_dense) return fail(B200PS_ENOTFOUND, "not a dense parameter");
  if (n_replicas < 1 || n_replicas > kMaxShards || !grads_dev) return fail(B200PS_EINVAL, "n_replicas out of range");
  if (divide && scale == 0.0f) return fail(B200PS_EINVAL, "divisor is zero");
  if (param_dev && ps->opt.kind != kSGD && ps->opt.kind != kMomentum && ps->opt.kind != kAdam && ps->opt.kind != kAMSGrad)
    return fail(B200PS_EINVAL, "the torch allreduce update covers SGD, momentum, Adam and AMSGrad only");
  DeviceGuard g(ps->client_device);
  const Table& t = ps->tables[dense_id];
  ReplicaGrads rg{};
  bool vec = (t.rows * t.dim) % 4 == 0 && (!param_dev || aligned16(param_dev));
  for (int r = 0; r < n_replicas; ++r) {
    rg.g[r] = grads_dev[r];
    vec = vec && aligned16(grads_dev[r]);
  }
  rg.n = n_replicas;
  rg.scale = scale;
  rg.divide = divide ? 1 : 0;
  rg.param = param_dev;
  if (adam) {
    rg.alpha = adam[0];
    rg.eps = adam[1];
    rg.c1 = adam[2];
    rg.c2 = adam[3];
  }
  long long numel = t.rows * t.dim;
  GroupView gv = group_view(ps);
  cudaStream_t st = (cudaStream_t)stream;
  OptParams o = ps->opt;
  int grid = grid_for(ps, vec ? numel / 4 : numel);
  if (param_dev) {
    DISPATCH_OPT(o.kind, {
      if (vec) k_push_dense_reduce<OPT, 4, false, true><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
      else k_push_dense_reduce<OPT, 1, false, true><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
    });
  } else if ((ps->flags & 1u) && o.kind == kAMSGrad) {
    if (vec) k_push_dense_reduce<kAMSGrad, 4, true, false><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
    else k_push_dense_reduce<kAMSGrad, 1, true, false><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
  } else {
    DISPATCH_OPT(o.kind, {
      if (vec) k_push_dense_reduce<OPT, 4, false, false><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
      else k_push_dense_reduce<OPT, 1, false, false><<<grid, 256, 0, st>>>(gv, dense_id, rg, o);
    });
  }
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_push_dense_reduce(b200ps_t* ps, int dense_id, const float* const* grads_dev, int n_replicas, float scale,
                             int divide, void* stream) {
  return push_dense_reduce_impl(ps, dense_id, grads_dev, n_replicas, scale, divide, nullptr, nullptr, stream);
}

int b200ps_push_dense_allreduce(b200ps_t* ps, int dense_id, const float* param_dev, const float* const* grads_dev,
                                int n_replicas, float scale, float alpha, float epsilon, float one_minus_beta1,
                                float one_minus_beta2, void* stream) {
  if (!param_dev) return fail(B200PS_EINVAL, "param_dev is null");
  const float adam[4] = {alpha, epsilon, one_minus_beta1, one_minus_beta2};
  return push_dense_reduce_impl(ps, dense_id, grads_dev, n_replicas, scale, 0, param_dev, adam, stream);
}

static int push_end_impl(b200ps_t* ps, int32_t* versions_out_host, void* stream, int only_shard);
int b200ps_push_end(b200ps_t* ps, int32_t* versions_out_host, void* stream) {
  return push_end_impl(ps, versions_out_host, stream, -1);
}
int b200ps_push_end_shard(b200ps_t* ps, int shard, void* stream) {
  if (!ps || shard < 0 || shard >= ps->n_shards) return fail(B200PS_EINVAL, "bad shard id");
  return push_end_impl(ps, nullptr, stream, shard);
}
static int push_end_impl(b200ps_t* ps, int32_t* versions_out_host, void* stream, int only_shard) {
  int rc = ready(ps);
  if (rc) return rc;
  DeviceGuard g(ps->client_device);
  cudaStream_t st = (cudaStream_t)stream;
  k_push_end<<<1, 32, 0, st>>>(group_view(ps), ps->d_versions, only_shard);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  if (versions_out_host)
    CUDA_OK(cudaMemcpyAsync(versions_out_host, ps->d_versions, sizeof(int) * ps->n_shards, cudaMemcpyDeviceToHost, st));
  return B200PS_OK;
}

// ---- kernel_api.h drop-ins on raw device arrays --------------------------------
}  // extern "C"

template <int OPT>
static int raw_dense(const float* g, float* p, float* s0, float* s1, float* s2, long long n, float lr, float alpha,
                     float l2adj, const OptParams& o, void* stream) {
  if (!g || !p || n < 0) return fail(B200PS_EINVAL, "null array");
  if (n == 0) return B200PS_OK;
  bool vec = n % 4 == 0 && aligned16(g) && aligned16(p) && (!s0 || aligned16(s0)) && (!s1 || aligned16(s1)) &&
             (!s2 || aligned16(s2));
  long long work = vec ? n / 4 : n;
  int grid = grid_for(nullptr, work);
  cudaStream_t st = (cudaStream_t)stream;
  if (vec) k_raw_dense<OPT, 4><<<grid, 256, 0, st>>>(g, p, s0, s1, s2, n, lr, alpha, l2adj, o);
  else k_raw_dense<OPT, 1><<<grid, 256, 0, st>>>(g, p, s0, s1, s2, n, lr, alpha, l2adj, o);
  count_launch(nullptr, 1);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

extern "C" {

int b200ps_kernel_sgd(const float* grad, float* param, float lr, long long size, void* stream) {
  OptParams o{};
  o.kind = kSGD;
  return raw_dense<kSGD>(grad, param, nullptr, nullptr, nullptr, size, lr, 0.f, 0.f, o, stream);
}

int b200ps_kernel_momentum(const float* grad, float* param, float* velocity, float mu, int nesterov, float lr,
                           long long size, void* stream) {
  if (!velocity) return fail(B200PS_EINVAL, "null velocity");
  OptParams o{};
  o.kind = kMomentum;
  o.mu = mu;
  o.nesterov = nesterov;
  return raw_dense<kMomentum>(grad, param, velocity, nullptr, nullptr, size, lr, 0.f, 0.f, o, stream);
}

int b200ps_kernel_adam(const float* grad, float* param, float* m, float* v, float lr, long long size, long long step,
                       float beta1, float beta2, float epsilon, float* max_square, void* stream) {
  if (!m || !v) return fail(B200PS_EINVAL, "null moment array");
  OptParams o{};
  o.kind = max_square ? kAMSGrad : kAdam;
  o.beta1 = beta1;
  o.beta2 = beta2;
  o.epsilon = epsilon;
  o.c1 = (float)(1.0 - (double)beta1);
  o.c2 = (float)(1.0 - (double)beta2);
  // kernel_api.cc:67: lr *= sqrt(1 - pow(beta2, step)) / (1 - pow(beta1, step)), double math on the host
  float alpha = (float)((double)lr * (std::sqrt(1.0 - std::pow((double)beta2, (double)step)) /
                                      (1.0 - std::pow((double)beta1, (double)step))));
  if (max_square) return raw_dense<kAMSGrad>(grad, param, m, v, max_square, size, lr, alpha, 0.f, o, stream);
  return raw_dense<kAdam>(grad, param, m, v, nullptr, size, lr, alpha, 0.f, o, stream);
}

int b200ps_kernel_adagrad(const float* grad, float* param, float* m, float lr, long long size, float epsilon,
                          void* stream) {
  if (!m) return fail(B200PS_EINVAL, "null accumulator");
  OptParams o{};
  o.kind = kAdagrad;
  o.epsilon = epsilon;
  return raw_dense<kAdagrad>(grad, param, m, nullptr, nullptr, size, lr, 0.f, 0.f, o, stream);
}

// ---- unique / segment sum ------------------------------------------------------

static int uniq_cap(int64_t k) {
  int cap = 64;
  while ((int64_t)cap < 2 * k) cap <<= 1;
  return cap;
}

static size_t align256(size_t x) { return (x + 255) / 256 * 256; }

static size_t bounded_extra(int T, const int64_t* bounds) {
  size_t extra = 0;
  if (bounds && T <= kMaxSegs)
    for (int t = 0; t < T; ++t)
      if (bounds[t] > 0 && bounds[t] <= (1LL << 30)) extra += align256((size_t)bounds[t] * 4);
  return extra;
}

size_t b200ps_unique_bounded_workspace(int T, int64_t k, const int64_t* bounds) {
  return b200ps_unique_workspace(T, k) + bounded_extra(T, bounds);
}

// Look-back descriptors are sized for the smallest tile (256 x 4 positions).
constexpr int kUMinTile = kUUnit;

size_t b200ps_unique_workspace(int T, int64_t k) {
  if (T < 1 || k < 1) return 256;
  size_t cap = (size_t)uniq_cap(k);
  size_t ntiles = (size_t)((k + kUMinTile - 1) / kUMinTile);
  return align256((size_t)T * cap * 8) + align256((size_t)T * cap * 4) + 2 * align256((size_t)T * k * 4) +
         align256((size_t)T * ntiles * 8) + 256;
}

static long long* g_dbg_buf = nullptr;  // b200ps_debug_buffer: per-block phase time stamps (profiling aid)
static size_t g_dbg_bytes = 0;

static int unique_impl(b200ps_t* ps, const void* ids_dev, int ids32, int T, int64_t k, const int64_t* bounds,
                       int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                       size_t workspace_bytes, void* stream, int blocks_per_sm = 0, const int32_t* widths = nullptr) {
  if (T < 1 || T > 65535 || k < 1 || k > (1LL << 29)) return fail(B200PS_EINVAL, "bad unique shape");
  if (!ids_dev || !uniq_dev || !inv_dev || !n_unique_dev || !workspace_dev) return fail(B200PS_EINVAL, "null argument");
  if (workspace_bytes < b200ps_unique_workspace(T, k)) return fail(B200PS_EINVAL, "unique workspace too small");
  if (bounds && workspace_bytes < b200ps_unique_bounded_workspace(T, k, bounds)) bounds = nullptr;  // no room: hash everything
  const int dev = client_dev(ps);
  DeviceGuard g(dev);
  cudaStream_t st = (cudaStream_t)stream;
  UArgs a{};
  a.ids = ids_dev;
  a.ids32 = ids32;
  a.k = k;
  a.T = T;
  a.cap = uniq_cap(k);
  // co-resident grid (the kernel synchronises its phases with a grid barrier)
  static int occ[64] = {0};
  static int sms[64] = {0};
  if (dev < 64 && occ[dev] == 0) {
    int o = 0, n = 0;
    CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k_unique, kUThreads, 0));
    CUDA_OK(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
    occ[dev] = o < 1 ? 1 : (o > 4 ? 4 : o);
    sms[dev] = n < 1 ? 1 : n;
  }
  long long max_blocks = dev < 64 ? (long long)occ[dev] * sms[dev] : 132;
  // a caller that overlaps the dedup with other kernels (lookahead pipeline) asks for a thin grid: the
  // persistent blocks hold their registers for the whole call, including the time spent at the grid barriers
  if (blocks_per_sm > 0 && dev < 64 && (long long)blocks_per_sm * sms[dev] < max_blocks) max_blocks = (long long)blocks_per_sm * sms[dev];
  a.ntiles = (int)((k + kUUnit - 1) / kUUnit);  // units per segment
  char* p = (char*)workspace_dev;
  a.keys = (long long*)p; p += align256((size_t)T * a.cap * 8);
  a.minpos = (int*)p; p += align256((size_t)T * a.cap * 4);
  a.fp = (int*)p; p += align256((size_t)T * k * 4);
  a.rank_at = (int*)p; p += align256((size_t)T * k * 4);
  a.status = (unsigned long long*)p;
  a.hdr = (unsigned long long*)((char*)workspace_dev + b200ps_unique_workspace(T, k) - 256);
  a.magic = 0xB2005EED00000000ULL ^ mix64(((uint64_t)T << 40) ^ (uint64_t)k);
  a.use_bounds = bounds != nullptr && T <= kMaxSegs;
  a.n_direct = 0;
  if (a.use_bounds) {
    a.ub.dpos = (int*)((char*)workspace_dev + b200ps_unique_workspace(T, k));
    long long off = 0;
    for (int t = 0; t < T; ++t) {
      a.ub.bound[t] = bounds[t] > 0 && bounds[t] <= (1LL << 30) ? (int)bounds[t] : 0;
      a.ub.off[t] = off;
      off += (long long)(align256((size_t)a.ub.bound[t] * 4) / 4);
      if (a.ub.bound[t] > 0) a.n_direct++;
    }
  }
  a.n_hashed = T - a.n_direct;
  a.tagged = a.use_bounds && k <= (1LL << kUniqPosBits);
  a.uniq = uniq_dev;
  a.inv = inv_dev;
  a.n_unique = n_unique_dev;
  a.err = ps ? ps->d_err : nullptr;
  a.dbg = (g_dbg_buf && g_dbg_bytes >= (size_t)max_blocks * 64) ? g_dbg_buf : nullptr;
  // block -> run of units: sparse / hashed segments (an atomic and two uncached sector reads per position) one
  // unit per block, segments with a tiny id range (cache-resident, mostly duplicates) four times as many
  URuns ur{};
  const long long ups = a.ntiles;
  long long blocks = 0;
  // segments with an id range of at most kUSmallMax go to k_unique_small: one block each, position array in
  // shared memory
  USmall us{};
  bool is_small[kMaxSegs] = {};
  int small_bound = 0;
  if (a.use_bounds && T <= kMaxSegs && k <= 32LL * kUSThreads) {
    for (int t = 0; t < T; ++t) {
      if (a.ub.bound[t] > 0 && a.ub.bound[t] <= kUSmallMax) {
        is_small[t] = true;
        us.seg[us.n++] = t;
        if (a.ub.bound[t] > small_bound) small_bound = a.ub.bound[t];
      }
    }
  }
  if (T <= kMaxSegs) {
    ur.per_seg = 1;
    for (long long rh = 1;; rh += (rh < 8 ? 1 : rh / 4)) {
      const long long rl = rh * 4;
      blocks = 0;
      for (int t = 0; t < T; ++t) {
        const bool light = a.use_bounds && a.ub.bound[t] > 0 && (long long)a.ub.bound[t] * 2 < k;
        long long r = light ? rl : rh;
        if (r > ups) r = ups;
        ur.run[t] = (int)r;
        ur.blk_prefix[t] = (int)blocks;
        if (!is_small[t]) blocks += (ups + r - 1) / r;  // a small segment has no slots in the grid-wide kernel
      }
      ur.blk_prefix[T] = (int)blocks;
      if (blocks <= max_blocks || rh >= ups) break;
    }
  } else {
    // many segments: equal runs; once there are more segments than resident blocks, one slot per segment
    ur.per_seg = 0;
    long long r = 1;
    while (r < ups && (long long)T * ((ups + r - 1) / r) > max_blocks) r += (r < 8 ? 1 : r / 4);
    if (r > ups) r = ups;
    ur.uniform_run = (int)r;
    ur.bps = (int)((ups + r - 1) / r);
    blocks = (long long)T * ur.bps;
  }
  ur.nslots = (int)blocks;
  const bool any_large = blocks > 0;
  if (blocks > max_blocks) blocks = max_blocks;  // the grid walks the slots (slot = block, block + grid, ...)
  if (blocks < 1) blocks = 1;
  if (any_large) CUDA_OK(cudaMemsetAsync(a.hdr + 4, 0, 8, st));  // the grid-barrier counter
  UIdLayout idl{};
  if (widths != nullptr) {  // packed ids: segment t holds k elements of widths[t] bytes, segments back to back, 16 B aligned
    if (T > kMaxSegs) return fail(B200PS_EINVAL, "per-segment id widths need T <= " + std::to_string(kMaxSegs));
    long long off = 0;
    for (int t = 0; t < T; ++t) {
      const int w = widths[t];
      if (w != 1 && w != 2 && w != 4 && w != 8) return fail(B200PS_EINVAL, "id width must be 1, 2, 4 or 8 bytes");
      idl.off[t] = off;
      idl.width[t] = (unsigned char)w;
      off += ((long long)k * w + 15) / 16 * 16;
    }
    a.ids32 = 2;
  }
  if (us.n > 0) {
    static bool attr_done[64] = {};
    if (dev < 64 && !attr_done[dev]) {
      CUDA_OK(cudaFuncSetAttribute(k_unique_small<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, kUSmallMax * 4));
      CUDA_OK(cudaFuncSetAttribute(k_unique_small<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, kUSmallMax * 4));
      CUDA_OK(cudaFuncSetAttribute(k_unique_small<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, kUSmallMax * 4));
      attr_done[dev] = true;
    }
    const size_t smem = (size_t)small_bound * 4;
    // with a handle and work for both kernels the small-segment kernel runs on the handle's side stream, beside
    // the grid-wide one (fork / join through events: also valid inside a stream capture); they share no output
    cudaStream_t ss = st;
    const bool fork = ps != nullptr && any_large;
    if (fork) {
      if (!ps->u_side) {
        CUDA_OK(cudaStreamCreateWithFlags(&ps->u_side, cudaStreamNonBlocking));
        CUDA_OK(cudaEventCreateWithFlags(&ps->u_fork, cudaEventDisableTiming));
        CUDA_OK(cudaEventCreateWithFlags(&ps->u_join, cudaEventDisableTiming));
      }
      ss = ps->u_side;
      CUDA_OK(cudaEventRecord(ps->u_fork, st));
      CUDA_OK(cudaStreamWaitEvent(ss, ps->u_fork, 0));
    }
    if (k <= 8LL * kUSThreads) k_unique_small<8><<<(unsigned)us.n, kUSThreads, smem, ss>>>(a, idl, us);
    else if (k <= 16LL * kUSThreads) k_unique_small<16><<<(unsigned)us.n, kUSThreads, smem, ss>>>(a, idl, us);
    else k_unique_small<32><<<(unsigned)us.n, kUSThreads, smem, ss>>>(a, idl, us);
    count_launch(ps, 1);
    if (fork) CUDA_OK(cudaEventRecord(ps->u_join, ss));
    if (any_large) {
      k_unique<<<(unsigned)blocks, kUThreads, 0, st>>>(a, ur, idl);
      count_launch(ps, 1);
    }
    if (fork) CUDA_OK(cudaStreamWaitEvent(st, ps->u_join, 0));
  } else if (any_large) {
    k_unique<<<(unsigned)blocks, kUThreads, 0, st>>>(a, ur, idl);
    count_launch(ps, 1);
  }
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_unique(b200ps_t* ps, const int64_t* ids_dev, int T, int64_t k, int64_t* uniq_dev, int32_t* inv_dev,
                  int32_t* n_unique_dev, void* workspace_dev, size_t workspace_bytes, void* stream) {
  return unique_impl(ps, ids_dev, 0, T, k, nullptr, uniq_dev, inv_dev, n_unique_dev, workspace_dev, workspace_bytes,
                     stream);
}

int b200ps_unique_bounded(b200ps_t* ps, const int64_t* ids_dev, int T, int64_t k, const int64_t* bounds,
                          int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                          size_t workspace_bytes, void* stream) {
  return unique_impl(ps, ids_dev, 0, T, k, bounds, uniq_dev, inv_dev, n_unique_dev, workspace_dev, workspace_bytes,
                     stream);
}

int b200ps_unique_bounded_i32(b200ps_t* ps, const int32_t* ids32_dev, int T, int64_t k, const int64_t* bounds,
                              int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                              size_t workspace_bytes, void* stream) {
  return unique_impl(ps, ids32_dev, 1, T, k, bounds, uniq_dev, inv_dev, n_unique_dev, workspace_dev, workspace_bytes,
                     stream);
}

int b200ps_unique_bounded_ex(b200ps_t* ps, const void* ids_dev, int ids_are_int32, int T, int64_t k, const int64_t* bounds,
                             int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                             size_t workspace_bytes, int blocks_per_sm, void* stream) {
  return unique_impl(ps, ids_dev, ids_are_int32 ? 1 : 0, T, k, bounds, uniq_dev, inv_dev, n_unique_dev, workspace_dev,
                     workspace_bytes, stream, blocks_per_sm);
}

int b200ps_unique_packed(b200ps_t* ps, const void* ids_dev, const int32_t* widths, int T, int64_t k, const int64_t* bounds,
                         int64_t* uniq_dev, int32_t* inv_dev, int32_t* n_unique_dev, void* workspace_dev,
                         size_t workspace_bytes, int blocks_per_sm, void* stream) {
  if (!widths) return fail(B200PS_EINVAL, "widths is null");
  return unique_impl(ps, ids_dev, 2, T, k, bounds, uniq_dev, inv_dev, n_unique_dev, workspace_dev, workspace_bytes, stream,
                     blocks_per_sm, widths);
}

size_t b200ps_packed_ids_bytes(const int32_t* widths, int T, int64_t k) {
  size_t off = 0;
  for (int t = 0; widths && t < T; ++t) off += ((size_t)k * (size_t)widths[t] + 15) / 16 * 16;
  return off;
}

int b200ps_debug_buffer(void* dev_ptr, size_t bytes) {
  g_dbg_buf = (long long*)dev_ptr;
  g_dbg_bytes = dev_ptr ? bytes : 0;
  return B200PS_OK;
}

static int dim_class(int dim, const void* a, const void* b) {
  if (!aligned16(a) || !aligned16(b)) return 0;
  return dim % 8 == 0 ? 2 : dim % 4 == 0 ? 1 : 0;
}

int b200ps_segment_sum(b200ps_t* ps, const float* values_dev, const int32_t* inv_dev, int T, int64_t k, int dim,
                       float* out_dev, void* stream) {
  if (T < 1 || T > 65535 || k < 1 || dim < 1) return fail(B200PS_EINVAL, "bad segment_sum shape");
  int c = dim_class(dim, values_dev, out_dev);
  int W = c == 0 ? 1 : 4 * c;
  // the kernel's 32-bit warp key is row * chunks + chunk (a 64-bit one made the dim-1 sum of a DeepFM batch 17 %
  // slower): refuse what would wrap it
  if (k * (dim / W) > INT32_MAX)
    return fail(B200PS_EINVAL, "segment_sum: k * (dim / " + std::to_string(W) + ") = " + std::to_string(k * (dim / W)) +
                                   " work items per segment, more than INT32_MAX (2147483647)");
  DeviceGuard g(client_dev(ps));
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_OK(cudaMemsetAsync(out_dev, 0, (size_t)T * k * dim * sizeof(float), st));
  dim3 grid(grid_for(ps, k * (dim / W)), T);
  if (c == 2) k_segment_sum<2><<<grid, 256, 0, st>>>(values_dev, inv_dev, k, dim, out_dev);
  else if (c == 1) k_segment_sum<1><<<grid, 256, 0, st>>>(values_dev, inv_dev, k, dim, out_dev);
  else k_segment_sum<0><<<grid, 256, 0, st>>>(values_dev, inv_dev, k, dim, out_dev);
  count_launch(ps, 1);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_gather_rows(b200ps_t* ps, const float* bet_dev, const int32_t* inv_dev, int T, int64_t k, int dim,
                       float* out_dev, void* stream) {
  if (T < 1 || T > 65535 || k < 1 || dim < 1) return fail(B200PS_EINVAL, "bad gather shape");
  DeviceGuard g(client_dev(ps));
  cudaStream_t st = (cudaStream_t)stream;
  int c = dim_class(dim, bet_dev, out_dev);
  int W = c == 0 ? 1 : 4 * c;
  dim3 grid(grid_for(ps, k * (dim / W)), T);
  if (c == 2) k_gather_rows<2><<<grid, 256, 0, st>>>(bet_dev, inv_dev, k, dim, out_dev);
  else if (c == 1) k_gather_rows<1><<<grid, 256, 0, st>>>(bet_dev, inv_dev, k, dim, out_dev);
  else k_gather_rows<0><<<grid, 256, 0, st>>>(bet_dev, inv_dev, k, dim, out_dev);
  count_launch(ps, 1);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

// ---- pooled lookup of sparse input --------------------------------------------

static int sparse_shape(int64_t B, int64_t nnz, int dim, const void* ws, size_t ws_bytes) {
  if (B < 1 || nnz < 0 || dim < 1) return fail(B200PS_EINVAL, "sparse lookup: bad shape (B >= 1, nnz >= 0, dim >= 1)");
  if (nnz + B > INT32_MAX)
    return fail(B200PS_EINVAL, "sparse lookup: nnz + B = " + std::to_string(nnz + B) + " filled entries, more than INT32_MAX");
  if (!ws || ((uintptr_t)ws & 15u)) return fail(B200PS_EINVAL, "sparse lookup: workspace null or not 16 B aligned");
  if (ws_bytes < b200ps_sparse_workspace(B, nnz, dim))
    return fail(B200PS_EINVAL, "sparse lookup: workspace smaller than b200ps_sparse_workspace(B, nnz, dim)");
  return B200PS_OK;
}

size_t b200ps_sparse_workspace(int64_t B, int64_t nnz, int dim) {
  if (B < 1 || nnz < 0 || dim < 1) return 0;
  return (size_t)SparseLayout(B, nnz, dim).words * sizeof(int);
}

int b200ps_sparse_prep(b200ps_t* ps, const int64_t* rows_dev, const void* vals_dev, int vals_are_int32, int64_t B,
                       int64_t nnz, int dim, int64_t* ids_dev, void* ws, size_t ws_bytes, void* stream) {
  if (int rc = sparse_shape(B, nnz, dim, ws, ws_bytes)) return rc;
  if (!ids_dev || (nnz > 0 && (!rows_dev || !vals_dev))) return fail(B200PS_EINVAL, "sparse_prep: null pointer");
  DeviceGuard g(client_dev(ps));
  cudaStream_t st = (cudaStream_t)stream;
  const SparseLayout L(B, nnz, dim);
  int* w = (int*)ws;
  CUDA_OK(cudaMemsetAsync(w, 0, (size_t)L.off * sizeof(int), st));  // bad count and cnt
  const int gc = grid_for(ps, L.NT * 256), gs = grid_for(ps, L.K);
  long long* ids = (long long*)ids_dev;
  const long long* rows = (const long long*)rows_dev;
  if (vals_are_int32) {
    const int* v = (const int*)vals_dev;
    k_sparse_count<<<gc, 256, 0, st>>>(rows, v, L, w);
    k_sparse_scan<<<1, kSpScanThreads, 0, st>>>(v, L, w);
    k_sparse_scatter<<<gs, 256, 0, st>>>(rows, v, L, w, ids);
  } else {
    const long long* v = (const long long*)vals_dev;
    k_sparse_count<<<gc, 256, 0, st>>>(rows, v, L, w);
    k_sparse_scan<<<1, kSpScanThreads, 0, st>>>(v, L, w);
    k_sparse_scatter<<<gs, 256, 0, st>>>(rows, v, L, w, ids);
  }
  count_launch(ps, 3);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_sparse_combine(b200ps_t* ps, const float* bet_dev, const int32_t* inv_dev, void* ws, size_t ws_bytes,
                          int64_t B, int64_t nnz, int dim, int combiner, float* out_dev, void* stream) {
  if (int rc = sparse_shape(B, nnz, dim, ws, ws_bytes)) return rc;
  if (combiner < kSpSum || combiner > kSpSqrtn) return fail(B200PS_EINVAL, "sparse_combine: combiner must be 0 (sum), 1 (mean) or 2 (sqrtn)");
  if (!bet_dev || !inv_dev || !out_dev) return fail(B200PS_EINVAL, "sparse_combine: null pointer");
  DeviceGuard g(client_dev(ps));
  cudaStream_t st = (cudaStream_t)stream;
  const SparseLayout L(B, nnz, dim);
  const int c = dim_class(dim, bet_dev, out_dev);
  const int grid = grid_for(ps, L.PB * 32);
  int* w = (int*)ws;
  if (c == 2) k_sparse_combine<2><<<grid, 256, 0, st>>>(bet_dev, inv_dev, L, w, dim, combiner, out_dev);
  else if (c == 1) k_sparse_combine<1><<<grid, 256, 0, st>>>(bet_dev, inv_dev, L, w, dim, combiner, out_dev);
  else k_sparse_combine<0><<<grid, 256, 0, st>>>(bet_dev, inv_dev, L, w, dim, combiner, out_dev);
  count_launch(ps, 1);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

int b200ps_sparse_combine_grad(b200ps_t* ps, const float* gout_dev, const int32_t* inv_dev, const void* ws,
                               size_t ws_bytes, int64_t B, int64_t nnz, int dim, int combiner, int64_t n_unique,
                               float* gbet_dev, void* stream) {
  if (int rc = sparse_shape(B, nnz, dim, ws, ws_bytes)) return rc;
  if (combiner < kSpSum || combiner > kSpSqrtn)
    return fail(B200PS_EINVAL, "sparse_combine_grad: combiner must be 0 (sum), 1 (mean) or 2 (sqrtn)");
  if (n_unique < 1 || n_unique > nnz + B) return fail(B200PS_EINVAL, "sparse_combine_grad: n_unique outside [1, nnz + B]");
  if (!gout_dev || !inv_dev || !gbet_dev) return fail(B200PS_EINVAL, "sparse_combine_grad: null pointer");
  const SparseLayout L(B, nnz, dim);
  const int c = dim_class(dim, gout_dev, gbet_dev);
  const int W = c == 0 ? 1 : 4 * c;
  if (L.K * (dim / W) > INT32_MAX)  // segment_sum_loop's 32-bit warp key, as in b200ps_segment_sum
    return fail(B200PS_EINVAL, "sparse_combine_grad: (nnz + B) * (dim / " + std::to_string(W) + ") = " +
                                   std::to_string(L.K * (dim / W)) + " work items, more than INT32_MAX (2147483647)");
  DeviceGuard g(client_dev(ps));
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_OK(cudaMemsetAsync(gbet_dev, 0, (size_t)n_unique * dim * sizeof(float), st));
  const int grid = grid_for(ps, L.K * (dim / W));
  const int* w = (const int*)ws;
  if (c == 2) k_sparse_combine_grad<2><<<grid, 256, 0, st>>>(gout_dev, inv_dev, L, w, dim, combiner, gbet_dev);
  else if (c == 1) k_sparse_combine_grad<1><<<grid, 256, 0, st>>>(gout_dev, inv_dev, L, w, dim, combiner, gbet_dev);
  else k_sparse_combine_grad<0><<<grid, 256, 0, st>>>(gout_dev, inv_dev, L, w, dim, combiner, gbet_dev);
  count_launch(ps, 1);
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

// ---- state ---------------------------------------------------------------------

int b200ps_shard_state(b200ps_t* ps, int shard, int32_t* version, int64_t* step, int32_t* initialized) {
  if (!ps || shard < 0 || shard >= ps->n_shards || !ps->shard[shard].attached) return fail(B200PS_EINVAL, "bad shard");
  DeviceGuard g(ps->client_device);
  CUDA_OK(cudaDeviceSynchronize());
  ShardCtl c;
  CUDA_OK(cudaMemcpy(&c, ps->shard[shard].ctl.ptr, sizeof(c), cudaMemcpyDefault));
  if (version) *version = c.version;
  if (step) *step = c.step;
  if (initialized) *initialized = c.initialized;
  return B200PS_OK;
}

int b200ps_set_shard_state(b200ps_t* ps, int shard, int32_t version, int64_t step, int32_t initialized) {
  if (!ps || shard < 0 || shard >= ps->n_shards || !ps->shard[shard].attached) return fail(B200PS_EINVAL, "bad shard");
  DeviceGuard g(ps->client_device);
  CUDA_OK(cudaDeviceSynchronize());
  ShardCtl c;
  CUDA_OK(cudaMemcpy(&c, ps->shard[shard].ctl.ptr, sizeof(c), cudaMemcpyDefault));
  if (version >= 0) c.version = version;
  if (step >= 0) c.step = step;
  if (initialized >= 0) c.initialized = initialized;
  CUDA_OK(cudaMemcpy(ps->shard[shard].ctl.ptr, &c, sizeof(c), cudaMemcpyDefault));
  return B200PS_OK;
}

int b200ps_snapshot_state(b200ps_t* ps, int64_t* out_host, void* stream) {
  int rc = ready(ps);
  if (rc) return rc;
  if (!out_host) return fail(B200PS_EINVAL, "out_host is null");
  DeviceGuard g(ps->client_device);
  cudaStream_t st = (cudaStream_t)stream;
  k_snapshot<<<1, 32, 0, st>>>(group_view(ps), (long long*)ps->d_state);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  CUDA_OK(cudaMemcpyAsync(out_host, ps->d_state, sizeof(int64_t) * 3 * ps->n_shards, cudaMemcpyDeviceToHost, st));
  return B200PS_OK;
}

int b200ps_try_init(b200ps_t* ps, int shard, int* won) {
  if (!ps || shard < 0 || shard >= ps->n_shards || !ps->shard[shard].attached || !won) return fail(B200PS_EINVAL, "bad shard");
  DeviceGuard g(ps->client_device);
  CUDA_OK(cudaDeviceSynchronize());  // synchronous query on the legacy stream: order it after the caller's non-blocking streams
  k_try_init<<<1, 1>>>((ShardCtl*)ps->shard[shard].ctl.ptr, (int*)ps->d_count);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  int w = 0;
  CUDA_OK(cudaMemcpy(&w, ps->d_count, sizeof(int), cudaMemcpyDeviceToHost));
  *won = w;
  return B200PS_OK;
}

int b200ps_finish_init(b200ps_t* ps, int shard, int32_t version, void* stream) {
  if (!ps || shard < 0 || shard >= ps->n_shards || !ps->shard[shard].attached) return fail(B200PS_EINVAL, "bad shard");
  DeviceGuard g(ps->client_device);
  k_finish_init<<<1, 1, 0, (cudaStream_t)stream>>>((ShardCtl*)ps->shard[shard].ctl.ptr, version);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  return B200PS_OK;
}

static int present_scan(b200ps_t* ps, int table, int shard, int64_t* ids_dev, int64_t cap, int64_t* n) {
  if (!ps || table < 0 || table >= (int)ps->tables.size() || shard < 0 || shard >= ps->n_shards || !n) return fail(B200PS_EINVAL, "bad argument");
  const Table& t = ps->tables[table];
  if (t.is_dense || (!t.present_off && !t.hashed)) return fail(B200PS_ESTATE, "created rows are not tracked for " + t.name);
  if (!t.alloc[shard].ptr) return fail(B200PS_ESTATE, "shard not attached");
  DeviceGuard g(ps->client_device);
  CUDA_OK(cudaDeviceSynchronize());  // synchronous query on the legacy stream: order it after the caller's non-blocking streams
  CUDA_OK(cudaMemsetAsync(ps->d_count, 0, 8, 0));
  if (t.hashed) {
    k_key_ids<<<grid_for(ps, t.rows), 256>>>((const long long*)((const char*)t.alloc[shard].ptr + t.keys_off), t.rows, ids_dev,
                                              cap, ps->d_count);
    ps->launches++;
    CUDA_OK(cudaGetLastError());
    unsigned long long c = 0;
    CUDA_OK(cudaMemcpy(&c, ps->d_count, 8, cudaMemcpyDeviceToHost));
    *n = (int64_t)c;
    return B200PS_OK;
  }
  k_present_ids<<<grid_for(ps, t.rows), 256>>>((const uint32_t*)((const char*)t.alloc[shard].ptr + t.present_off), t.rows,
                                                shard, ps->n_shards, ids_dev, cap, ps->d_count);
  ps->launches++;
  CUDA_OK(cudaGetLastError());
  unsigned long long c = 0;
  CUDA_OK(cudaMemcpy(&c, ps->d_count, 8, cudaMemcpyDeviceToHost));
  *n = (int64_t)c;
  return B200PS_OK;
}

int b200ps_table_size(b200ps_t* ps, int table, int shard, int64_t* rows) { return present_scan(ps, table, shard, nullptr, 0, rows); }
int b200ps_table_ids(b200ps_t* ps, int table, int shard, int64_t* ids_dev, int64_t cap, int64_t* n) {
  return present_scan(ps, table, shard, ids_dev, cap, n);
}

int b200ps_check(b200ps_t* ps) {
  if (!ps) return fail(B200PS_EINVAL, "null group");
  DeviceGuard g(ps->client_device);
  CUDA_OK(cudaDeviceSynchronize());
  unsigned e = 0;
  CUDA_OK(cudaMemcpy(&e, ps->d_err, 4, cudaMemcpyDeviceToHost));
  if (e) {
    CUDA_OK(cudaMemset(ps->d_err, 0, 4));
    if (e & kErrTimeout) return fail(B200PS_ESTATE, "exchange wait timed out: a peer rank did not run the same step");
    if (e & kErrFull) return fail(B200PS_ERANGE, "hashed embedding table is full (raise expected_rows)");
    if (e & kErrRange) return fail(B200PS_ERANGE, "embedding id outside the registered table capacity (or negative)");
    return fail(B200PS_EINVAL, "device-side error word " + std::to_string(e));
  }
  return B200PS_OK;
}

int64_t b200ps_launch_count(b200ps_t* ps) { return ps ? ps->launches : g_free_launches; }

}  // extern "C"
