// Feature-id generation on the GPU (include/b200_features.h): Hashing / Discretization / IndexLookup /
// LogRound / RoundIdentity / ConcatenateWithOffset / Normalizer of elasticdl_preprocessing/layers, fused
// into one launch that writes the [G][B] id matrix b200ps_unique consumes -- the worker's feature transform
// (model_zoo/dac_ctr/feature_transform.py:36-118, census_wide_deep_model/wide_deep_functional_api.py:120-161)
// no longer runs on the host.
//
// HBM-bound integer / byte work: one thread per (group, sample); inputs are feature-major so a warp
// reads 32 consecutive values of one feature (coalesced), ids are written coalesced.  IndexLookup probes a
// vocabulary table built on the host (b200feat_vocab_build) straight from global memory through the
// read-only cache: one 16-byte slot load per probe step, the term bytes only on a fingerprint match.
#include <cuda_runtime.h>

#include <cmath>
#include <cstddef>
#include <cstdint>
#include <algorithm>
#include <cstring>
#include <string>
#include <type_traits>

#include "../../include/b200_features.h"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::Features>;
entry::LaunchCount g_launches{0};

constexpr int kMaxGroups = 64, kMaxDense = 32, kMaxBoundaries = 256, kMaxW = 64;

// ---------------------------------------------------------------------------
// FarmHash Fingerprint64 = farmhashna::Hash64 (FarmHash 1.1, public domain / MIT), lengths 0..64.
// TensorFlow's to_hash_bucket_fast is Fingerprint64(s) % num_buckets (unsigned).  Restated from the
// published algorithm; pinned by elasticdl_preprocessing/layers/hashing.py:35-39.
// ---------------------------------------------------------------------------
constexpr uint64_t k0 = 0xc3a5c85c97cb3127ULL, k1 = 0xb492b66fbe98f273ULL, k2 = 0x9ae16a3b2f90404fULL;

__host__ __device__ inline uint64_t rot(uint64_t v, int s) { return s == 0 ? v : (v >> s) | (v << (64 - s)); }
__host__ __device__ inline uint64_t shift_mix(uint64_t v) { return v ^ (v >> 47); }
__host__ __device__ inline uint64_t fetch64(const unsigned char* p) {
  uint64_t v = 0;
#pragma unroll
  for (int i = 7; i >= 0; --i) v = (v << 8) | p[i];
  return v;
}
__host__ __device__ inline uint64_t fetch32(const unsigned char* p) {
  return (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24);
}
__host__ __device__ inline uint64_t hash_len16(uint64_t u, uint64_t v, uint64_t mul) {
  uint64_t a = (u ^ v) * mul;
  a ^= (a >> 47);
  uint64_t b = (v ^ a) * mul;
  b ^= (b >> 47);
  return b * mul;
}
__host__ __device__ inline uint64_t hash_0to16(const unsigned char* s, int len) {
  if (len >= 8) {
    const uint64_t mul = k2 + (uint64_t)len * 2;
    const uint64_t a = fetch64(s) + k2;
    const uint64_t b = fetch64(s + len - 8);
    const uint64_t c = rot(b, 37) * mul + a;
    const uint64_t d = (rot(a, 25) + b) * mul;
    return hash_len16(c, d, mul);
  }
  if (len >= 4) {
    const uint64_t mul = k2 + (uint64_t)len * 2;
    const uint64_t a = fetch32(s);
    return hash_len16((uint64_t)len + (a << 3), fetch32(s + len - 4), mul);
  }
  if (len > 0) {
    const uint32_t a = s[0], b = s[len >> 1], c = s[len - 1];
    const uint32_t y = a + (b << 8);
    const uint32_t z = (uint32_t)len + (c << 2);
    return shift_mix((uint64_t)y * k2 ^ (uint64_t)z * k0) * k2;
  }
  return k2;
}
__host__ __device__ inline uint64_t hash_17to32(const unsigned char* s, int len) {
  const uint64_t mul = k2 + (uint64_t)len * 2;
  const uint64_t a = fetch64(s) * k1;
  const uint64_t b = fetch64(s + 8);
  const uint64_t c = fetch64(s + len - 8) * mul;
  const uint64_t d = fetch64(s + len - 16) * k2;
  return hash_len16(rot(a + b, 43) + rot(c, 30) + d, a + rot(b + k2, 18) + c, mul);
}
__host__ __device__ inline uint64_t hash_33to64(const unsigned char* s, int len) {
  const uint64_t mul = k2 + (uint64_t)len * 2;
  const uint64_t a = fetch64(s) * k2;
  const uint64_t b = fetch64(s + 8);
  const uint64_t c = fetch64(s + len - 8) * mul;
  const uint64_t d = fetch64(s + len - 16) * k2;
  const uint64_t y = rot(a + b, 43) + rot(c, 30) + d;
  const uint64_t z = hash_len16(y, a + rot(b + k2, 18) + c, mul);
  const uint64_t e = fetch64(s + 16) * mul;
  const uint64_t f = fetch64(s + 24);
  const uint64_t g = (y + fetch64(s + len - 32)) * mul;
  const uint64_t h = (z + fetch64(s + len - 24)) * mul;
  return hash_len16(rot(e + f, 43) + rot(g, 30) + h, e + rot(f + a, 18) + g, mul);
}
__host__ __device__ inline uint64_t fingerprint64(const unsigned char* s, int len) {
  if (len <= 16) return hash_0to16(s, len);
  if (len <= 32) return hash_17to32(s, len);
  return hash_33to64(s, len);
}

// tf.as_string(int64): plain decimal, '-' for negatives
__device__ inline int as_string(long long v, unsigned char* out) {
  unsigned long long u = v < 0 ? 0ULL - (unsigned long long)v : (unsigned long long)v;
  unsigned char tmp[20];
  int n = 0;
  do {
    tmp[n++] = (unsigned char)('0' + u % 10);
    u /= 10;
  } while (u);
  int len = 0;
  if (v < 0) out[len++] = '-';
  while (n) out[len++] = tmp[--n];
  return len;
}

__device__ inline int load_string(const uint8_t* src, int W, unsigned char* buf) {
  int len = 0;
  bool open = true;
  for (int i = 0; i < W; ++i) {
    const unsigned char c = src[i];
    buf[i] = c;
    if (open && c != 0) len = i + 1; else open = false;  // zero-padded: the string ends at the first NUL
  }
  return len;
}

// math_ops._bucketize: std::upper_bound over the boundaries (bins include their left boundary)
__device__ inline int bucketize(float x, const float* b, int n) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (x < b[mid]) hi = mid; else lo = mid + 1;
  }
  return lo;
}

static_assert(sizeof(b200feat_vocab_slot_t) == 16 && offsetof(b200feat_vocab_slot_t, index) == 8 &&
                  offsetof(b200feat_vocab_slot_t, length) == 12,
              "b200feat_vocab_slot_t is one 16-byte load: {fingerprint, index | length << 32}");

// The launch's copy of b200feat_group_ext_t: the table's probe mask, and log(base) taken once on the host.
struct GroupExt {
  const ulonglong2* slots;
  const uint8_t* terms;
  unsigned long long mask;  // n_slots - 1
  int V, Wv;
  long long dflt;
  double log_base;
  int has_base;
};

struct Plan {  // passed by value (< 4 KB): the launch is self-contained and capturable in a CUDA graph
  b200feat_group_t group[kMaxGroups];
  b200feat_dense_t dense[kMaxDense];
  float bnd[kMaxBoundaries];
  int G, n_dense;
  unsigned long long absent;  // bit g: group g's ToSparse-dropped cells are absent (b200feat_group_ext_t::absent)
};
// A transform with LOOKUP / LOG_ROUND / ROUND_IDENTITY groups launches this one (7.4 KB, still by value); one without
// them launches the Plan instance, whose parameters and code are those of the dac_ctr kinds alone.
struct PlanExt : Plan {
  GroupExt ext[kMaxGroups];
};
// kernel parameters may take 32,764 bytes on sm_70+ from CUDA 12.1; the other arguments take 48
static_assert(sizeof(PlanExt) + 64 <= 32764, "PlanExt no longer fits the kernel parameter space");

// IndexLookup: linear probing from the home slot, at most n_slots steps (a malformed table cannot hang the
// launch).  An empty slot ends the chain; a slot whose fingerprint and length match is compared byte by byte.
// Out of vocabulary: V + fp % num_oov (IdTableWithHashBuckets over FastHashSpec), or -1 without OOV buckets.
__device__ inline long long vocab_lookup(uint64_t fp, const unsigned char* buf, int len, const GroupExt& e,
                                         long long num_oov) {
  unsigned long long h = fp & e.mask;
  for (unsigned long long n = 0; n <= e.mask; ++n) {
    const ulonglong2 slot = __ldg(e.slots + h);
    const int index = (int)(unsigned)slot.y, length = (int)(slot.y >> 32);
    if (index < 0) break;
    if (slot.x == fp && length == len && index < e.V && len <= e.Wv) {
      const uint8_t* t = e.terms + (long long)index * e.Wv;
      int i = 0;
      while (i < len && __ldg(t + i) == buf[i]) ++i;
      if (i == len) return index;
    }
    h = (h + 1) & e.mask;
  }
  return num_oov > 0 ? (long long)e.V + (long long)(fp % (unsigned long long)num_oov) : -1;
}

// ToSparse's default ignore_value of a numeric column (to_sparse.py:55-63): -1 for integers, 0.0 for floats
__device__ __forceinline__ bool ignored(long long x) { return x == -1; }
__device__ __forceinline__ bool ignored(float x) { return x == 0.f; }

// The id written for a cell: -1 for an absent one (the offset is not added), else id + offset
__device__ __forceinline__ long long placed(long long id, bool absent, long long offset) {
  return absent ? -1 : id + offset;
}

// LogRound / RoundIdentity: tf.cast(r, int64) then `r < 0 || r >= num_bins -> default`.  NaN, +-inf and
// r >= 2^63 go to the default too: TF on x86 casts them to INT64_MIN (cvttsd2si), which is < 0.
__device__ inline long long rounded_id(double r, long long num_bins, long long dflt) {
  if (!(r >= 0.0) || r >= 9223372036854775808.0) return dflt;
  const long long v = (long long)r;
  return v < num_bins ? v : dflt;
}

// LOOKUP / LOG_ROUND / ROUND_IDENTITY ids of group g (the kind is uniform over the block row)
template <typename T>
__device__ __forceinline__ void ext_group_ids(const b200feat_group_t& gr, const GroupExt& ex, int g, bool drop,
                                              const T* numeric, const uint8_t* __restrict__ strings, int W, long long B,
                                              void* ids_out, int ids32) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += stride) {
    long long id;
    bool absent;
    if (gr.kind == B200FEAT_LOOKUP) {
      unsigned char buf[kMaxW];
      const int len = load_string(strings + ((long long)gr.column * B + b) * W, W, buf);
      id = vocab_lookup(fingerprint64(buf, len), buf, len, ex, gr.num_bins);
      absent = drop && len == 0;
    } else if (gr.kind == B200FEAT_LOG_ROUND) {
      // tf.cast(x, float64), then log(x) or log(x) / log(base) in float64, tf.math.round = half to even
      const T x = numeric[(long long)gr.column * B + b];
      double q = log((double)x);
      if (ex.has_base) q = q / ex.log_base;
      id = rounded_id(rint(q), gr.num_bins, ex.dflt);
      absent = drop && ignored(x);
    } else {  // ROUND_IDENTITY
      const T x = numeric[(long long)gr.column * B + b];
      if constexpr (std::is_same<T, long long>::value)  // integers pass through K.round unchanged
        id = x >= 0 && x < gr.num_bins ? x : ex.dflt;
      else  // K.round of float32 = rint in float32
        id = rounded_id((double)rintf(x), gr.num_bins, ex.dflt);
      absent = drop && ignored(x);
    }
    id = placed(id, absent, gr.offset);
    if (ids32) reinterpret_cast<int*>(ids_out)[(long long)g * B + b] = (int)id;
    else reinterpret_cast<long long*>(ids_out)[(long long)g * B + b] = id;
  }
}

// T: the numeric columns' type (long long or float); P: Plan, or PlanExt when a group has a kind >= LOOKUP
template <typename T, typename P>
__global__ void __launch_bounds__(256) k_feature_transform(P p, const T* numeric, const uint8_t* __restrict__ strings,
                                                           int W, long long B, void* ids_out, int ids32, float* dense_out) {
  __shared__ float s_bnd[kMaxBoundaries];
  const int g = blockIdx.y;
  if (g < p.G) {
    const b200feat_group_t& gr = p.group[g];
    const bool drop = (p.absent >> g) & 1ull;
    if constexpr (std::is_same<P, PlanExt>::value) {
      if (gr.kind > B200FEAT_HASH_INT) {
        ext_group_ids(gr, p.ext[g], g, drop, numeric, strings, W, B, ids_out, ids32);
        return;
      }
    }
    if (gr.kind == B200FEAT_DISCRETIZE) {
      for (int i = threadIdx.x; i < gr.n_boundaries; i += blockDim.x) s_bnd[i] = p.bnd[gr.boundary_off + i];
      __syncthreads();
    }
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += stride) {
      long long id;
      bool absent = false;
      if (gr.kind == B200FEAT_DISCRETIZE) {
        // int64 inputs compare against float boundaries in float, like TF's BucketizeOp<T>
        const T x = numeric[(long long)gr.column * B + b];
        id = bucketize((float)x, s_bnd, gr.n_boundaries);
        absent = drop && ignored(x);
      } else {
        unsigned char buf[kMaxW];
        int len = 0;
        if (gr.kind == B200FEAT_HASH_STRING) {
          len = load_string(strings + ((long long)gr.column * B + b) * W, W, buf);
          absent = drop && len == 0;
        } else if constexpr (std::is_same<T, long long>::value) {  // the host refuses HASH_INT over float columns
          const long long x = numeric[(long long)gr.column * B + b];
          len = as_string(x, buf);
          absent = drop && ignored(x);
        }
        id = (long long)(fingerprint64(buf, len) % (uint64_t)gr.num_bins);
      }
      id = placed(id, absent, gr.offset);
      if (ids32) reinterpret_cast<int*>(ids_out)[(long long)g * B + b] = (int)id;
      else reinterpret_cast<long long*>(ids_out)[(long long)g * B + b] = id;
    }
  } else {  // blockIdx.y >= G: the Normalizer columns
    const int j = g - p.G;
    const b200feat_dense_t& d = p.dense[j];
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < B; b += stride) {
      const double x = (double)numeric[(long long)d.column * B + b];
      dense_out[b * p.n_dense + j] = (float)((x - d.subtractor) / d.divisor);
    }
  }
}

__global__ void __launch_bounds__(256) k_fingerprint(const uint8_t* __restrict__ strings, int W, long long n, uint64_t* out) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    unsigned char buf[kMaxW];
    const int len = load_string(strings + i * W, W, buf);
    out[i] = fingerprint64(buf, len);
  }
}

// 8 resident blocks of 256 threads per SM of the current device
int max_blocks(int* out) {
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  *out = d.sms * 8;
  return 0;
}

int grid_x(long long n, int cap) {
  long long b = (n + 255) / 256;
  if (b > cap) b = cap;
  return (int)(b < 1 ? 1 : b);
}

}  // namespace

extern "C" {

const char* b200feat_last_error(void) { return E::last_error().c_str(); }
int64_t b200feat_launch_count(void) { return g_launches.load(); }

int b200feat_transform(const b200feat_group_t* groups, int G, const float* boundaries, int n_boundaries,
                       const b200feat_dense_t* dense, int n_dense, const void* numeric_dev, int n_numeric,
                       int numeric_is_float, const uint8_t* strings_dev, int n_string, int W, int64_t B,
                       void* ids_out_dev, int ids32, float* dense_out_dev, void* stream) {
  return b200feat_transform_ext(groups, nullptr, G, boundaries, n_boundaries, dense, n_dense, numeric_dev, n_numeric,
                                numeric_is_float, strings_dev, n_string, W, B, ids_out_dev, ids32, dense_out_dev, stream);
}

int b200feat_transform_ext(const b200feat_group_t* groups, const b200feat_group_ext_t* ext, int G,
                           const float* boundaries, int n_boundaries, const b200feat_dense_t* dense, int n_dense,
                           const void* numeric_dev, int n_numeric, int numeric_is_float, const uint8_t* strings_dev,
                           int n_string, int W, int64_t B, void* ids_out_dev, int ids32, float* dense_out_dev,
                           void* stream) {
  if (G < 0 || G > kMaxGroups) return E::fail(-1, "bad group count (max 64)");
  if (n_dense < 0 || n_dense > kMaxDense) return E::fail(-1, "bad dense column count (max 32)");
  if (B < 1) return E::fail(-1, "bad batch size");
  if (n_boundaries < 0 || n_boundaries > kMaxBoundaries) return E::fail(-1, "too many boundaries (max 256)");
  if (G > 0 && (!groups || !ids_out_dev)) return E::fail(-1, "groups / ids_out is null");
  if (n_dense > 0 && (!dense || !dense_out_dev)) return E::fail(-1, "dense / dense_out is null");
  if (W < 0 || W > kMaxW) return E::fail(-1, "strings longer than 64 bytes are not supported (FarmHash restated for lengths 0..64)");
  PlanExt p;
  memset(&p, 0, sizeof(p));
  bool ext_kinds = false;
  p.G = ids_out_dev ? G : 0;
  p.n_dense = dense_out_dev ? n_dense : 0;
  for (int g = 0; g < p.G; ++g) {
    const b200feat_group_t& gr = groups[g];
    int64_t lo = 0, hi;  // smallest and largest id before the offset
    if (gr.kind == B200FEAT_DISCRETIZE) {
      if (gr.column < 0 || gr.column >= n_numeric || !numeric_dev) return E::fail(-1, "discretize: bad numeric column");
      if (gr.n_boundaries < 0 || gr.boundary_off < 0 || gr.boundary_off + gr.n_boundaries > n_boundaries || (gr.n_boundaries && !boundaries))
        return E::fail(-1, "discretize: boundaries out of range");
      // the kernel binary-searches them; TF's Bucketize refuses unsorted boundaries
      for (int i = gr.boundary_off; i < gr.boundary_off + gr.n_boundaries; ++i)
        if (boundaries[i] != boundaries[i] || (i > gr.boundary_off && boundaries[i] < boundaries[i - 1]))
          return E::fail(-1, "discretize: boundaries are not sorted in ascending order (or hold a NaN)");
      hi = gr.n_boundaries;
    } else if (gr.kind == B200FEAT_HASH_STRING) {
      if (gr.column < 0 || gr.column >= n_string || !strings_dev || W < 1) return E::fail(-1, "hash: bad string column");
      if (gr.num_bins <= 0) return E::fail(-1, "`num_bins` cannot be `None` or non-positive values.");  // hashing.py:53-56
      hi = gr.num_bins - 1;
    } else if (gr.kind == B200FEAT_HASH_INT) {
      if (gr.column < 0 || gr.column >= n_numeric || !numeric_dev) return E::fail(-1, "hash: bad numeric column");
      if (gr.num_bins <= 0) return E::fail(-1, "`num_bins` cannot be `None` or non-positive values.");
      // Hashing converts integer inputs only (hashing.py:63-72); to_hash_bucket_fast refuses float tensors
      if (numeric_is_float) return E::fail(-1, "hash_int: Hashing takes integer columns, these numeric columns are float32");
      hi = gr.num_bins - 1;
    } else if (ext && gr.kind == B200FEAT_LOOKUP) {
      const b200feat_group_ext_t& e = ext[g];
      if (gr.column < 0 || gr.column >= n_string || !strings_dev || W < 1)
        return E::fail(-1, "lookup: bad string column (IndexLookup takes string columns)");
      if (!e.slots_dev || !e.terms_dev) return E::fail(-1, "lookup: null table");
      if (e.V < 1) return E::fail(-1, "lookup: vocabulary size V must be >= 1");
      if (e.Wv < 1 || e.Wv > kMaxW) return E::fail(-1, "lookup: term width Wv must be 1..64");
      if (e.n_slots < 2 * (int64_t)e.V || (e.n_slots & (e.n_slots - 1)))
        return E::fail(-1, "lookup: n_slots must be a power of two >= 2V");
      if (gr.num_bins < 0) return E::fail(-1, "lookup: num_oov_tokens must be >= 0");
      if (gr.num_bins > INT64_MAX - e.V) return E::fail(-1, "lookup: V + num_oov_tokens overflows int64");
      if (gr.num_bins == 0) lo = -1;  // the table's default_value
      hi = gr.num_bins > 0 ? e.V + gr.num_bins - 1 : e.V - 1;
      p.ext[g].slots = reinterpret_cast<const ulonglong2*>(e.slots_dev);
      p.ext[g].terms = e.terms_dev;
      p.ext[g].mask = (unsigned long long)e.n_slots - 1;
      p.ext[g].V = e.V;
      p.ext[g].Wv = e.Wv;
    } else if (ext && (gr.kind == B200FEAT_LOG_ROUND || gr.kind == B200FEAT_ROUND_IDENTITY)) {
      const b200feat_group_ext_t& e = ext[g];
      if (gr.column < 0 || gr.column >= n_numeric || !numeric_dev)
        return E::fail(-1, gr.kind == B200FEAT_LOG_ROUND ? "log_round: bad numeric column" : "round_identity: bad numeric column");
      // ids: [0, num_bins) u {default_value}; num_bins <= 0 is accepted (log_round.py:53-57): every id is the default
      lo = gr.num_bins > 0 ? std::min<int64_t>(0, e.default_value) : e.default_value;
      hi = gr.num_bins > 0 ? std::max<int64_t>(gr.num_bins - 1, e.default_value) : e.default_value;
      p.ext[g].dflt = e.default_value;
      p.ext[g].has_base = gr.kind == B200FEAT_LOG_ROUND && e.has_base;
      p.ext[g].log_base = std::log(e.base);  // base = 0: -inf, and log(x) / -inf = -+0 (not refused, like the reference)
    } else {
      return E::fail(-1, "unknown group kind");
    }
    if (ids32 && ((__int128)gr.offset + lo < INT32_MIN || (__int128)gr.offset + hi > INT32_MAX))
      return E::fail(-1, "int32 ids: offset + id range of a group does not fit int32");
    if (ext && ext[g].absent != 0 && ext[g].absent != 1) return E::fail(-1, "absent must be 0 or 1");
    if (ext && ext[g].absent) p.absent |= 1ull << g;
    p.group[g] = gr;
    ext_kinds |= gr.kind > B200FEAT_HASH_INT;
  }
  for (int j = 0; j < p.n_dense; ++j) {
    if (dense[j].column < 0 || dense[j].column >= n_numeric || !numeric_dev) return E::fail(-1, "normalizer: bad numeric column");
    if (dense[j].divisor == 0.0) return E::fail(-1, "The divisor cannot be 0");  // normalizer.py build()
    p.dense[j] = dense[j];
  }
  if (p.G + p.n_dense == 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  for (int i = 0; i < n_boundaries; ++i) p.bnd[i] = boundaries[i];
  int cap = 0;
  if (int rc = max_blocks(&cap)) return rc;
  int gx = grid_x(B, cap);
  const int per = (cap + p.G + p.n_dense - 1) / (p.G + p.n_dense);
  if (gx > per) gx = per < 1 ? 1 : per;
  dim3 grid(gx, p.G + p.n_dense);
  const Plan& base = p;
  if (numeric_is_float && ext_kinds)
    k_feature_transform<<<grid, 256, 0, st>>>(p, (const float*)numeric_dev, strings_dev, W, (long long)B, ids_out_dev,
                                              ids32, dense_out_dev);
  else if (numeric_is_float)
    k_feature_transform<<<grid, 256, 0, st>>>(base, (const float*)numeric_dev, strings_dev, W, (long long)B, ids_out_dev,
                                              ids32, dense_out_dev);
  else if (ext_kinds)
    k_feature_transform<<<grid, 256, 0, st>>>(p, (const long long*)numeric_dev, strings_dev, W, (long long)B,
                                              ids_out_dev, ids32, dense_out_dev);
  else
    k_feature_transform<<<grid, 256, 0, st>>>(base, (const long long*)numeric_dev, strings_dev, W, (long long)B,
                                              ids_out_dev, ids32, dense_out_dev);
  return E::launched("k_feature_transform", g_launches);
}

int64_t b200feat_vocab_slots(int64_t V) {
  if (V < 1 || V >= (1LL << 31)) return -1;
  int64_t n = 2;
  while (n < 2 * V) n <<= 1;
  return n;
}

int b200feat_vocab_build(const uint8_t* terms, int64_t V, int Wv, int64_t n_slots, b200feat_vocab_slot_t* slots,
                         int64_t* dup_pos) {
  if (V < 1 || V >= (1LL << 31)) return E::fail(-1, "vocab build: V must be 1 .. 2^31 - 1");
  if (Wv < 1 || Wv > kMaxW) return E::fail(-1, "vocab build: term width Wv must be 1..64");
  if (n_slots < 2 * V || (n_slots & (n_slots - 1))) return E::fail(-1, "vocab build: n_slots must be a power of two >= 2V");
  if (!terms || !slots) return E::fail(-1, "vocab build: terms / slots is null");
  for (int64_t i = 0; i < n_slots; ++i) slots[i] = b200feat_vocab_slot_t{0, -1, 0};
  const uint64_t mask = (uint64_t)n_slots - 1;
  for (int64_t v = 0; v < V; ++v) {
    const uint8_t* t = terms + v * Wv;
    int len = 0;
    while (len < Wv && t[len]) ++len;
    for (int i = len; i < Wv; ++i)
      if (t[i]) return E::fail(-1, "vocab build: term " + std::to_string(v) + " holds a NUL byte (rows are zero padded)");
    const uint64_t fp = fingerprint64(t, len);
    uint64_t h = fp & mask;
    for (; slots[h].index >= 0; h = (h + 1) & mask) {  // load <= 1/2: an empty slot is always reached
      const b200feat_vocab_slot_t& s = slots[h];
      if (s.fingerprint == fp && s.length == len && memcmp(terms + (int64_t)s.index * Wv, t, len) == 0) {
        if (dup_pos) *dup_pos = v;
        return E::fail(-1, "vocab build: term " + std::to_string(v) + " repeats term " + std::to_string(s.index));
      }
    }
    slots[h] = b200feat_vocab_slot_t{fp, (int32_t)v, len};
  }
  return 0;
}

int b200feat_hash_strings(const uint8_t* strings_dev, int W, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_HASH_STRING;
  g.num_bins = num_bins;
  return b200feat_transform(&g, 1, nullptr, 0, nullptr, 0, nullptr, 0, 0, strings_dev, 1, W, n, out_dev, 0, nullptr, stream);
}

int b200feat_hash_ints(const int64_t* values_dev, int64_t n, int64_t num_bins, int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_HASH_INT;
  g.num_bins = num_bins;
  return b200feat_transform(&g, 1, nullptr, 0, nullptr, 0, values_dev, 1, 0, nullptr, 0, 0, n, out_dev, 0, nullptr, stream);
}

int b200feat_bucketize(const float* x_dev, int64_t n, const float* boundaries, int n_boundaries, int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_DISCRETIZE;
  g.n_boundaries = n_boundaries;
  return b200feat_transform(&g, 1, boundaries, n_boundaries, nullptr, 0, x_dev, 1, 1, nullptr, 0, 0, n, out_dev, 0, nullptr, stream);
}

int b200feat_index_lookup(const uint8_t* strings_dev, int W, int64_t n, const b200feat_vocab_slot_t* slots_dev,
                          const uint8_t* terms_dev, int64_t n_slots, int32_t V, int32_t Wv, int64_t num_oov_tokens,
                          int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_LOOKUP;
  g.num_bins = num_oov_tokens;
  b200feat_group_ext_t e{};
  e.slots_dev = slots_dev;
  e.terms_dev = terms_dev;
  e.n_slots = n_slots;
  e.V = V;
  e.Wv = Wv;
  return b200feat_transform_ext(&g, &e, 1, nullptr, 0, nullptr, 0, nullptr, 0, 0, strings_dev, 1, W, n, out_dev, 0,
                                nullptr, stream);
}

int b200feat_log_round(const void* x_dev, int x_is_float, int64_t n, int64_t num_bins, int64_t default_value,
                       int has_base, double base, int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_LOG_ROUND;
  g.num_bins = num_bins;
  b200feat_group_ext_t e{};
  e.default_value = default_value;
  e.has_base = has_base;
  e.base = base;
  return b200feat_transform_ext(&g, &e, 1, nullptr, 0, nullptr, 0, x_dev, 1, x_is_float, nullptr, 0, 0, n, out_dev, 0,
                                nullptr, stream);
}

int b200feat_round_identity(const void* x_dev, int x_is_float, int64_t n, int64_t num_buckets, int64_t default_value,
                            int64_t* out_dev, void* stream) {
  b200feat_group_t g{};
  g.kind = B200FEAT_ROUND_IDENTITY;
  g.num_bins = num_buckets;
  b200feat_group_ext_t e{};
  e.default_value = default_value;
  return b200feat_transform_ext(&g, &e, 1, nullptr, 0, nullptr, 0, x_dev, 1, x_is_float, nullptr, 0, 0, n, out_dev, 0,
                                nullptr, stream);
}

int b200feat_fingerprint64(const uint8_t* strings_dev, int W, int64_t n, uint64_t* out_dev, void* stream) {
  if (!strings_dev || !out_dev || n < 1 || W < 1 || W > kMaxW) return E::fail(-1, "bad fingerprint arguments");
  int cap = 0;
  if (int rc = max_blocks(&cap)) return rc;
  k_fingerprint<<<grid_x(n, cap), 256, 0, (cudaStream_t)stream>>>(strings_dev, W, (long long)n, out_dev);
  return E::launched("k_fingerprint", g_launches);
}

}  // extern "C"
