// deepctr WDL tower (include/b200_deepctr_wdl.h): one training step of deepctr's WDL on Criteo-shaped rows, from
// hashed ids to the loss and the dense gradient of all 61 parameters, in five launches with no float atomics.  The
// sort and the DNN are deepctr_dnn.cuh's, shared with the DeepFM estimator tower.
//
//   k_deepctr_wdl_hist     grid (NCH, 26): each CTA counts its sample chunk's ids per row of one table.
//   k_deepctr_wdl_scatter  grid (NCH, 26): a stable counting sort of each table's occurrences by row -- each
//                          CTA's cursors start at the row's offset plus the earlier chunks' counts; inside a
//                          chunk, warps take their turn in order and lanes of one row rank by lane.  perm[j] then
//                          lists, row by row, the samples that read the row in sample order.
//   k_deepctr_wdl_tower    at most one CTA per SM, grid-striding over tiles of 64 samples: gather x (one 16-byte
//                          load per deep row) and the linear logit, the three hidden layers forward, the loss and
//                          dz, the backward, dx of the 104 sparse columns and dz per sample (to the workspace),
//                          and every dense weight's batch sum into the CTA's own partial (read-add-write, each
//                          entry owned by one thread).  The hidden layers' forward, data and weight contractions
//                          are 3xTF32 mma.sync (mma_tf32.cuh); the activations are rewritten in place by their
//                          gradients, so a tile holds x, h1, h2 and h3 only (152 KB).
//   k_deepctr_wdl_tables   one warp per (table, row): the row's occurrences in perm order, a fixed shuffle tree,
//                          plus 2 lambda W, written for every row; the rows' sum of squares into per-CTA partials.
//   k_deepctr_wdl_reduce   grid-wide: entry i of the dense gradient is the sum of the tower CTAs' partials in CTA
//                          order (so no single CTA streams the 38 MB of partials); thread 0 forms the loss.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_deepctr_wdl.h"
#include "deepctr_dnn.cuh"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::DeepctrWdl>;
entry::LaunchCount g_launches{0};

using deepctr::DIM;
using deepctr::F;
using deepctr::N1;
using deepctr::N2;
using deepctr::N3;
using deepctr::NCH;
using deepctr::ND;
using deepctr::NF;
using deepctr::NS;
using deepctr::S1;
using deepctr::S2;
using deepctr::S3;
using deepctr::SORT_THREADS;
using deepctr::THREADS;
using deepctr::TILE;
using deepctr::WARPS;
using deepctr::XS;
constexpr int ROWS = B200_DEEPCTR_WDL_ROWS;
static_assert(NF == B200_DEEPCTR_WDL_FIELDS && ND == B200_DEEPCTR_WDL_DENSE && DIM == B200_DEEPCTR_WDL_DIM &&
                  TILE == B200_DEEPCTR_WDL_TILE,
              "shapes of include/b200_deepctr_wdl.h");
constexpr float LAMBDA = 1e-5f;  // l2_reg_embedding = l2_reg_linear = 1e-5

// flat offsets (floats)
constexpr int64_t O_DEEP = 0, O_LIN = (int64_t)NF * ROWS * DIM, O_DNN = O_LIN + (int64_t)NF * ROWS;
// offsets inside the dense block (and of a tower CTA's partial, whose last entry is the loss sum)
constexpr int P_WLIN = 0, P_W0 = P_WLIN + ND, P_B0 = P_W0 + F * N1, P_W1 = P_B0 + N1, P_B1 = P_W1 + N1 * N2;
constexpr int P_W2 = P_B1 + N2, P_B2 = P_W2 + N2 * N3, P_WD = P_B2 + N3, P_GB = P_WD + N3, N_DNN = P_GB + 1;
constexpr int P_BCE = N_DNN, Q = N_DNN + 1;
struct Dnn {  // the DNN layout in the dense block and the partial
  static constexpr int W0 = P_W0, B0 = P_B0, W1 = P_W1, B1 = P_B1, W2 = P_W2, B2 = P_B2, WD = P_WD;
};
static_assert(O_DNN + N_DNN == B200_DEEPCTR_WDL_PARAMS, "flat layout of include/b200_deepctr_wdl.h");
static_assert(O_DNN + P_W0 == 1300013 && O_DNN + P_B2 == 1371309 && O_DNN + P_GB == 1371437, "flat offsets");

// shared memory of the tower (floats): x | h1 | h2 | h3 (deepctr_dnn.cuh) | dz | lin / loss
constexpr int SM_H1 = TILE * XS, SM_H2 = SM_H1 + TILE * S1, SM_H3 = SM_H2 + TILE * S2, SM_DZ = SM_H3 + TILE * S3;
constexpr int SM_LS = SM_DZ + TILE, SMEM_FLOATS = SM_LS + TILE;
constexpr int SMEM_BYTES = SMEM_FLOATS * 4;

constexpr int TABLE_BLOCKS_PER_SM = 4;

struct Work {  // the workspace, carved by carve()
  float* parts;   // [grid][Q] the tower CTAs' partials
  float* tparts;  // [table blocks] sums of squares of the table rows
  float* dx;      // [B][104]
  float* dz;      // [B]
  int* counts;    // [26][NCH][ROWS]
  int* offsets;   // [26][ROWS + 1]
  int* perm;      // [26][B]
};

__host__ __device__ inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

__host__ __device__ inline size_t carve(void* base, int64_t B, int grid, int tblocks, Work* w) {
  size_t o = 0;
  char* p = reinterpret_cast<char*>(base);
  auto take = [&](size_t bytes) {
    char* r = p ? p + o : nullptr;
    o = align256(o + bytes);
    return r;
  };
  Work k;
  k.parts = reinterpret_cast<float*>(take((size_t)grid * Q * 4));
  k.tparts = reinterpret_cast<float*>(take((size_t)tblocks * 4));
  k.dx = reinterpret_cast<float*>(take((size_t)B * NS * 4));
  k.dz = reinterpret_cast<float*>(take((size_t)B * 4));
  k.counts = reinterpret_cast<int*>(take((size_t)NF * NCH * ROWS * 4));
  k.offsets = reinterpret_cast<int*>(take((size_t)NF * (ROWS + 1) * 4));
  k.perm = reinterpret_cast<int*>(take((size_t)NF * B * 4));
  if (w) *w = k;
  return o;
}

struct Rows {  // an id outside [0, 10000) is read as row 0
  static constexpr bool kSkips = false;
  __device__ __forceinline__ static int row(int id) { return (unsigned)id < (unsigned)ROWS ? id : 0; }
};

__global__ void __launch_bounds__(SORT_THREADS) k_deepctr_wdl_hist(const int32_t* __restrict__ ids, int64_t B,
                                                                   int* __restrict__ counts) {
  deepctr::sort_hist<ROWS, Rows>(ids, B, counts);
}

__global__ void __launch_bounds__(SORT_THREADS) k_deepctr_wdl_scatter(const int32_t* __restrict__ ids, int64_t B,
                                                                      const int* __restrict__ counts,
                                                                      int* __restrict__ offsets,
                                                                      int* __restrict__ perm) {
  deepctr::sort_scatter<ROWS, Rows>(ids, B, counts, offsets, perm);
}

// ---- the tower
__global__ void __launch_bounds__(THREADS, 1) k_deepctr_wdl_tower(b200_deepctr_wdl_args_t a, Work w, int ntiles,
                                                                 int train) {
  extern __shared__ __align__(16) float sm[];
  float* X = sm;
  float* A1 = sm + SM_H1;
  float* A2 = sm + SM_H2;
  float* A3 = sm + SM_H3;
  float* dzs = sm + SM_DZ;
  float* ls = sm + SM_LS;
  const float* __restrict__ P = a.params;
  const float* __restrict__ D = P + O_DNN;
  const int t = threadIdx.x;
  const int64_t B = a.B;
  float* mine = w.parts + (size_t)blockIdx.x * Q;

  for (int i = t; i < TILE * (XS - F); i += THREADS) X[(i / (XS - F)) * XS + F + i % (XS - F)] = 0.f;
  bool first = true;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, first = false) {
    const int64_t base = (int64_t)tile * TILE;
    const int n = B - base < TILE ? (int)(B - base) : TILE;
    // x: the 26 deep rows (float4 each) and the 13 dense values; rows past the batch are zero
    for (int i = t; i < TILE * NF; i += THREADS) {
      const int r = i % TILE, j = i / TILE;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < n) {
        int id = __ldg(a.ids + j * B + base + r);
        if ((unsigned)id >= (unsigned)ROWS) {
          atomicAdd(a.error, 1);
          id = 0;
        }
        v = __ldg(reinterpret_cast<const float4*>(P + O_DEEP + ((int64_t)j * ROWS + id) * DIM));
      }
      *reinterpret_cast<float4*>(X + r * XS + DIM * j) = v;
    }
    for (int i = t; i < TILE * ND; i += THREADS) {
      const int r = i % TILE, c = i / TILE;
      X[r * XS + NS + c] = r < n ? __ldg(a.dense + c * B + base + r) : 0.f;
    }
    __syncthreads();
    // the linear logit, one thread per sample: the 26 linear rows in order, then I . w_lin
    if (t < TILE) {
      float s = 0.f;
      if (t < n) {
        for (int j = 0; j < NF; ++j) s += __ldg(P + O_LIN + (int64_t)j * ROWS + Rows::row(__ldg(a.ids + j * B + base + t)));
        for (int i = 0; i < ND; ++i) s = fmaf(X[t * XS + NS + i], __ldg(D + P_WLIN + i), s);
      }
      ls[t] = s;
    }
    deepctr::dnn_forward<Dnn>(X, A1, A2, A3, D);
    // z, four threads per sample (16 units each, then a fixed shuffle tree); the loss and dz
    {
      const int r = t >> 2, q = t & 3;
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < 16; ++i) s = fmaf(A3[r * S3 + 16 * q + i], __ldg(D + P_WD + 16 * q + i), s);
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      const float z = s + ls[r] + __ldg(D + P_GB);
      float dz = 0.f, loss = 0.f;
      if (r < n) {
        if (q == 0) a.logits[base + r] = z;
        if (train) {
          const float y = __ldg(a.labels + base + r);
          const float p = 1.f / (1.f + expf(-z));
          const float eps = 1e-7f, hi = 1.f - eps;  // Keras backend.epsilon(), clip_by_value(p, eps, 1 - eps)
          const float pc = fminf(fmaxf(p, eps), hi);
          loss = -(y * logf(pc + eps) + (1.f - y) * logf(1.f - pc + eps));
          if (p >= eps && p <= hi) {  // the clip passes the gradient only inside [eps, 1 - eps]
            const float dldp = -(y / (pc + eps) - (1.f - y) / (1.f - pc + eps));
            dz = dldp * (p * (1.f - p)) / (float)B;
          }
        }
      }
      __syncthreads();  // every z read ls before it becomes the loss
      if (q == 0) {
        dzs[r] = dz;
        ls[r] = loss;
      }
    }
    __syncthreads();
    if (!train) continue;

    // the tile's sums of per-sample products, one entry per thread, rows in order
    for (int e = t; e < N3 + ND + 2; e += THREADS) {
      float s = 0.f;
      if (e < N3) {
        for (int r = 0; r < TILE; ++r) s = fmaf(A3[r * S3 + e], dzs[r], s);
        deepctr::add_part(mine + P_WD + e, s, first);
      } else if (e < N3 + ND) {
        for (int r = 0; r < TILE; ++r) s = fmaf(X[r * XS + NS + e - N3], dzs[r], s);
        deepctr::add_part(mine + P_WLIN + e - N3, s, first);
      } else if (e == N3 + ND) {
        for (int r = 0; r < TILE; ++r) s += dzs[r];
        deepctr::add_part(mine + P_GB, s, first);
      } else {
        for (int r = 0; r < TILE; ++r) s += ls[r];
        deepctr::add_part(mine + P_BCE, s, first);
      }
    }
    __syncthreads();
    // the DNN's weight gradients, and dx of the sparse columns per sample
    deepctr::dnn_backward<Dnn>(X, A1, A2, A3, dzs, D, mine, first, [&](int m, int c, float v) {
      if (m < n) __stcg(w.dx + (base + m) * NS + c, v);
    });
    if (t < n) __stcg(w.dz + base + t, dzs[t]);
    __syncthreads();
  }
}

// one warp per (table, row): 2 lambda W + the row's occurrences in perm order, for the deep and the linear row
__global__ void __launch_bounds__(THREADS) k_deepctr_wdl_tables(b200_deepctr_wdl_args_t a, Work w) {
  __shared__ float wsq[WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* __restrict__ P = a.params;
  const int64_t B = a.B;
  float sq = 0.f;
  for (int row = blockIdx.x * WARPS + warp; row < NF * ROWS; row += gridDim.x * WARPS) {
    const int j = row / ROWS, r = row - j * ROWS;
    const int s = __ldg(w.offsets + (size_t)j * (ROWS + 1) + r), e = __ldg(w.offsets + (size_t)j * (ROWS + 1) + r + 1);
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    float gl = 0.f;
    for (int p = s + lane; p < e; p += 32) {
      const int b = __ldg(w.perm + (size_t)j * B + p);
      const float4 v = __ldcg(reinterpret_cast<const float4*>(w.dx + (int64_t)b * NS + DIM * j));
      g.x += v.x;
      g.y += v.y;
      g.z += v.z;
      g.w += v.w;
      gl += __ldcg(w.dz + b);
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) {
      g.x += __shfl_xor_sync(0xffffffffu, g.x, d);
      g.y += __shfl_xor_sync(0xffffffffu, g.y, d);
      g.z += __shfl_xor_sync(0xffffffffu, g.z, d);
      g.w += __shfl_xor_sync(0xffffffffu, g.w, d);
      gl += __shfl_xor_sync(0xffffffffu, gl, d);
    }
    if (lane == 0) {
      const int64_t od = O_DEEP + ((int64_t)j * ROWS + r) * DIM, ol = O_LIN + (int64_t)j * ROWS + r;
      const float4 W = __ldg(reinterpret_cast<const float4*>(P + od));
      const float L = __ldg(P + ol);
      const float l2 = 2.f * LAMBDA;
      *reinterpret_cast<float4*>(a.grads + od) =
          make_float4(fmaf(l2, W.x, g.x), fmaf(l2, W.y, g.y), fmaf(l2, W.z, g.z), fmaf(l2, W.w, g.w));
      a.grads[ol] = fmaf(l2, L, gl);
      sq = fmaf(W.x, W.x, sq);
      sq = fmaf(W.y, W.y, sq);
      sq = fmaf(W.z, W.z, sq);
      sq = fmaf(W.w, W.w, sq);
      sq = fmaf(L, L, sq);
    }
  }
  if (lane == 0) wsq[warp] = sq;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int i = 0; i < WARPS; ++i) s += wsq[i];
    w.tparts[blockIdx.x] = s;
  }
}

// entry i of the dense gradient: the tower CTAs' partials in CTA order (+ 2 lambda w_lin); thread 0 of CTA 0
// forms the loss
__global__ void __launch_bounds__(THREADS) k_deepctr_wdl_reduce(b200_deepctr_wdl_args_t a, Work w, int grid,
                                                                int tblocks) {
  const float* __restrict__ D = a.params + O_DNN;
  for (int i = blockIdx.x * THREADS + threadIdx.x; i < N_DNN; i += gridDim.x * THREADS) {
    float s = deepctr::cta_order_sum(w.parts, Q, grid, i);
    if (i < P_W0) s = fmaf(2.f * LAMBDA, __ldg(D + i), s);
    a.grads[O_DNN + i] = s;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const float bce = deepctr::cta_order_sum(w.parts, Q, grid, P_BCE);
    float sq = 0.f;
    for (int c = 0; c < tblocks; ++c) sq += __ldcg(w.tparts + c);
    for (int i = 0; i < ND; ++i) sq = fmaf(__ldg(D + P_WLIN + i), __ldg(D + P_WLIN + i), sq);
    *a.loss = bce / (float)a.B + LAMBDA * sq;
  }
}

struct Grid {
  int tower, tblocks;
};

int grids(int64_t B, Grid* g) {
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int64_t tiles = (B + TILE - 1) / TILE;
  g->tower = (int)(tiles < d.sms ? tiles : d.sms);
  g->tblocks = TABLE_BLOCKS_PER_SM * d.sms;
  return 0;
}

int check_args(const b200_deepctr_wdl_args_t* args, int train) {
  if (!args) return E::fail(-1, "args is null");
  const b200_deepctr_wdl_args_t& a = *args;
  if (a.B < 1 || a.B > B200_DEEPCTR_WDL_MAX_B)
    return E::fail(-1, "batch size must be in [1, " + std::to_string(B200_DEEPCTR_WDL_MAX_B) + "]");
  if (!a.ids || !a.dense || !a.params || !a.logits || !a.error) return E::fail(-1, "a buffer is null");
  if (train && (!a.labels || !a.loss || !a.grads || !a.workspace)) return E::fail(-1, "a buffer is null");
  if (reinterpret_cast<uintptr_t>(a.params) & 15u) return E::fail(-1, "params must be 16-byte aligned");
  if (train && (reinterpret_cast<uintptr_t>(a.grads) & 15u)) return E::fail(-1, "grads must be 16-byte aligned");
  if (train && (reinterpret_cast<uintptr_t>(a.workspace) & 255u))
    return E::fail(-1, "workspace must be 256-byte aligned");
  return 0;
}

int launch(const b200_deepctr_wdl_args_t* args, void* stream, int train) {
  if (int rc = check_args(args, train)) return rc;
  const b200_deepctr_wdl_args_t& a = *args;
  Grid g;
  if (int rc = grids(a.B, &g)) return rc;
  Work w{};
  if (train) {
    const size_t need = carve(nullptr, a.B, g.tower, g.tblocks, nullptr);
    if (a.workspace_bytes < need)
      return E::fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, batch " + std::to_string(a.B) +
                             " needs " + std::to_string(need));
    carve(a.workspace, a.B, g.tower, g.tblocks, &w);
  }
  if (int rc = E::raise_smem_limit(k_deepctr_wdl_tower, SMEM_BYTES)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  if (!train) {
    k_deepctr_wdl_tower<<<g.tower, THREADS, SMEM_BYTES, st>>>(a, w, ntiles, 0);
    return E::launched("k_deepctr_wdl_tower", g_launches);
  }
  const dim3 sort_grid(NCH, NF);
  k_deepctr_wdl_hist<<<sort_grid, SORT_THREADS, 0, st>>>(a.ids, a.B, w.counts);
  if (int rc = E::launched("k_deepctr_wdl_hist", g_launches)) return rc;
  k_deepctr_wdl_scatter<<<sort_grid, SORT_THREADS, 0, st>>>(a.ids, a.B, w.counts, w.offsets, w.perm);
  if (int rc = E::launched("k_deepctr_wdl_scatter", g_launches)) return rc;
  k_deepctr_wdl_tower<<<g.tower, THREADS, SMEM_BYTES, st>>>(a, w, ntiles, 1);
  if (int rc = E::launched("k_deepctr_wdl_tower", g_launches)) return rc;
  k_deepctr_wdl_tables<<<g.tblocks, THREADS, 0, st>>>(a, w);
  if (int rc = E::launched("k_deepctr_wdl_tables", g_launches)) return rc;
  k_deepctr_wdl_reduce<<<(N_DNN + THREADS - 1) / THREADS, THREADS, 0, st>>>(a, w, g.tower, g.tblocks);
  return E::launched("k_deepctr_wdl_reduce", g_launches);
}

}  // namespace

extern "C" {

const char* b200_deepctr_wdl_last_error(void) { return E::last_error().c_str(); }
int64_t b200_deepctr_wdl_launch_count(void) { return g_launches.load(); }

size_t b200_deepctr_wdl_workspace_bytes(int64_t B) {
  Grid g;
  if (B < 1 || B > B200_DEEPCTR_WDL_MAX_B || grids(B, &g)) return 0;
  return carve(nullptr, B, g.tower, g.tblocks, nullptr);
}

int b200_deepctr_wdl_tower(const b200_deepctr_wdl_args_t* args, void* stream) { return launch(args, stream, 1); }
int b200_deepctr_wdl_forward(const b200_deepctr_wdl_args_t* args, void* stream) { return launch(args, stream, 0); }

}  // extern "C"
