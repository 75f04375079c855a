// deepctr DeepFM estimator tower (include/b200_deepctr_deepfm.h): one training step of deepctr's DeepFMEstimator on
// Criteo-shaped rows, from hashed ids (-1 absent) to the summed loss and the dense gradient of all 73 parameters, in
// five launches with no float atomics.  The sort and the DNN are deepctr_dnn.cuh's, shared with the WDL tower.
//
//   k_deepctr_deepfm_hist     grid (NCH, 26): each CTA counts its sample chunk's present ids per row of one table.
//   k_deepctr_deepfm_scatter  grid (NCH, 26): the stable counting sort of each table's present occurrences by row.
//   k_deepctr_deepfm_tower    at most one CTA per SM, grid-striding over tiles of 64 samples: gather x (a zero row
//                             for an absent id), the linear logit in the columns' name order, the FM term and the
//                             samples' embedding squares, the DNN forward, the loss and dz = sigmoid(z) - y, the
//                             backward into the CTA's own partial, and per sample dz and dx + dz (S - e) + lambda e
//                             of the 104 embedding columns (to the workspace).
//   k_deepctr_deepfm_tables   one warp per (table, row): the embedding row's occurrences of dx in perm order and the
//                             linear row's lambda w + its occurrences of dz, written for every row; the linear rows'
//                             sum of squares into per-CTA partials.
//   k_deepctr_deepfm_reduce   grid-wide: the DNN, numeric-weight and bias_weights gradients from the tower CTAs'
//                             partials in CTA order; thread 0 forms the loss.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_deepctr_deepfm.h"
#include "deepctr_dnn.cuh"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::DeepctrDeepfm>;
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
constexpr int ROWS = B200_DEEPCTR_DEEPFM_ROWS;
static_assert(NF == B200_DEEPCTR_DEEPFM_FIELDS && ND == B200_DEEPCTR_DEEPFM_DENSE && DIM == B200_DEEPCTR_DEEPFM_DIM &&
                  TILE == B200_DEEPCTR_DEEPFM_TILE,
              "shapes of include/b200_deepctr_deepfm.h");
constexpr float LAMBDA = 1e-5f;  // l2_reg_embedding = l2_reg_linear = 1e-5

// offsets inside the dnn block (and of a tower CTA's partial, which then holds the numeric weights', bias_weights'
// and the loss's sums)
constexpr int P_W0 = 0, P_B0 = P_W0 + F * N1, P_W1 = P_B0 + N1, P_B1 = P_W1 + N1 * N2, P_W2 = P_B1 + N2;
constexpr int P_B2 = P_W2 + N2 * N3, P_WD = P_B2 + N3, N_DNN = P_WD + N3;
constexpr int P_NUM = N_DNN, P_BW = P_NUM + ND, P_LOSS = P_BW + 1, Q = P_LOSS + 1;
struct Dnn {
  static constexpr int W0 = P_W0, B0 = P_B0, W1 = P_W1, B1 = P_B1, W2 = P_W2, B2 = P_B2, WD = P_WD;
};
// flat offsets (floats): the embeddings, the dnn block, the linear rows, the numeric weights, bias_weights
constexpr int64_t O_EMB = 0, O_DNN = (int64_t)NF * ROWS * DIM, O_LIN = O_DNN + N_DNN;
constexpr int64_t O_NUM = O_LIN + (int64_t)NF * ROWS, O_BW = O_NUM + ND;
static_assert(O_LIN == B200_DEEPCTR_DEEPFM_DNN_FLOATS && O_BW + 1 == B200_DEEPCTR_DEEPFM_PARAMS,
              "flat layout of include/b200_deepctr_deepfm.h");
static_assert(O_DNN + P_B0 == 133952 && O_DNN + P_WD == 175360 && O_NUM == 201424, "flat offsets");

// the linear model's columns in name order (C1, C10 .. C19, C2, C20 .. C26, C3 .. C9, then I1, I10 .. I13, I2 ..
// I9), as 0-based field and numeric indices
__constant__ unsigned char C_ORDER[NF] = {0, 9, 10, 11, 12, 13, 14, 15, 16, 17, 18, 1, 19,
                                          20, 21, 22, 23, 24, 25, 2, 3, 4, 5, 6, 7, 8};
__constant__ unsigned char I_ORDER[ND] = {0, 9, 10, 11, 12, 1, 2, 3, 4, 5, 6, 7, 8};

// shared memory of the tower (floats): x | h1 | h2 | h3 (deepctr_dnn.cuh) | dz | lin + fm, then the loss | the
// samples' sum of squared embeddings | the samples' field sums S [TILE][4]
constexpr int SM_H1 = TILE * XS, SM_H2 = SM_H1 + TILE * S1, SM_H3 = SM_H2 + TILE * S2, SM_DZ = SM_H3 + TILE * S3;
constexpr int SM_LS = SM_DZ + TILE, SM_E2 = SM_LS + TILE, SM_S = SM_E2 + TILE, SMEM_FLOATS = SM_S + TILE * DIM;
constexpr int SMEM_BYTES = SMEM_FLOATS * 4;

constexpr int TABLE_BLOCKS_PER_SM = 4;

struct Work {  // the workspace, carved by carve()
  float* parts;   // [grid][Q] the tower CTAs' partials
  float* tparts;  // [table blocks] sums of squares of the linear rows
  float* dx;      // [B][104] per occurrence: dx + dz (S - e) + lambda e
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

struct Rows {  // -1 (an empty cell) and ids outside [0, 1000) are absent: no row, no occurrence
  static constexpr bool kSkips = true;
  __device__ __forceinline__ static int row(int id) { return (unsigned)id < (unsigned)ROWS ? id : -1; }
};

__global__ void __launch_bounds__(SORT_THREADS) k_deepctr_deepfm_hist(const int32_t* __restrict__ ids, int64_t B,
                                                                      int* __restrict__ counts) {
  deepctr::sort_hist<ROWS, Rows>(ids, B, counts);
}

__global__ void __launch_bounds__(SORT_THREADS) k_deepctr_deepfm_scatter(const int32_t* __restrict__ ids, int64_t B,
                                                                         const int* __restrict__ counts,
                                                                         int* __restrict__ offsets,
                                                                         int* __restrict__ perm) {
  deepctr::sort_scatter<ROWS, Rows>(ids, B, counts, offsets, perm);
}

// ---- the tower
__global__ void __launch_bounds__(THREADS, 1) k_deepctr_deepfm_tower(b200_deepctr_deepfm_args_t a, Work w,
                                                                     int ntiles, int train) {
  extern __shared__ __align__(16) float sm[];
  float* X = sm;
  float* A1 = sm + SM_H1;
  float* A2 = sm + SM_H2;
  float* A3 = sm + SM_H3;
  float* dzs = sm + SM_DZ;
  float* ls = sm + SM_LS;
  float* e2 = sm + SM_E2;
  float* S = sm + SM_S;
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
    // x: the 26 embedding rows (float4 each, zero when absent) and the 13 dense values; rows past the batch are zero
    for (int i = t; i < TILE * NF; i += THREADS) {
      const int r = i % TILE, j = i / TILE;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (r < n) {
        const int id = __ldg(a.ids + j * B + base + r);
        if (id < -1 || id >= ROWS) atomicAdd(a.error, 1);
        if (Rows::row(id) >= 0) v = __ldg(reinterpret_cast<const float4*>(P + O_EMB + ((int64_t)j * ROWS + id) * DIM));
      }
      *reinterpret_cast<float4*>(X + r * XS + DIM * j) = v;
    }
    for (int i = t; i < TILE * ND; i += THREADS) {
      const int r = i % TILE, c = i / TILE;
      X[r * XS + NS + c] = r < n ? __ldg(a.dense + c * B + base + r) : 0.f;
    }
    __syncthreads();
    // one thread per sample: the linear logit (columns in name order, then bias_weights), the field sums S, the FM
    // term 1/2 sum_d (S_d^2 - sum_j e_jd^2) and the sum of squared embeddings
    if (t < TILE) {
      float lin = 0.f, fm = 0.f, sq = 0.f;
      if (t < n) {
        for (int k = 0; k < NF; ++k) {
          const int j = C_ORDER[k];
          const int r = Rows::row(__ldg(a.ids + j * B + base + t));
          if (r >= 0) lin += __ldg(P + O_LIN + (int64_t)j * ROWS + r);
        }
        for (int k = 0; k < ND; ++k) {
          const int i = I_ORDER[k];
          lin = fmaf(X[t * XS + NS + i], __ldg(P + O_NUM + i), lin);
        }
        lin += __ldg(P + O_BW);
#pragma unroll
        for (int d = 0; d < DIM; ++d) {
          float s = 0.f, q = 0.f;
          for (int j = 0; j < NF; ++j) {
            const float e = X[t * XS + DIM * j + d];
            s += e;
            q = fmaf(e, e, q);
          }
          S[t * DIM + d] = s;
          fm = fmaf(s, s, fm - q);
          sq += q;
        }
      }
      ls[t] = lin + 0.5f * fm;
      e2[t] = sq;
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
      const float z = ls[r] + s;
      float dz = 0.f, loss = 0.f;
      if (r < n) {
        if (q == 0) a.logits[base + r] = z;
        if (train) {
          const float y = __ldg(a.labels + base + r);
          const float ez = expf(-fabsf(z));  // sigmoid_cross_entropy_with_logits, stable in z
          loss = fmaxf(z, 0.f) - z * y + log1pf(ez);
          const float sig = z >= 0.f ? 1.f / (1.f + ez) : ez / (1.f + ez);
          dz = sig - y;
          loss = fmaf(0.5f * LAMBDA, e2[r], loss);  // l2_loss of this sample's looked-up embeddings
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
        deepctr::add_part(mine + P_NUM + e - N3, s, first);
      } else if (e == N3 + ND) {
        for (int r = 0; r < TILE; ++r) s += dzs[r];
        deepctr::add_part(mine + P_BW, s, first);
      } else {
        for (int r = 0; r < TILE; ++r) s += ls[r];
        deepctr::add_part(mine + P_LOSS, s, first);
      }
    }
    __syncthreads();
    // the DNN's weight gradients; per sample and embedding column, dx + the FM's dz (S_d - e) + lambda e
    deepctr::dnn_backward<Dnn>(X, A1, A2, A3, dzs, D, mine, first, [&](int m, int c, float v) {
      if (m < n) {
        const float e = X[m * XS + c];
        __stcg(w.dx + (base + m) * NS + c, fmaf(LAMBDA, e, fmaf(dzs[m], S[m * DIM + (c & (DIM - 1))] - e, v)));
      }
    });
    if (t < n) __stcg(w.dz + base + t, dzs[t]);
    __syncthreads();
  }
}

// one warp per (table, row): the embedding row's occurrences of dx in perm order, and the linear row's lambda w + its
// occurrences of dz; a row no sample read gets 0 and lambda w
__global__ void __launch_bounds__(THREADS) k_deepctr_deepfm_tables(b200_deepctr_deepfm_args_t a, Work w) {
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
      const int64_t oe = O_EMB + ((int64_t)j * ROWS + r) * DIM, ol = O_LIN + (int64_t)j * ROWS + r;
      const float L = __ldg(P + ol);
      *reinterpret_cast<float4*>(a.grads + oe) = g;
      a.grads[ol] = fmaf(LAMBDA, L, gl);
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

// entry i of the DNN, numeric-weight and bias_weights gradients: the tower CTAs' partials in CTA order (+ lambda w
// for the numeric weights); thread 0 of CTA 0 forms the loss
__global__ void __launch_bounds__(THREADS) k_deepctr_deepfm_reduce(b200_deepctr_deepfm_args_t a, Work w, int grid,
                                                                   int tblocks) {
  const float* __restrict__ P = a.params;
  for (int i = blockIdx.x * THREADS + threadIdx.x; i < P_LOSS; i += gridDim.x * THREADS) {
    float s = deepctr::cta_order_sum(w.parts, Q, grid, i);
    if (i < N_DNN) {
      a.grads[O_DNN + i] = s;
    } else {
      const int64_t o = O_NUM + (i - P_NUM);  // the numeric weights, then bias_weights
      if (i < P_BW) s = fmaf(LAMBDA, __ldg(P + o), s);
      a.grads[o] = s;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    const float ce = deepctr::cta_order_sum(w.parts, Q, grid, P_LOSS);
    float sq = 0.f;
    for (int c = 0; c < tblocks; ++c) sq += __ldcg(w.tparts + c);
    for (int i = 0; i < ND; ++i) sq = fmaf(__ldg(P + O_NUM + i), __ldg(P + O_NUM + i), sq);
    *a.loss = fmaf(0.5f * LAMBDA, sq, ce);
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

int check_args(const b200_deepctr_deepfm_args_t* args, int train) {
  if (!args) return E::fail(-1, "args is null");
  const b200_deepctr_deepfm_args_t& a = *args;
  if (a.B < 1 || a.B > B200_DEEPCTR_DEEPFM_MAX_B)
    return E::fail(-1, "batch size must be in [1, " + std::to_string(B200_DEEPCTR_DEEPFM_MAX_B) + "]");
  if (!a.ids || !a.dense || !a.params || !a.logits || !a.error) return E::fail(-1, "a buffer is null");
  if (train && (!a.labels || !a.loss || !a.grads || !a.workspace)) return E::fail(-1, "a buffer is null");
  if (reinterpret_cast<uintptr_t>(a.params) & 15u) return E::fail(-1, "params must be 16-byte aligned");
  if (train && (reinterpret_cast<uintptr_t>(a.grads) & 15u)) return E::fail(-1, "grads must be 16-byte aligned");
  if (train && (reinterpret_cast<uintptr_t>(a.workspace) & 255u))
    return E::fail(-1, "workspace must be 256-byte aligned");
  return 0;
}

int launch(const b200_deepctr_deepfm_args_t* args, void* stream, int train) {
  if (int rc = check_args(args, train)) return rc;
  const b200_deepctr_deepfm_args_t& a = *args;
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
  if (int rc = E::raise_smem_limit(k_deepctr_deepfm_tower, SMEM_BYTES)) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  if (!train) {
    k_deepctr_deepfm_tower<<<g.tower, THREADS, SMEM_BYTES, st>>>(a, w, ntiles, 0);
    return E::launched("k_deepctr_deepfm_tower", g_launches);
  }
  const dim3 sort_grid(NCH, NF);
  k_deepctr_deepfm_hist<<<sort_grid, SORT_THREADS, 0, st>>>(a.ids, a.B, w.counts);
  if (int rc = E::launched("k_deepctr_deepfm_hist", g_launches)) return rc;
  k_deepctr_deepfm_scatter<<<sort_grid, SORT_THREADS, 0, st>>>(a.ids, a.B, w.counts, w.offsets, w.perm);
  if (int rc = E::launched("k_deepctr_deepfm_scatter", g_launches)) return rc;
  k_deepctr_deepfm_tower<<<g.tower, THREADS, SMEM_BYTES, st>>>(a, w, ntiles, 1);
  if (int rc = E::launched("k_deepctr_deepfm_tower", g_launches)) return rc;
  k_deepctr_deepfm_tables<<<g.tblocks, THREADS, 0, st>>>(a, w);
  if (int rc = E::launched("k_deepctr_deepfm_tables", g_launches)) return rc;
  k_deepctr_deepfm_reduce<<<(P_LOSS + THREADS - 1) / THREADS, THREADS, 0, st>>>(a, w, g.tower, g.tblocks);
  return E::launched("k_deepctr_deepfm_reduce", g_launches);
}

}  // namespace

extern "C" {

const char* b200_deepctr_deepfm_last_error(void) { return E::last_error().c_str(); }
int64_t b200_deepctr_deepfm_launch_count(void) { return g_launches.load(); }

size_t b200_deepctr_deepfm_workspace_bytes(int64_t B) {
  Grid g;
  if (B < 1 || B > B200_DEEPCTR_DEEPFM_MAX_B || grids(B, &g)) return 0;
  return carve(nullptr, B, g.tower, g.tblocks, nullptr);
}

int b200_deepctr_deepfm_tower(const b200_deepctr_deepfm_args_t* args, void* stream) { return launch(args, stream, 1); }
int b200_deepctr_deepfm_forward(const b200_deepctr_deepfm_args_t* args, void* stream) {
  return launch(args, stream, 0);
}

}  // extern "C"
