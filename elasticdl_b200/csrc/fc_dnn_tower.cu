// Feature-column DNN tower (include/b200_fc_dnn.h): DenseFeatures x [F] from numeric columns, bucket one-hots and
// embedding-column rows, Dense(16, relu) -> Dense(16, relu) -> Dense(1, sigmoid), Keras binary cross-entropy on
// the probability, the backward, the MLP gradients and every table's unique-row gradient sums, in one launch.
//
// Grid: at most one CTA per SM, grid-striding over tiles of 64 samples; 256 threads, four per sample in the
// forward and backward (thread q of a sample owns hidden units 4q .. 4q + 3 of both layers).  A sample's x, h1,
// h2, dh1, dh2, dz and loss are one row of the tile matrix S in shared memory; every MLP gradient is a batch sum
// of one product S[r][a] S[r][b] (a = 1 for the biases), owned by one thread that sweeps the tile's rows in
// order.  A table's rows enter x directly, so the gradient of unique row u is W1[block rows]^T applied to the
// sum of dh1 over the samples that read u: thread (table k, hidden unit j) sweeps the tile's rows in order and
// adds dh1[j] into its (u, j) accumulator.  No float atomics: each CTA writes one partial of its sums, the last
// CTA to arrive adds the partials in CTA order, forms the outputs and resets the arrival counter.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_fc_dnn.h"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::FcDnn>;
entry::LaunchCount g_launches{0};

constexpr int H = B200_FC_DNN_HIDDEN;
constexpr int TILE = B200_FC_DNN_TILE;
constexpr int THREADS = 256;
constexpr int MAXT = B200_FC_DNN_MAX_TABLES;
constexpr int NP_MAX = H * B200_FC_DNN_MAX_F + 305;
constexpr int KP = (NP_MAX + 1 + THREADS - 1) / THREADS;  // dense sums per thread (the MLP gradients + the loss)
static_assert(THREADS == 4 * TILE, "four threads per sample");

// What the kernel derives from a checked layout.
struct Plan {
  b200_fc_layout_t L;
  int NP;                // 16 F + 305
  int SR;                // row stride of S (odd, >= F + 67)
  int slots;             // sum of table_rows
  int slot0[MAXT];       // first accumulator slot of table k
  int roff[MAXT];        // float offset of table k in rows / gsum
  int xoff[MAXT];        // first column of table k in x
  int Q;                 // floats of one CTA's partial: NP + 1 dense sums, slots * 16 row sums
  int smem_floats;
};

// columns of a row of S after x [0, F)
__host__ __device__ inline int c_h1(int F) { return F; }
__host__ __device__ inline int c_h2(int F) { return F + H; }
__host__ __device__ inline int c_d1(int F) { return F + 2 * H; }
__host__ __device__ inline int c_d2(int F) { return F + 3 * H; }
__host__ __device__ inline int c_dz(int F) { return F + 4 * H; }
__host__ __device__ inline int c_one(int F) { return F + 4 * H + 1; }
__host__ __device__ inline int c_loss(int F) { return F + 4 * H + 2; }

// shared memory (floats): params [NP rounded to 4] | S [TILE][SR] | R [slots][16] | inv [TILE][MAXT] | cols [F]
__host__ __device__ inline int sm_S(const Plan& p) { return (p.NP + 3) & ~3; }
__host__ __device__ inline int sm_R(const Plan& p) { return sm_S(p) + TILE * p.SR; }
__host__ __device__ inline int sm_inv(const Plan& p) { return sm_R(p) + p.slots * H; }
__host__ __device__ inline int sm_cols(const Plan& p) { return sm_inv(p) + TILE * MAXT; }

__global__ void __launch_bounds__(THREADS, 1) k_fc_dnn_tower(b200_fc_dnn_args_t a, Plan pl, int ntiles, int train) {
  extern __shared__ __align__(16) float sm[];
  const b200_fc_layout_t& L = pl.L;
  const int t = threadIdx.x, q = t & 3, rloc = t >> 2, j0 = 4 * q;
  const int F = L.F, NP = pl.NP, SR = pl.SR;
  const int64_t B = a.B;
  float* P = sm;
  float* S = sm + sm_S(pl);
  float* R = sm + sm_R(pl);
  int* invs = reinterpret_cast<int*>(sm + sm_inv(pl));
  int* cols = reinterpret_cast<int*>(sm + sm_cols(pl));
  __shared__ int last;

  for (int i = t; i < NP; i += THREADS) P[i] = __ldg(a.params + i);
  for (int i = t; i < pl.slots * H; i += THREADS) R[i] = 0.f;
  for (int bi = 0; bi < L.n_blocks; ++bi) {
    const b200_fc_block_t& blk = L.blocks[bi];
    for (int i = t; i < blk.width; i += THREADS) cols[blk.offset + i] = blk.kind | (blk.src << 2) | (i << 10);
  }
  const int OW1 = 0, OB1 = H * F, OW2 = OB1 + H, OB2 = OW2 + H * H, OW3 = OB2 + H, OB3 = OW3 + H;
  const int H1 = c_h1(F), H2 = c_h2(F), D1 = c_d1(F), D2 = c_d2(F), DZ = c_dz(F), ONE = c_one(F), LS = c_loss(F);

  // this thread's dense sums: p = t + 256 k is the product S[r][ca] S[r][cb]; p == NP is the loss sum
  int ca[KP], cb[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    const int p = t + THREADS * k;
    int x = -1, y = -1;
    if (p < OB1) { x = p / H; y = D1 + p % H; }
    else if (p < OW2) { x = ONE; y = D1 + (p - OB1); }
    else if (p < OB2) { x = H1 + (p - OW2) / H; y = D2 + (p - OW2) % H; }
    else if (p < OW3) { x = ONE; y = D2 + (p - OB2); }
    else if (p < OB3) { x = H2 + (p - OW3); y = DZ; }
    else if (p == OB3) { x = ONE; y = DZ; }
    else if (p == NP) { x = ONE; y = LS; }
    ca[k] = x;
    cb[k] = y;
  }
  float acc[KP];
#pragma unroll
  for (int k = 0; k < KP; ++k) acc[k] = 0.f;
  // this thread's row sums: table rk, hidden unit rj
  const int rk = t >> 4, rj = t & (H - 1);
  const bool rowsum = train && rk < L.n_tables;
  __syncthreads();

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = (int64_t)tile * TILE;
    const int n = B - base < TILE ? (int)(B - base) : TILE;
    const bool act = rloc < n;
    const int64_t b = base + rloc;
    float* row = S + rloc * SR;
    // x: the sample's unique row per table (-1: empty string), then its columns
    if (act) {
      for (int k = q; k < L.n_tables; k += 4) {
        const bool empty = __ldg(a.strings + ((int64_t)L.table_string[k] * B + b) * a.W) == 0;
        const int u = __ldg(a.inv + (int64_t)k * B + b);
        invs[rloc * MAXT + k] = (empty || (unsigned)u >= (unsigned)L.table_rows[k]) ? -1 : u;
      }
    }
    __syncthreads();
    if (act) {
      for (int c = q; c < F; c += 4) {
        const int d = cols[c], kind = d & 3, src = (d >> 2) & 255, sub = d >> 10;
        float v;
        if (kind == B200_FC_NUMERIC) {
          v = __ldg(a.numeric + (int64_t)src * B + b);
        } else if (kind == B200_FC_BUCKET) {
          v = __ldg(a.ids + (int64_t)src * B + b) == sub ? 1.f : 0.f;
        } else {
          const int u = invs[rloc * MAXT + src];
          v = u < 0 ? 0.f : __ldg(a.rows + pl.roff[src] + (int64_t)u * L.table_dim[src] + sub);
        }
        row[c] = v;
      }
    }
    __syncthreads();
    // h1 = relu(x W1 + b1), units j0 .. j0 + 3
    float h1[4], h2[4];
    {
      float4 acc4 = *reinterpret_cast<const float4*>(P + OB1 + j0);
      for (int i = 0; i < F; ++i) {
        const float x = row[i];
        const float4 w = *reinterpret_cast<const float4*>(P + OW1 + i * H + j0);
        acc4.x = fmaf(x, w.x, acc4.x);
        acc4.y = fmaf(x, w.y, acc4.y);
        acc4.z = fmaf(x, w.z, acc4.z);
        acc4.w = fmaf(x, w.w, acc4.w);
      }
      h1[0] = fmaxf(acc4.x, 0.f); h1[1] = fmaxf(acc4.y, 0.f); h1[2] = fmaxf(acc4.z, 0.f); h1[3] = fmaxf(acc4.w, 0.f);
      if (act) {
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) row[H1 + j0 + jj] = h1[jj];
      }
    }
    __syncthreads();
    float z;
    {
      float4 acc4 = *reinterpret_cast<const float4*>(P + OB2 + j0);
#pragma unroll
      for (int i = 0; i < H; ++i) {
        const float x = row[H1 + i];
        const float4 w = *reinterpret_cast<const float4*>(P + OW2 + i * H + j0);
        acc4.x = fmaf(x, w.x, acc4.x);
        acc4.y = fmaf(x, w.y, acc4.y);
        acc4.z = fmaf(x, w.z, acc4.z);
        acc4.w = fmaf(x, w.w, acc4.w);
      }
      h2[0] = fmaxf(acc4.x, 0.f); h2[1] = fmaxf(acc4.y, 0.f); h2[2] = fmaxf(acc4.z, 0.f); h2[3] = fmaxf(acc4.w, 0.f);
      float zp = fmaf(h2[0], P[OW3 + j0], fmaf(h2[1], P[OW3 + j0 + 1], fmaf(h2[2], P[OW3 + j0 + 2], h2[3] * P[OW3 + j0 + 3])));
      zp += __shfl_xor_sync(0xffffffffu, zp, 1);  // the same sum in all four lanes: + is commutative
      zp += __shfl_xor_sync(0xffffffffu, zp, 2);
      z = zp + P[OB3];
    }
    if (act && q == 0) a.logits[b] = z;
    if (!train) continue;  // uniform: the forward form has no further barrier in the tile
    float dz = 0.f;
    if (act) {
      const float y = __ldg(a.labels + b);
      const float p = 1.f / (1.f + expf(-z));
      const float eps = 1e-7f, hi = 1.f - eps;  // Keras backend.epsilon(), clip_by_value(output, eps, 1 - eps)
      const float pc = fminf(fmaxf(p, eps), hi);
      const float lo = logf(pc + eps), l1 = logf(1.f - pc + eps);
      const float loss = -(y * lo + (1.f - y) * l1);
      if (p >= eps && p <= hi) {  // the clip passes the gradient only inside [eps, 1 - eps]
        const float dldp = -(y / (pc + eps) - (1.f - y) / (1.f - pc + eps));
        dz = dldp * (p * (1.f - p));
        if (L.loss_mean) dz = dz / (float)B;
      }
      if (q == 0) {
        row[DZ] = dz;
        row[ONE] = 1.f;
        row[LS] = loss;
      }
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        row[H2 + j0 + jj] = h2[jj];
        row[D2 + j0 + jj] = h2[jj] > 0.f ? dz * P[OW3 + j0 + jj] : 0.f;
      }
    }
    __syncthreads();
    if (act) {
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        float s = 0.f;
#pragma unroll
        for (int k = 0; k < H; ++k) s = fmaf(P[OW2 + (j0 + jj) * H + k], row[D2 + k], s);
        row[D1 + j0 + jj] = h1[jj] > 0.f ? s : 0.f;
      }
    }
    __syncthreads();
    // the tile's dense sums and row sums, rows in order
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      if (ca[k] >= 0) {
        const float* sa = S + ca[k];
        const float* sb = S + cb[k];
        float s = acc[k];
        for (int r = 0; r < n; ++r) s = fmaf(sa[r * SR], sb[r * SR], s);
        acc[k] = s;
      }
    }
    if (rowsum) {
      float* racc = R + pl.slot0[rk] * H + rj;
      for (int r = 0; r < n; ++r) {
        const int u = invs[r * MAXT + rk];
        if (u >= 0) racc[u * H] += S[r * SR + D1 + rj];
      }
    }
    __syncthreads();
  }
  if (!train) return;

  unsigned* counter = entry::arrival_counter(a.workspace);
  float* parts = entry::partials(a.workspace);
  float* mine = parts + (size_t)blockIdx.x * pl.Q;
#pragma unroll
  for (int k = 0; k < KP; ++k) {
    const int p = t + THREADS * k;
    if (p <= NP) mine[p] = acc[k];
  }
  for (int i = t; i < pl.slots * H; i += THREADS) mine[NP + 1 + i] = R[i];
  if (!entry::last_to_arrive(counter, last)) return;

  // totals: the dense sums into S, the row sums into R
  entry::sum_partials<THREADS>(parts, pl.Q, [&](int i, float s) {
    if (i <= NP) S[i] = s;
    else R[i - NP - 1] = s;
  });
  __syncthreads();
  for (int i = t; i < NP; i += THREADS) a.grads[i] = S[i];
  if (t == 0) {
    *a.loss = L.loss_mean ? S[NP] / (float)B : S[NP];
    *counter = 0u;
  }
  for (int k = 0; k < L.n_tables; ++k) {
    const int dim = L.table_dim[k];
    int nu = a.n_unique[k];
    nu = nu < 0 ? 0 : (nu > L.table_rows[k] ? L.table_rows[k] : nu);
    const float* W = P + OW1 + pl.xoff[k] * H;
    for (int e = t; e < nu * dim; e += THREADS) {
      const int u = e / dim, d = e - u * dim;
      const float* rs = R + (pl.slot0[k] + u) * H;
      float g = 0.f;
#pragma unroll
      for (int j = 0; j < H; ++j) g = fmaf(W[d * H + j], rs[j], g);
      a.gsum[pl.roff[k] + e] = g;
    }
  }
}

__global__ void k_fc_dnn_fill_empty(b200_fc_layout_t L, int32_t* ids, const uint8_t* strings, int64_t B, int W) {
  const int64_t n = (int64_t)L.n_tables * B;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / B);
    const int64_t b = i - k * B;
    if (__ldg(strings + ((int64_t)L.table_string[k] * B + b) * W) == 0) ids[i] = 0;
  }
}

// at most one CTA per SM
int grid_for(int64_t B, int* grid) {
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int64_t tiles = (B + TILE - 1) / TILE;
  *grid = (int)(tiles < d.sms ? tiles : d.sms);
  return 0;
}

// Check a layout and derive its plan; "" when it is sound.
std::string make_plan(const b200_fc_layout_t* layout, Plan* out) {
  if (!layout) return "layout is null";
  const b200_fc_layout_t& L = *layout;
  if (L.F < 1 || L.F > B200_FC_DNN_MAX_F) return "F must be in [1, " + std::to_string(B200_FC_DNN_MAX_F) + "]";
  if (L.n_blocks < 1 || L.n_blocks > B200_FC_DNN_MAX_BLOCKS) return "n_blocks must be in [1, 16]";
  if (L.n_tables < 0 || L.n_tables > MAXT) return "n_tables must be in [0, 8]";
  if (L.loss_mean != 0 && L.loss_mean != 1) return "loss_mean must be 0 or 1";
  Plan p{};
  p.L = L;
  int slots = 0, roff = 0;
  for (int k = 0; k < L.n_tables; ++k) {
    if (L.table_rows[k] < 1 || L.table_dim[k] < 1 || L.table_string[k] < 0)
      return "table " + std::to_string(k) + ": rows and dim must be >= 1, the string column >= 0";
    p.slot0[k] = slots;
    p.roff[k] = roff;
    p.xoff[k] = -1;
    slots += L.table_rows[k];
    roff += L.table_rows[k] * L.table_dim[k];
    if (slots > B200_FC_DNN_MAX_SLOTS) return "the tables have more than 512 rows in all";
  }
  unsigned char cover[B200_FC_DNN_MAX_F] = {0};
  for (int bi = 0; bi < L.n_blocks; ++bi) {
    const b200_fc_block_t& b = L.blocks[bi];
    const std::string who = "block " + std::to_string(bi) + ": ";
    if (b.width < 1 || b.offset < 0 || b.offset + b.width > L.F) return who + "columns outside [0, F)";
    if (b.src < 0 || b.src > 255) return who + "src must be in [0, 255]";
    if (b.kind == B200_FC_NUMERIC) {
      if (b.width != 1) return who + "a numeric column is 1 wide";
    } else if (b.kind == B200_FC_EMBEDDING) {
      if (b.src >= L.n_tables) return who + "no such table";
      if (b.width != L.table_dim[b.src]) return who + "width must be the table's dim";
      if (p.xoff[b.src] >= 0) return who + "a table feeds one block";
      p.xoff[b.src] = b.offset;
    } else if (b.kind != B200_FC_BUCKET) {
      return who + "unknown kind";
    }
    for (int i = 0; i < b.width; ++i)
      if (cover[b.offset + i]++) return who + "overlaps another block";
  }
  for (int c = 0; c < L.F; ++c)
    if (!cover[c]) return "column " + std::to_string(c) + " of x is in no block";
  for (int k = 0; k < L.n_tables; ++k)
    if (p.xoff[k] < 0) return "table " + std::to_string(k) + " feeds no block";
  p.NP = H * L.F + 305;
  p.SR = (L.F + 4 * H + 3) | 1;
  p.slots = slots;
  p.Q = p.NP + 1 + slots * H;
  p.smem_floats = sm_cols(p) + L.F;
  *out = p;
  return "";
}

int check_args(const Plan& p, const b200_fc_dnn_args_t* args, int train) {
  if (!args) return E::fail(-1, "args is null");
  const b200_fc_dnn_args_t& a = *args;
  const b200_fc_layout_t& L = p.L;
  if (a.B < 1 || a.B > INT32_MAX) return E::fail(-1, "batch size must be in [1, 2^31)");
  if (a.W < 1 || a.n_numeric < 0 || a.n_ids < 0 || a.n_strings < 0) return E::fail(-1, "bad input shape");
  for (int bi = 0; bi < L.n_blocks; ++bi) {
    const b200_fc_block_t& b = L.blocks[bi];
    if (b.kind == B200_FC_NUMERIC && b.src >= a.n_numeric) return E::fail(-1, "a numeric block reads a missing row");
    if (b.kind == B200_FC_BUCKET && b.src >= a.n_ids) return E::fail(-1, "a bucket block reads a missing ids row");
  }
  for (int k = 0; k < L.n_tables; ++k)
    if (L.table_string[k] >= a.n_strings) return E::fail(-1, "a table's string column is missing");
  const bool need_num = a.n_numeric > 0, need_ids = a.n_ids > 0, need_tab = L.n_tables > 0;
  if ((need_num && !a.numeric) || (need_ids && !a.ids) || (need_tab && (!a.strings || !a.inv || !a.rows)) ||
      !a.params || !a.logits)
    return E::fail(-1, "a buffer is null");
  if (train && (!a.labels || !a.loss || !a.grads || !a.workspace || (need_tab && (!a.n_unique || !a.gsum))))
    return E::fail(-1, "a buffer is null");
  return 0;
}

int launch(const b200_fc_layout_t* layout, const b200_fc_dnn_args_t* args, void* stream, int train) {
  Plan p;
  const std::string why = make_plan(layout, &p);
  if (!why.empty()) return E::fail(-1, why);
  int rc = check_args(p, args, train);
  if (rc) return rc;
  const b200_fc_dnn_args_t& a = *args;
  if (reinterpret_cast<uintptr_t>(a.params) & 3u) return E::fail(-1, "params must be 4-byte aligned");
  int grid = 0;
  if (int rc = grid_for(a.B, &grid)) return rc;
  if (train) {
    const size_t need = entry::partials_bytes(grid, p.Q);
    if (a.workspace_bytes < need)
      return E::fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, batch " + std::to_string(a.B) +
                             " needs " + std::to_string(need));
  }
  const int smem = p.smem_floats * (int)sizeof(float);
  if (int rc = E::raise_smem_limit(k_fc_dnn_tower, smem)) return rc;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  k_fc_dnn_tower<<<grid, THREADS, smem, (cudaStream_t)stream>>>(a, p, ntiles, train);
  return E::launched("k_fc_dnn_tower", g_launches);
}

}  // namespace

extern "C" {

const char* b200_fc_dnn_last_error(void) { return E::last_error().c_str(); }
int64_t b200_fc_dnn_launch_count(void) { return g_launches.load(); }

int64_t b200_fc_dnn_params(const b200_fc_layout_t* layout) {
  Plan p;
  const std::string why = make_plan(layout, &p);
  if (!why.empty()) return E::fail(0, why);
  return p.NP;
}

size_t b200_fc_dnn_workspace_bytes(const b200_fc_layout_t* layout, int64_t B) {
  Plan p;
  int grid = 0;
  if (B < 1 || !make_plan(layout, &p).empty() || grid_for(B, &grid)) return 0;
  return entry::partials_bytes(grid, p.Q);
}

int b200_fc_dnn_fill_empty(const b200_fc_layout_t* layout, int32_t* ids, const uint8_t* strings, int64_t B, int W,
                           void* stream) {
  Plan p;
  const std::string why = make_plan(layout, &p);
  if (!why.empty()) return E::fail(-1, why);
  if (B < 1 || W < 1) return E::fail(-1, "batch size and string width must be >= 1");
  if (p.L.n_tables == 0) return 0;
  if (!ids || !strings) return E::fail(-1, "a buffer is null");
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int64_t n = (int64_t)p.L.n_tables * B;
  const int64_t want = (n + 255) / 256;
  const int grid = (int)(want < 4 * d.sms ? want : 4 * d.sms);
  k_fc_dnn_fill_empty<<<grid, 256, 0, (cudaStream_t)stream>>>(p.L, ids, strings, B, W);
  return E::launched("k_fc_dnn_fill_empty", g_launches, 0);
}

int b200_fc_dnn_tower(const b200_fc_layout_t* layout, const b200_fc_dnn_args_t* args, void* stream) {
  return launch(layout, args, stream, 1);
}
int b200_fc_dnn_forward(const b200_fc_layout_t* layout, const b200_fc_dnn_args_t* args, void* stream) {
  return launch(layout, args, stream, 0);
}

}  // extern "C"
