// What the census (census_tower.cu) and census_model_sqlflow (census_sqlflow_tower.cu) wide & deep towers share.
// Both models have three id groups of four ids each per sample; wide tables over groups 0 and 1 (dim 1), deep
// tables over groups 0..2 (dim 8) feeding Dense 24 -> 16 -> 8 -> 4 without activation; the logit is the wide
// outputs plus the sum of h3; the loss is the mean sigmoid cross-entropy.  They differ in the groups' rows (Shape)
// and in how a group is pooled, which each tower's own file does.
//
// The MLP has no activation and its output is summed, so the backward is linear: with v3 = W3 1, v2 = W2 v3 and
// v1 = W1 v2, a sample's dh2 = dz v3, dh1 = dz v2 and dx = dz v1.  Every gradient is therefore a batch sum of
// scalars times one of these vectors:
//   dW1 = (sum dz x) v2^T, dW2 = (sum dz h1) v3^T, dW3 = (sum dz h2) 1^T, db1 = (sum dz) v2, db2 = (sum dz) v3,
//   db3 = (sum dz) 1, a wide row's gradient = the sum of its occurrences' pooled gradients, and a deep row's
//   gradient = sum over DNN input slots k of (the same sum over its occurrences in slot k) v1[8k .. 8k+8].
// A tower accumulates those 50 dense sums and 5 scalars per (group, row) column -- wide, slots 0..2, occurrences --
// in registers of the threads that own them, sweeping each tile's samples in order; no float atomics, so the
// summation order is fixed.
//
// Grid: at most one CTA per SM, grid-striding over tiles of 256 samples; the whole model is staged in shared
// memory.  Each CTA writes one partial of its sums; the last CTA to arrive adds the partials in CTA order, writes
// the outputs, compacts the touched rows and resets the arrival counter.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "launch.cuh"

namespace census {

constexpr int TILE = 256;     // samples per tile
constexpr int THREADS = 288;  // TILE samples in the forward; the row columns and NDQ dense sums in the sweep
// the MLP block of the flat parameters
constexpr int OW1 = 0, OB1 = 384, OW2 = 400, OB2 = 528, OW3 = 536, OB3 = 568, MLP = 572;
constexpr int NDQ = 50;       // dense sums: dz, dz x[24] @1, dz h1[16] @25, dz h2[8] @41, loss @49
constexpr int CQ = 5;         // per column: wide, slot 0, slot 1, slot 2, occurrences
constexpr int SV = TILE + 1;  // padded: the dense sums read column q of row r conflict-free

// A model's shape: id groups 0, 1, 2 of R0, R1, R2 rows.  Flat parameters [MLP | wide groups 0, 1 (dim 1) | deep
// groups 0, 1, 2 (dim 8)]; tables t = 0..4 are wide groups 0, 1 and deep groups 0..2.
template <int R0, int R1, int R2>
struct Shape {
  static constexpr int WIDE0 = MLP, WIDE1 = WIDE0 + R0, DEEP0 = WIDE1 + R1, NPARAM = DEEP0 + 8 * (R0 + R1 + R2);
  static constexpr int SDEEP = (DEEP0 + 3) / 4 * 4;     // the deep block in shared memory, 16-byte aligned
  static constexpr int SP = SDEEP + (NPARAM - DEEP0);  // floats of the parameters in shared memory
  static constexpr int NCOL = R0 + R1 + R2;            // (group, row) columns: group 1 from COL1, group 2 from COL2
  static constexpr int COL1 = R0, COL2 = R0 + R1;
  static constexpr int Q = NDQ + NCOL * CQ;            // floats of one CTA's partial
  // table t's push_rows segment starts at uniq + UNIQ_OFFt and gsum + GSUM_OFFt (its parameter offset minus MLP)
  static constexpr int UNIQ_OFF1 = R0, UNIQ_OFF2 = R0 + R1, UNIQ_OFF3 = 2 * R0 + R1, UNIQ_OFF4 = 2 * (R0 + R1);
  static constexpr int GSUM_OFF1 = WIDE1 - MLP, GSUM_OFF2 = DEEP0 - MLP, GSUM_OFF3 = GSUM_OFF2 + 8 * R0,
                       GSUM_OFF4 = GSUM_OFF3 + 8 * R1;
  static constexpr int UNIQ_ROWS = UNIQ_OFF4 + R2, GSUM_FLOATS = NPARAM - MLP;
  static_assert(NCOL + NDQ <= THREADS && THREADS / 32 >= 5, "a thread per column and dense sum, a warp per table");

  __device__ static int rows(int g) { return g == 0 ? R0 : (g == 1 ? R1 : R2); }
  __device__ static int deep_soff(int g) { return SDEEP + (g == 0 ? 0 : (g == 1 ? 8 * R0 : 8 * (R0 + R1))); }
};

// ---- device side
// Each kernel stages its parameters and computes the backward's v3, v2, v1 itself: the same code as a helper here
// compiles to different SASS.

// The id group g and sample smp that DNN input slot k of sample b pools.
__device__ __forceinline__ void slot_source(bool quirk, int64_t b, int k, int64_t B, int& g, int64_t& smp) {
  if (quirk) {  // Q11: slot k of row b is stacked row 3b + k of [3, B, 8]
    const int64_t f = 3 * b + k;
    g = (int)(f / B);
    smp = f - g * B;
  } else {
    g = k;
    smp = b;
  }
}

// The MLP of one sample: h1 and h2 of DNN input x, and the logit, wide + the sum of h3.
__device__ __forceinline__ float mlp_forward(const float* p, const float (&x)[24], float wide, float (&h1)[16],
                                             float (&h2)[8]) {
  float h3[4];
#pragma unroll
  for (int j = 0; j < 16; ++j) h1[j] = p[OB1 + j];
#pragma unroll
  for (int i = 0; i < 24; ++i)
#pragma unroll
    for (int j = 0; j < 16; ++j) h1[j] = fmaf(x[i], p[OW1 + i * 16 + j], h1[j]);
#pragma unroll
  for (int j = 0; j < 8; ++j) h2[j] = p[OB2 + j];
#pragma unroll
  for (int i = 0; i < 16; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) h2[j] = fmaf(h1[i], p[OW2 + i * 8 + j], h2[j]);
#pragma unroll
  for (int j = 0; j < 4; ++j) h3[j] = p[OB3 + j];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) h3[j] = fmaf(h2[i], p[OW3 + i * 4 + j], h3[j]);
  return wide + ((h3[0] + h3[1]) + (h3[2] + h3[3]));
}

// One sample's sigmoid cross-entropy with logits z against label y, and p = sigmoid(z): its dz is (p - y) / B.
__device__ __forceinline__ float sample_loss(float z, float y, float& p) {
  const float lb = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
  p = 1.f / (1.f + expf(-z));
  return lb;
}

// Tile row t's values of dense sums 1 .. NDQ - 1: x, h1, h2 and the loss.
__device__ __forceinline__ void put_row(float (*sv)[SV], int t, const float (&x)[24], const float (&h1)[16],
                                        const float (&h2)[8], float lb) {
#pragma unroll
  for (int i = 0; i < 24; ++i) sv[1 + i][t] = x[i];
#pragma unroll
  for (int i = 0; i < 16; ++i) sv[25 + i][t] = h1[i];
#pragma unroll
  for (int i = 0; i < 8; ++i) sv[41 + i][t] = h2[i];
  sv[49][t] = lb;
}

// A thread's part in the sweep: (group, row) column (g, row), or, with g = -1, dense sum dq when dq < NDQ.
struct Column {
  int g, row, dq;
};

template <class S>
__device__ __forceinline__ Column column_of(int t) {
  Column c{-1, 0, t - S::NCOL};
  if (t < S::COL1) {
    c.g = 0;
    c.row = t;
  } else if (t < S::COL2) {
    c.g = 1;
    c.row = t - S::COL1;
  } else if (t < S::NCOL) {
    c.g = 2;
    c.row = t - S::COL2;
  }
  return c;
}

// A thread's sums at the end of the sweep: its column's wide and slot 0..2 sums and occurrences, or its dense sum.
struct Sums {
  float w, s0, s1, s2;
  int occ;
  float q;
};

// Dense sum dq over tile rows 0 .. n-1, added to acc: of dz (dq = 0), of the loss (dq = NDQ - 1), else of dz
// times the rows' values.
__device__ __forceinline__ float dense_sweep(const float* dz, const float (*sv)[SV], int dq, int n, float acc) {
  if (dq == 0) {
    for (int r = 0; r < n; ++r) acc += dz[r];
  } else if (dq == NDQ - 1) {
    for (int r = 0; r < n; ++r) acc += sv[dq][r];
  } else {
    for (int r = 0; r < n; ++r) acc = fmaf(dz[r], sv[dq][r], acc);
  }
  return acc;
}

// After the last tile, in every thread: write this CTA's partial and add `bad` to *a.error.  Without
// reference_reshape (quirk), slot k pools the sample's own group k, so a column's slot sums are its wide sum.  The
// last CTA to arrive adds the partials in CTA order, writes the loss, the MLP gradients and the five tables'
// push_rows segments (touched rows ascending, their count, their gradients) and resets the arrival counter.
template <class S, class Args, class Smem>
__device__ __forceinline__ void finish(const Args& a, Smem& s, Column c, Sums sums, int bad, bool quirk) {
  const int t = threadIdx.x;
  const int64_t B = a.B;
  unsigned* counter = entry::arrival_counter(a.workspace);
  float* parts = entry::partials(a.workspace);
  float* mine = parts + (size_t)blockIdx.x * S::Q;
  if (c.g >= 0) {
    float* col = mine + NDQ + t * CQ;
    col[0] = sums.w;
    col[1] = quirk ? sums.s0 : (c.g == 0 ? sums.w : 0.f);
    col[2] = quirk ? sums.s1 : (c.g == 1 ? sums.w : 0.f);
    col[3] = quirk ? sums.s2 : (c.g == 2 ? sums.w : 0.f);
    col[4] = (float)sums.occ;
  } else if (c.dq < NDQ) {
    mine[c.dq] = sums.q;
  }
  if (bad) atomicAdd(a.error, bad);
  if (!entry::last_to_arrive(counter, s.last)) return;

  float* tot = &s.sv[0][0];
  entry::sum_partials<THREADS>(parts, S::Q, [&](int q, float v) { tot[q] = v; });
  __syncthreads();
  const float* v3 = s.v;
  const float* v2 = s.v + 8;
  const float* v1 = s.v + 24;
  if (t == 0) *a.loss = tot[NDQ - 1] / (float)B;
  for (int i = t; i < MLP; i += THREADS) {
    float g;
    if (i < OB1) g = tot[1 + i / 16] * v2[i % 16];
    else if (i < OW2) g = tot[0] * v2[i - OB1];
    else if (i < OB2) g = tot[25 + (i - OW2) / 8] * v3[(i - OW2) % 8];
    else if (i < OW3) g = tot[0] * v3[i - OB2];
    else if (i < OB3) g = tot[41 + (i - OW3) / 4];
    else g = tot[0];
    a.grads[i] = g;
  }
  const int w = t >> 5, lane = t & 31;
  if (w < 5) {  // table w: wide groups 0, 1 (w = 0, 1), deep groups 0..2 (w = 2..4)
    const int g = w < 2 ? w : w - 2;
    const int rows = S::rows(g);
    const int col0 = g == 0 ? 0 : (g == 1 ? S::COL1 : S::COL2);
    const int uoff = w == 0 ? 0 : w == 1 ? S::UNIQ_OFF1 : w == 2 ? S::UNIQ_OFF2 : w == 3 ? S::UNIQ_OFF3 : S::UNIQ_OFF4;
    const int goff = w == 0 ? 0 : w == 1 ? S::GSUM_OFF1 : w == 2 ? S::GSUM_OFF2 : w == 3 ? S::GSUM_OFF3 : S::GSUM_OFF4;
    int cnt = 0;
    for (int r0 = 0; r0 < rows; r0 += 32) {
      const int row = r0 + lane;
      const float* c = tot + NDQ + (col0 + row) * CQ;
      const bool touched = row < rows && c[4] > 0.f;
      const unsigned m = __ballot_sync(0xffffffffu, touched);
      if (touched) {
        const int pos = cnt + __popc(m & ((1u << lane) - 1u));
        a.uniq[uoff + pos] = row;
        if (w < 2) {
          a.gsum[goff + pos] = c[0];
        } else {
#pragma unroll
          for (int d = 0; d < 8; ++d) a.gsum[goff + pos * 8 + d] = (c[1] * v1[d] + c[2] * v1[8 + d]) + c[3] * v1[16 + d];
        }
      }
      cnt += __popc(m);
    }
    if (lane == 0) a.n_unique[w] = cnt;
  }
  if (t == 0) *counter = 0u;
}

// ---- host side

// At most one CTA per SM.
template <class E>
int grid_for(int64_t B, int* grid) {
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int64_t tiles = (B + TILE - 1) / TILE;
  *grid = (int)(tiles < d.sms ? tiles : d.sms);
  return 0;
}

template <class S, class E>
size_t workspace_bytes(int64_t B) {
  int grid = 0;
  if (B < 1 || grid_for<E>(B, &grid)) return 0;
  return entry::partials_bytes(grid, S::Q);
}

// Check the arguments (train = false: the forward's, which needs no labels, workspace or outputs beyond the
// logits), raise `kernel`'s shared-memory limit to smem and launch it on (*args, the number of tiles, extra...).
template <class S, class E, class Args, class K, class... Extra>
int launch(K* kernel, const char* name, entry::LaunchCount& launches, size_t smem, const Args* args, void* stream,
           bool train, Extra... extra) {
  if (!args) return E::fail(-1, "args is null");
  const Args& a = *args;
  // 12 B ids must be addressable with a 32-bit row stride times 12
  if (a.B < 1 || (int64_t)a.B * 12 > INT32_MAX) return E::fail(-1, "batch size must be in [1, 2^31 / 12)");
  if (a.reference_reshape != 0 && a.reference_reshape != 1) return E::fail(-1, "reference_reshape must be 0 or 1");
  if (!a.ids || !a.params || !a.logits || !a.error) return E::fail(-1, "a buffer is null");
  if (train && (!a.labels || !a.loss || !a.grads || !a.uniq || !a.n_unique || !a.gsum || !a.workspace))
    return E::fail(-1, "a buffer is null");
  int grid = 0;
  if (int rc = grid_for<E>(a.B, &grid)) return rc;
  if (train) {
    const size_t need = entry::partials_bytes(grid, S::Q);
    if (a.workspace_bytes < need)
      return E::fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, batch " + std::to_string(a.B) +
                             " needs " + std::to_string(need));
  }
  if (int rc = E::raise_smem_limit(kernel, smem)) return rc;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  kernel<<<grid, THREADS, smem, (cudaStream_t)stream>>>(a, ntiles, extra...);
  return E::launched(name, launches);
}

}  // namespace census
