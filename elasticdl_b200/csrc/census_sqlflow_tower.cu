// census_model_sqlflow wide & deep tower (include/b200_census_sqlflow.h): mean-pooled sparse lookups over the
// present ids, forward, loss, backward, MLP gradients and the five compacted push_rows segments in one launch.
//
// The census tower's linear backward (csrc/census_tower.cu) with a per-sample divisor: the MLP has no activation
// and its output is summed, so with v3 = W3 1, v2 = W2 v3 and v1 = W1 v2 every gradient is a batch sum of scalars
// times a fixed vector.  A pooled vector is the mean over n_g(s) present ids, so where the census tower adds dz
// to a (group, row) column per occurrence, this one adds dz / n_g(s):
//   wide row r of group g:  sum over samples b and occurrences of r among b's present ids of dz(b) / n_g(b)
//   deep row r of group g:  sum over DNN input slots k of (the same sum over the samples s slot k reads) v1[8k..]
// A group with no present id pools to zero and touches no row.  The kernel accumulates 50 dense sums and 5
// scalars per (group, row) -- wide, slots 0..2, occurrences -- in registers of the threads that own them,
// sweeping each tile's samples in order; no float atomics, so the summation order is fixed.
//
// Grid: at most one CTA per SM, grid-striding over tiles of 256 samples; the whole model (9.5 KB) is staged in
// shared memory.  Each CTA writes one partial of its sums; the last CTA to arrive adds the partials in CTA order,
// writes the outputs, compacts the touched rows and resets the arrival counter.  The forward form stops after
// the logits.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_census_sqlflow.h"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::CensusSqlflow>;
entry::LaunchCount g_launches{0};

constexpr int TILE = B200_CSQL_TILE;
constexpr int THREADS = 288;  // 256 samples in the forward; 213 row columns + 50 dense sums in the sweep
// flat parameter offsets (b200_census_sqlflow.h)
constexpr int OW1 = 0, OB1 = 384, OW2 = 400, OB2 = 528, OW3 = 536, OB3 = 568, MLP = B200_CSQL_MLP;
constexpr int WIDE0 = 572, WIDE1 = 599, DEEP0 = 672, NPARAM = B200_CSQL_PARAMS;
static_assert(DEEP0 % 4 == 0, "the deep block is read as float4 from shared memory");
constexpr int NCOL = 213;  // (group, row) columns: group 0 at 0..26, 1 at 27..99, 2 at 100..212
constexpr int NDQ = 50;    // dense sums: dz, dz x[24] @1, dz h1[16] @25, dz h2[8] @41, loss @49
constexpr int CQ = 5;      // per column: wide, slot 0, slot 1, slot 2, occurrences
constexpr int Q = NDQ + NCOL * CQ;  // floats of one CTA's partial
constexpr int SV = TILE + 1;        // padded: the dense sums read column q of row r conflict-free

struct Smem {
  int4 ent[3][TILE];   // the four ids of DNN input slot k of tile row r (-1 = absent)
  int4 own[2][TILE];   // the four ids of wide groups 0 and 1 of tile row r
  float p[NPARAM];     // parameters
  float v[48];         // v3 @0, v2 @8, v1 @24
  int entg[3][TILE];   // the id group of slot k of row r
  float ds[3][TILE];   // dz of row r over the present-id count of slot k's group and sample (0 when none)
  float dw[2][TILE];   // dz of row r over the present-id count of its own wide group g (0 when none)
  float dz[TILE];
  float sv[NDQ][SV];   // per-row values of the dense sums; the last CTA's totals afterwards
  int last;
};

__device__ __forceinline__ int group_rows(int g) { return g == 0 ? 27 : (g == 1 ? 73 : 113); }
__device__ __forceinline__ int deep_off(int g) { return g == 0 ? DEEP0 : (g == 1 ? 888 : 1472); }

// -1 for an absent id; an id outside [-1, rows) is counted in `bad` and read as absent
__device__ __forceinline__ int load_id(const int32_t* ids, int row, int64_t B, int64_t s, int rows, int& bad) {
  int v = __ldg(ids + (size_t)row * B + s);
  if (v < -1 || v >= rows) {
    ++bad;
    v = -1;
  }
  return v;
}

__device__ __forceinline__ int4 load_group(const int32_t* ids, int g, int64_t B, int64_t s, int& bad) {
  const int rows = group_rows(g);
  int4 e;
  e.x = load_id(ids, 4 * g + 0, B, s, rows, bad);
  e.y = load_id(ids, 4 * g + 1, B, s, rows, bad);
  e.z = load_id(ids, 4 * g + 2, B, s, rows, bad);
  e.w = load_id(ids, 4 * g + 3, B, s, rows, bad);
  return e;
}

__device__ __forceinline__ int present(int4 e) { return (e.x >= 0) + (e.y >= 0) + (e.z >= 0) + (e.w >= 0); }

__global__ void __launch_bounds__(THREADS, 1) k_census_sqlflow_tower(b200_csql_args_t a, int ntiles, int train) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int t = threadIdx.x;
  const int64_t B = a.B;
  const bool quirk = a.reference_reshape != 0;
  for (int i = t; i < NPARAM; i += THREADS) s.p[i] = __ldg(a.params + i);
  __syncthreads();
  if (train) {
    if (t < 8) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) acc += s.p[OW3 + t * 4 + k];
      s.v[t] = acc;
    }
    __syncthreads();
    if (t < 16) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc = fmaf(s.p[OW2 + t * 8 + j], s.v[j], acc);
      s.v[8 + t] = acc;
    }
    __syncthreads();
    if (t < 24) {
      float acc = 0.f;
#pragma unroll
      for (int j = 0; j < 16; ++j) acc = fmaf(s.p[OW1 + t * 16 + j], s.v[8 + j], acc);
      s.v[24 + t] = acc;
    }
  }

  int cg = -1, crow = 0;  // this thread's (group, row) column in the sweep
  if (t < 27) {
    cg = 0;
    crow = t;
  } else if (t < 100) {
    cg = 1;
    crow = t - 27;
  } else if (t < NCOL) {
    cg = 2;
    crow = t - 100;
  }
  const int dq = t - NCOL;  // this thread's dense sum when 0 <= dq < NDQ
  float acc_w = 0.f, acc_0 = 0.f, acc_1 = 0.f, acc_2 = 0.f, acc_q = 0.f;
  int occ = 0, bad = 0;

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = (int64_t)tile * TILE;
    const int n = B - base < TILE ? (int)(B - base) : TILE;
    if (t < n) {
      const int64_t b = base + t;
      float x[24];
      int cnt[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int g;
        int64_t smp;
        if (quirk) {  // Q11: slot k of row b is stacked row 3b + k of [3, B, 8]
          const int64_t f = 3 * b + k;
          g = (int)(f / B);
          smp = f - g * B;
        } else {
          g = k;
          smp = b;
        }
        const int4 e = load_group(a.ids, g, B, smp, bad);
        const float4* d = reinterpret_cast<const float4*>(s.p + deep_off(g));
        const int ids4[4] = {e.x, e.y, e.z, e.w};
        float4 lo = make_float4(0.f, 0.f, 0.f, 0.f), hi = lo;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (ids4[j] < 0) continue;
          const float4 l2 = d[2 * ids4[j]], h2 = d[2 * ids4[j] + 1];
          lo.x += l2.x; lo.y += l2.y; lo.z += l2.z; lo.w += l2.w;
          hi.x += h2.x; hi.y += h2.y; hi.z += h2.z; hi.w += h2.w;
        }
        cnt[k] = present(e);
        const float c = cnt[k] ? (float)cnt[k] : 1.f;  // an empty group's sum is already zero
        x[8 * k + 0] = lo.x / c; x[8 * k + 1] = lo.y / c; x[8 * k + 2] = lo.z / c; x[8 * k + 3] = lo.w / c;
        x[8 * k + 4] = hi.x / c; x[8 * k + 5] = hi.y / c; x[8 * k + 6] = hi.z / c; x[8 * k + 7] = hi.w / c;
        if (train) {
          s.ent[k][t] = e;
          s.entg[k][t] = g;
        }
      }
      float wide = 0.f;
      int wcnt[2];
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        int dummy = 0;  // counted once, through the slots above
        const int4 o = load_group(a.ids, g, B, b, dummy);
        const float* w = s.p + (g == 0 ? WIDE0 : WIDE1);
        float sum = 0.f;
        if (o.x >= 0) sum += w[o.x];
        if (o.y >= 0) sum += w[o.y];
        if (o.z >= 0) sum += w[o.z];
        if (o.w >= 0) sum += w[o.w];
        wcnt[g] = present(o);
        wide += sum / (wcnt[g] ? (float)wcnt[g] : 1.f);
        if (train) s.own[g][t] = o;
      }
      float h1[16], h2[8], h3[4];
#pragma unroll
      for (int j = 0; j < 16; ++j) h1[j] = s.p[OB1 + j];
#pragma unroll
      for (int i = 0; i < 24; ++i)
#pragma unroll
        for (int j = 0; j < 16; ++j) h1[j] = fmaf(x[i], s.p[OW1 + i * 16 + j], h1[j]);
#pragma unroll
      for (int j = 0; j < 8; ++j) h2[j] = s.p[OB2 + j];
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) h2[j] = fmaf(h1[i], s.p[OW2 + i * 8 + j], h2[j]);
#pragma unroll
      for (int j = 0; j < 4; ++j) h3[j] = s.p[OB3 + j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) h3[j] = fmaf(h2[i], s.p[OW3 + i * 4 + j], h3[j]);
      const float z = wide + ((h3[0] + h3[1]) + (h3[2] + h3[3]));
      a.logits[b] = z;
      if (train) {
        const float y = __ldg(a.labels + b);
        const float lb = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));  // sigmoid cross-entropy with logits
        const float p = 1.f / (1.f + expf(-z));
        const float dzb = (p - y) / (float)B;
        s.dz[t] = dzb;
#pragma unroll
        for (int k = 0; k < 3; ++k) s.ds[k][t] = cnt[k] ? dzb / (float)cnt[k] : 0.f;
#pragma unroll
        for (int g = 0; g < 2; ++g) s.dw[g][t] = wcnt[g] ? dzb / (float)wcnt[g] : 0.f;
#pragma unroll
        for (int i = 0; i < 24; ++i) s.sv[1 + i][t] = x[i];
#pragma unroll
        for (int i = 0; i < 16; ++i) s.sv[25 + i][t] = h1[i];
#pragma unroll
        for (int i = 0; i < 8; ++i) s.sv[41 + i][t] = h2[i];
        s.sv[49][t] = lb;
      }
    }
    if (!train) continue;  // uniform: the forward form has no sweep and no barrier in the tile
    __syncthreads();
    if (cg >= 0) {
      if (!quirk) {  // slot cg is the sample's own group cg: its sums are the wide sums
        for (int r = 0; r < n; ++r) {
          const int4 e = s.ent[cg][r];
          const float d = s.ds[cg][r];
          if (e.x == crow) { acc_w += d; ++occ; }
          if (e.y == crow) { acc_w += d; ++occ; }
          if (e.z == crow) { acc_w += d; ++occ; }
          if (e.w == crow) { acc_w += d; ++occ; }
        }
      } else {
        for (int r = 0; r < n; ++r) {
          if (cg < 2) {
            const int4 o = s.own[cg][r];
            const float d = s.dw[cg][r];
            if (o.x == crow) acc_w += d;
            if (o.y == crow) acc_w += d;
            if (o.z == crow) acc_w += d;
            if (o.w == crow) acc_w += d;
          }
#define CSQL_SLOT(K, ACC)                                \
  if (s.entg[K][r] == cg) {                              \
    const int4 e = s.ent[K][r];                          \
    const float d = s.ds[K][r];                          \
    if (e.x == crow) { ACC += d; ++occ; }                \
    if (e.y == crow) { ACC += d; ++occ; }                \
    if (e.z == crow) { ACC += d; ++occ; }                \
    if (e.w == crow) { ACC += d; ++occ; }                \
  }
          CSQL_SLOT(0, acc_0)
          CSQL_SLOT(1, acc_1)
          CSQL_SLOT(2, acc_2)
#undef CSQL_SLOT
        }
      }
    } else if (dq < NDQ) {
      if (dq == 0) {
        for (int r = 0; r < n; ++r) acc_q += s.dz[r];
      } else if (dq == NDQ - 1) {
        for (int r = 0; r < n; ++r) acc_q += s.sv[dq][r];
      } else {
        for (int r = 0; r < n; ++r) acc_q = fmaf(s.dz[r], s.sv[dq][r], acc_q);
      }
    }
    __syncthreads();
  }
  if (!train) {
    if (bad) atomicAdd(a.error, bad);
    return;
  }

  unsigned* counter = entry::arrival_counter(a.workspace);
  float* parts = entry::partials(a.workspace);
  float* mine = parts + (size_t)blockIdx.x * Q;
  if (cg >= 0) {
    float* c = mine + NDQ + t * CQ;
    c[0] = acc_w;
    c[1] = quirk ? acc_0 : (cg == 0 ? acc_w : 0.f);
    c[2] = quirk ? acc_1 : (cg == 1 ? acc_w : 0.f);
    c[3] = quirk ? acc_2 : (cg == 2 ? acc_w : 0.f);
    c[4] = (float)occ;
  } else if (dq < NDQ) {
    mine[dq] = acc_q;
  }
  if (bad) atomicAdd(a.error, bad);
  if (!entry::last_to_arrive(counter, s.last)) return;

  float* tot = &s.sv[0][0];
  entry::sum_partials<THREADS>(parts, Q, [&](int q, float v) { tot[q] = v; });
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
    const int rows = group_rows(g);
    const int col0 = g == 0 ? 0 : (g == 1 ? 27 : 100);
    const int uoff = w == 0 ? 0 : w == 1 ? 27 : w == 2 ? 100 : w == 3 ? 127 : 200;
    const int goff = w == 0 ? 0 : w == 1 ? 27 : w == 2 ? 100 : w == 3 ? 316 : 900;
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

// at most one CTA per SM
int grid_for(int64_t B, int* grid) {
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int64_t tiles = (B + TILE - 1) / TILE;
  *grid = (int)(tiles < d.sms ? tiles : d.sms);
  return 0;
}

int launch(const b200_csql_args_t* args, void* stream, int train) {
  if (!args) return E::fail(-1, "args is null");
  const b200_csql_args_t& a = *args;
  // 12 B ids must be addressable with a 32-bit row stride times 12
  if (a.B < 1 || (int64_t)a.B * 12 > INT32_MAX) return E::fail(-1, "batch size must be in [1, 2^31 / 12)");
  if (a.reference_reshape != 0 && a.reference_reshape != 1) return E::fail(-1, "reference_reshape must be 0 or 1");
  if (!a.ids || !a.params || !a.logits || !a.error) return E::fail(-1, "a buffer is null");
  if (train && (!a.labels || !a.loss || !a.grads || !a.uniq || !a.n_unique || !a.gsum || !a.workspace))
    return E::fail(-1, "a buffer is null");
  int grid = 0;
  if (int rc = grid_for(a.B, &grid)) return rc;
  if (train) {
    const size_t need = entry::partials_bytes(grid, Q);
    if (a.workspace_bytes < need)
      return E::fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, batch " + std::to_string(a.B) +
                             " needs " + std::to_string(need));
  }
  const size_t smem = sizeof(Smem);
  if (int rc = E::raise_smem_limit(k_census_sqlflow_tower, smem)) return rc;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  k_census_sqlflow_tower<<<grid, THREADS, smem, (cudaStream_t)stream>>>(a, ntiles, train);
  return E::launched("k_census_sqlflow_tower", g_launches);
}

}  // namespace

extern "C" {

const char* b200_csql_last_error(void) { return E::last_error().c_str(); }
int64_t b200_csql_launch_count(void) { return g_launches.load(); }

size_t b200_csql_workspace_bytes(int64_t B) {
  int grid = 0;
  if (B < 1 || grid_for(B, &grid)) return 0;
  return entry::partials_bytes(grid, Q);
}

int b200_csql_tower(const b200_csql_args_t* args, void* stream) { return launch(args, stream, 1); }
int b200_csql_forward(const b200_csql_args_t* args, void* stream) { return launch(args, stream, 0); }

}  // extern "C"
