// Census wide & deep tower (include/b200_census.h): pooled multi-hot forward, loss, backward, MLP gradients and
// the five compacted push_rows segments in one launch.
//
// The MLP has no activation and its output is summed, so the backward is linear: with v3 = W3 1, v2 = W2 v3 and
// v1 = W1 v2, a sample's dh2 = dz v3, dh1 = dz v2 and dx = dz v1.  Every gradient is therefore a batch sum of
// scalars times one of these vectors:
//   dW1 = (sum dz x) v2^T, dW2 = (sum dz h1) v3^T, dW3 = (sum dz h2) 1^T, db1 = (sum dz) v2, db2 = (sum dz) v3,
//   db3 = (sum dz) 1, a wide row's gradient = the sum of dz over its occurrences, and a deep row's gradient =
//   sum over DNN input slots k of (the sum of dz over its occurrences in slot k) v1[8k .. 8k+8].
// The kernel accumulates those 50 dense sums and 5 scalars per (group, row) -- wide, slots 0..2, occurrences --
// in registers of the threads that own them, sweeping each tile's samples in order; no float atomics, so the
// summation order is fixed.
//
// Grid: at most one CTA per SM, grid-striding over tiles of 256 samples; the whole model (9.7 KB) is staged in
// shared memory.  Each CTA writes one partial of its sums; the last CTA to arrive adds the partials in CTA order,
// writes the outputs, compacts the touched rows and resets the arrival counter.
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_census.h"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::Census>;
entry::LaunchCount g_launches{0};

constexpr int TILE = B200_CENSUS_TILE;
constexpr int THREADS = 288;  // 256 samples in the forward; 218 row columns + 50 dense sums in the sweep
// flat parameter offsets (b200_census.h)
constexpr int OW1 = 0, OB1 = 384, OW2 = 400, OB2 = 528, OW3 = 536, OB3 = 568, MLP = B200_CENSUS_MLP;
constexpr int WIDE0 = 572, WIDE1 = 600, DEEP0 = 675, NPARAM = B200_CENSUS_PARAMS;
constexpr int SDEEP = 676;                 // the deep block in shared memory, 16-byte aligned
constexpr int SP = SDEEP + (NPARAM - DEEP0);  // 2420 floats
constexpr int NCOL = 218;                  // (group, row) columns: group 0 at 0..27, 1 at 28..102, 2 at 103..217
constexpr int NDQ = 50;                    // dense sums: dz, dz x[24] @1, dz h1[16] @25, dz h2[8] @41, loss @49
constexpr int CQ = 5;                      // per column: wide, slot 0, slot 1, slot 2, occurrences
constexpr int Q = NDQ + NCOL * CQ;         // floats of one CTA's partial
constexpr int SV = TILE + 1;               // padded: the dense sums read column q of row r conflict-free

struct Smem {
  int4 ent[3][TILE];   // the four ids of DNN input slot k of tile row r
  int4 own[2][TILE];   // the four ids of wide groups 0 and 1 of tile row r
  float p[SP];         // parameters
  float v[48];         // v3 @0, v2 @8, v1 @24
  int entg[3][TILE];   // the id group of slot k of row r
  float dz[TILE];
  float sv[NDQ][SV];   // per-row values of the dense sums; the last CTA's totals afterwards
  int last;
};

__device__ __forceinline__ int group_rows(int g) { return g == 0 ? 28 : (g == 1 ? 75 : 115); }
__device__ __forceinline__ int deep_soff(int g) { return SDEEP + (g == 0 ? 0 : (g == 1 ? 224 : 824)); }

__device__ __forceinline__ int load_id(const int32_t* ids, int row, int64_t B, int64_t s, int rows, int& bad) {
  int v = __ldg(ids + (size_t)row * B + s);
  if ((unsigned)v >= (unsigned)rows) {
    ++bad;
    v = 0;
  }
  return v;
}

__global__ void __launch_bounds__(THREADS, 1) k_census_tower(b200_census_args_t a, int ntiles) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& s = *reinterpret_cast<Smem*>(smem_raw);
  const int t = threadIdx.x;
  const int64_t B = a.B;
  const bool quirk = a.reference_reshape != 0;
  for (int i = t; i < NPARAM; i += THREADS) s.p[i < DEEP0 ? i : i + (SDEEP - DEEP0)] = __ldg(a.params + i);
  __syncthreads();
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

  int cg = -1, crow = 0;  // this thread's (group, row) column in the sweep
  if (t < 28) {
    cg = 0;
    crow = t;
  } else if (t < 103) {
    cg = 1;
    crow = t - 28;
  } else if (t < NCOL) {
    cg = 2;
    crow = t - 103;
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
        const int rows = group_rows(g);
        int4 e;
        e.x = load_id(a.ids, 4 * g + 0, B, smp, rows, bad);
        e.y = load_id(a.ids, 4 * g + 1, B, smp, rows, bad);
        e.z = load_id(a.ids, 4 * g + 2, B, smp, rows, bad);
        e.w = load_id(a.ids, 4 * g + 3, B, smp, rows, bad);
        s.ent[k][t] = e;
        s.entg[k][t] = g;
        const float4* d = reinterpret_cast<const float4*>(s.p + deep_soff(g));
        const int ids4[4] = {e.x, e.y, e.z, e.w};
        float4 lo = d[2 * ids4[0]], hi = d[2 * ids4[0] + 1];
#pragma unroll
        for (int j = 1; j < 4; ++j) {
          const float4 l2 = d[2 * ids4[j]], h2 = d[2 * ids4[j] + 1];
          lo.x += l2.x; lo.y += l2.y; lo.z += l2.z; lo.w += l2.w;
          hi.x += h2.x; hi.y += h2.y; hi.z += h2.z; hi.w += h2.w;
        }
        x[8 * k + 0] = lo.x; x[8 * k + 1] = lo.y; x[8 * k + 2] = lo.z; x[8 * k + 3] = lo.w;
        x[8 * k + 4] = hi.x; x[8 * k + 5] = hi.y; x[8 * k + 6] = hi.z; x[8 * k + 7] = hi.w;
      }
      float wide = 0.f;
#pragma unroll
      for (int g = 0; g < 2; ++g) {
        int dummy = 0;  // counted once, through the slots above
        const int rows = group_rows(g);
        int4 o;
        o.x = load_id(a.ids, 4 * g + 0, B, b, rows, dummy);
        o.y = load_id(a.ids, 4 * g + 1, B, b, rows, dummy);
        o.z = load_id(a.ids, 4 * g + 2, B, b, rows, dummy);
        o.w = load_id(a.ids, 4 * g + 3, B, b, rows, dummy);
        s.own[g][t] = o;
        const float* w = s.p + (g == 0 ? WIDE0 : WIDE1);
        wide += ((w[o.x] + w[o.y]) + w[o.z]) + w[o.w];
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
      const float y = __ldg(a.labels + b);
      const float lb = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));  // sigmoid cross-entropy with logits
      const float p = 1.f / (1.f + expf(-z));
      a.logits[b] = z;
      s.dz[t] = (p - y) / (float)B;
#pragma unroll
      for (int i = 0; i < 24; ++i) s.sv[1 + i][t] = x[i];
#pragma unroll
      for (int i = 0; i < 16; ++i) s.sv[25 + i][t] = h1[i];
#pragma unroll
      for (int i = 0; i < 8; ++i) s.sv[41 + i][t] = h2[i];
      s.sv[49][t] = lb;
    }
    __syncthreads();
    if (cg >= 0) {
      if (!quirk) {  // slot cg is the sample's own group cg: its sums are the wide sums
        for (int r = 0; r < n; ++r) {
          const int4 e = s.ent[cg][r];
          const float d = s.dz[r];
          if (e.x == crow) { acc_w += d; ++occ; }
          if (e.y == crow) { acc_w += d; ++occ; }
          if (e.z == crow) { acc_w += d; ++occ; }
          if (e.w == crow) { acc_w += d; ++occ; }
        }
      } else {
        for (int r = 0; r < n; ++r) {
          const float d = s.dz[r];
          if (cg < 2) {
            const int4 o = s.own[cg][r];
            if (o.x == crow) acc_w += d;
            if (o.y == crow) acc_w += d;
            if (o.z == crow) acc_w += d;
            if (o.w == crow) acc_w += d;
          }
#define CENSUS_SLOT(K, ACC)                              \
  if (s.entg[K][r] == cg) {                              \
    const int4 e = s.ent[K][r];                          \
    if (e.x == crow) { ACC += d; ++occ; }                \
    if (e.y == crow) { ACC += d; ++occ; }                \
    if (e.z == crow) { ACC += d; ++occ; }                \
    if (e.w == crow) { ACC += d; ++occ; }                \
  }
          CENSUS_SLOT(0, acc_0)
          CENSUS_SLOT(1, acc_1)
          CENSUS_SLOT(2, acc_2)
#undef CENSUS_SLOT
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
  if (w < 5) {  // table w: embedding (w = 0), embedding_1, embedding_2 .. embedding_4 (deep groups 0..2)
    const int g = w < 2 ? w : w - 2;
    const int rows = group_rows(g);
    const int col0 = g == 0 ? 0 : (g == 1 ? 28 : 103);
    const int uoff = w == 0 ? 0 : w == 1 ? 28 : w == 2 ? 103 : w == 3 ? 131 : 206;
    const int goff = w == 0 ? 0 : w == 1 ? 28 : w == 2 ? 103 : w == 3 ? 327 : 927;
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

}  // namespace

extern "C" {

const char* b200_census_last_error(void) { return E::last_error().c_str(); }
int64_t b200_census_launch_count(void) { return g_launches.load(); }

size_t b200_census_workspace_bytes(int64_t B) {
  int grid = 0;
  if (B < 1 || grid_for(B, &grid)) return 0;
  return entry::partials_bytes(grid, Q);
}

int b200_census_tower(const b200_census_args_t* args, void* stream) {
  if (!args) return E::fail(-1, "args is null");
  const b200_census_args_t& a = *args;
  // 12 B ids must be addressable with a 32-bit row stride times 12
  if (a.B < 1 || (int64_t)a.B * 12 > INT32_MAX) return E::fail(-1, "batch size must be in [1, 2^31 / 12)");
  if (a.reference_reshape != 0 && a.reference_reshape != 1) return E::fail(-1, "reference_reshape must be 0 or 1");
  if (!a.ids || !a.labels || !a.params || !a.loss || !a.logits || !a.grads || !a.uniq || !a.n_unique || !a.gsum ||
      !a.error || !a.workspace)
    return E::fail(-1, "a buffer is null");
  int grid = 0;
  if (int rc = grid_for(a.B, &grid)) return rc;
  const size_t need = entry::partials_bytes(grid, Q);
  if (a.workspace_bytes < need)
    return E::fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, batch " + std::to_string(a.B) +
                           " needs " + std::to_string(need));
  const size_t smem = sizeof(Smem);
  if (int rc = E::raise_smem_limit(k_census_tower, smem)) return rc;
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  k_census_tower<<<grid, THREADS, smem, (cudaStream_t)stream>>>(a, ntiles);
  return E::launched("k_census_tower", g_launches);
}

}  // extern "C"
