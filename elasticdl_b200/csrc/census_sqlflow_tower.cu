// census_model_sqlflow wide & deep tower (include/b200_census_sqlflow.h): mean-pooled sparse lookups over the
// present ids, forward, loss, backward, MLP gradients and the five compacted push_rows segments in one launch, on
// the machinery of census_tower.cuh.
//
// A pooled vector is the mean over the n_g(s) present ids of its group and sample, so where the census tower adds
// dz to a (group, row) column per occurrence, this one adds dz / n_g(s):
//   wide row r of group g:  sum over samples b and occurrences of r among b's present ids of dz(b) / n_g(b)
//   deep row r of group g:  sum over DNN input slots k of (the same sum over the samples s slot k reads) v1[8k..]
// A group with no present id pools to zero and touches no row.  The whole model (9.5 KB) is staged in shared
// memory.  The forward form stops after the logits.
#include "../../include/b200_census_sqlflow.h"
#include "census_tower.cuh"

namespace {

using namespace census;
using E = entry::Entry<entry::CensusSqlflow>;
using S = Shape<27, 73, 113>;
static_assert(S::NPARAM == B200_CSQL_PARAMS && MLP == B200_CSQL_MLP && S::UNIQ_ROWS == B200_CSQL_UNIQ_ROWS &&
                  S::GSUM_FLOATS == B200_CSQL_GSUM_FLOATS && TILE == B200_CSQL_TILE,
              "include/b200_census_sqlflow.h");
static_assert(S::SDEEP == S::DEEP0, "the parameters are staged as they are");
entry::LaunchCount g_launches{0};

struct Smem {
  int4 ent[3][TILE];   // the four ids of DNN input slot k of tile row r (-1 = absent)
  int4 own[2][TILE];   // the four ids of wide groups 0 and 1 of tile row r
  float p[S::SP];      // parameters
  float v[48];         // v3 @0, v2 @8, v1 @24
  int entg[3][TILE];   // the id group of slot k of row r
  float ds[3][TILE];   // dz of row r over the present-id count of slot k's group and sample (0 when none)
  float dw[2][TILE];   // dz of row r over the present-id count of its own wide group g (0 when none)
  float dz[TILE];
  float sv[NDQ][SV];   // per-row values of the dense sums; the last CTA's totals afterwards
  int last;
};

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
  const int rows = S::rows(g);
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
  for (int i = t; i < S::NPARAM; i += THREADS) s.p[i] = __ldg(a.params + i);
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

  const Column col = column_of<S>(t);
  const int cg = col.g, crow = col.row;
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
        slot_source(quirk, b, k, B, g, smp);
        const int4 e = load_group(a.ids, g, B, smp, bad);
        const float4* d = reinterpret_cast<const float4*>(s.p + S::deep_soff(g));
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
        const float* w = s.p + (g == 0 ? S::WIDE0 : S::WIDE1);
        float sum = 0.f;
        if (o.x >= 0) sum += w[o.x];
        if (o.y >= 0) sum += w[o.y];
        if (o.z >= 0) sum += w[o.z];
        if (o.w >= 0) sum += w[o.w];
        wcnt[g] = present(o);
        wide += sum / (wcnt[g] ? (float)wcnt[g] : 1.f);
        if (train) s.own[g][t] = o;
      }
      float h1[16], h2[8];
      const float z = mlp_forward(s.p, x, wide, h1, h2);
      a.logits[b] = z;
      if (train) {
        const float y = __ldg(a.labels + b);
        float p;
        const float lb = sample_loss(z, y, p);
        const float dzb = (p - y) / (float)B;
        s.dz[t] = dzb;
#pragma unroll
        for (int k = 0; k < 3; ++k) s.ds[k][t] = cnt[k] ? dzb / (float)cnt[k] : 0.f;
#pragma unroll
        for (int g = 0; g < 2; ++g) s.dw[g][t] = wcnt[g] ? dzb / (float)wcnt[g] : 0.f;
        put_row(s.sv, t, x, h1, h2, lb);
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
    } else if (col.dq < NDQ) {
      acc_q = dense_sweep(s.dz, s.sv, col.dq, n, acc_q);
    }
    __syncthreads();
  }
  if (!train) {
    if (bad) atomicAdd(a.error, bad);
    return;
  }
  finish<S>(a, s, col, Sums{acc_w, acc_0, acc_1, acc_2, occ, acc_q}, bad, quirk);
}

int launch_tower(const b200_csql_args_t* args, void* stream, int train) {
  return launch<S, E>(k_census_sqlflow_tower, "k_census_sqlflow_tower", g_launches, sizeof(Smem), args, stream,
                      train != 0, train);
}

}  // namespace

extern "C" {

const char* b200_csql_last_error(void) { return E::last_error().c_str(); }
int64_t b200_csql_launch_count(void) { return g_launches.load(); }
size_t b200_csql_workspace_bytes(int64_t B) { return workspace_bytes<S, E>(B); }

int b200_csql_tower(const b200_csql_args_t* args, void* stream) { return launch_tower(args, stream, 1); }
int b200_csql_forward(const b200_csql_args_t* args, void* stream) { return launch_tower(args, stream, 0); }

}  // extern "C"
