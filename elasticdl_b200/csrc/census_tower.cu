// Census wide & deep tower (include/b200_census.h): pooled multi-hot forward, loss, backward, MLP gradients and
// the five compacted push_rows segments in one launch, on the machinery of census_tower.cuh.
//
// A group pools the sum of its four ids' rows, so a column adds dz per occurrence; an id outside its group is
// counted in *error and read as row 0.  The whole model (9.7 KB) is staged in shared memory.
#include "../../include/b200_census.h"
#include "census_tower.cuh"

namespace {

using namespace census;
using E = entry::Entry<entry::Census>;
using S = Shape<28, 75, 115>;
static_assert(S::NPARAM == B200_CENSUS_PARAMS && MLP == B200_CENSUS_MLP && S::UNIQ_ROWS == B200_CENSUS_UNIQ_ROWS &&
                  S::GSUM_FLOATS == B200_CENSUS_GSUM_FLOATS && TILE == B200_CENSUS_TILE,
              "include/b200_census.h");
entry::LaunchCount g_launches{0};

struct Smem {
  int4 ent[3][TILE];   // the four ids of DNN input slot k of tile row r
  int4 own[2][TILE];   // the four ids of wide groups 0 and 1 of tile row r
  float p[S::SP];      // parameters
  float v[48];         // v3 @0, v2 @8, v1 @24
  int entg[3][TILE];   // the id group of slot k of row r
  float dz[TILE];
  float sv[NDQ][SV];   // per-row values of the dense sums; the last CTA's totals afterwards
  int last;
};

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
  for (int i = t; i < S::NPARAM; i += THREADS) s.p[i < S::DEEP0 ? i : i + (S::SDEEP - S::DEEP0)] = __ldg(a.params + i);
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
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        int g;
        int64_t smp;
        slot_source(quirk, b, k, B, g, smp);
        const int rows = S::rows(g);
        int4 e;
        e.x = load_id(a.ids, 4 * g + 0, B, smp, rows, bad);
        e.y = load_id(a.ids, 4 * g + 1, B, smp, rows, bad);
        e.z = load_id(a.ids, 4 * g + 2, B, smp, rows, bad);
        e.w = load_id(a.ids, 4 * g + 3, B, smp, rows, bad);
        s.ent[k][t] = e;
        s.entg[k][t] = g;
        const float4* d = reinterpret_cast<const float4*>(s.p + S::deep_soff(g));
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
        const int rows = S::rows(g);
        int4 o;
        o.x = load_id(a.ids, 4 * g + 0, B, b, rows, dummy);
        o.y = load_id(a.ids, 4 * g + 1, B, b, rows, dummy);
        o.z = load_id(a.ids, 4 * g + 2, B, b, rows, dummy);
        o.w = load_id(a.ids, 4 * g + 3, B, b, rows, dummy);
        s.own[g][t] = o;
        const float* w = s.p + (g == 0 ? S::WIDE0 : S::WIDE1);
        wide += ((w[o.x] + w[o.y]) + w[o.z]) + w[o.w];
      }
      float h1[16], h2[8], p;
      const float z = mlp_forward(s.p, x, wide, h1, h2);
      const float y = __ldg(a.labels + b);
      const float lb = sample_loss(z, y, p);
      a.logits[b] = z;
      s.dz[t] = (p - y) / (float)B;
      put_row(s.sv, t, x, h1, h2, lb);
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
    if (e.x == crow) { ACC += d; ++occ; }              \
    if (e.y == crow) { ACC += d; ++occ; }              \
    if (e.z == crow) { ACC += d; ++occ; }              \
    if (e.w == crow) { ACC += d; ++occ; }              \
  }
          CENSUS_SLOT(0, acc_0)
          CENSUS_SLOT(1, acc_1)
          CENSUS_SLOT(2, acc_2)
#undef CENSUS_SLOT
        }
      }
    } else if (col.dq < NDQ) {
      acc_q = dense_sweep(s.dz, s.sv, col.dq, n, acc_q);
    }
    __syncthreads();
  }
  finish<S>(a, s, col, Sums{acc_w, acc_0, acc_1, acc_2, occ, acc_q}, bad, quirk);
}

}  // namespace

extern "C" {

const char* b200_census_last_error(void) { return E::last_error().c_str(); }
int64_t b200_census_launch_count(void) { return g_launches.load(); }
size_t b200_census_workspace_bytes(int64_t B) { return workspace_bytes<S, E>(B); }

int b200_census_tower(const b200_census_args_t* args, void* stream) {
  return launch<S, E>(k_census_tower, "k_census_tower", g_launches, sizeof(Smem), args, stream, true);
}

}  // extern "C"
