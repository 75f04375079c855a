// The tile design both tile towers (deepfm_tower2.cu: DeepFM, dcn_tower.cu: DCN) run on, everything of it that is
// not model arithmetic: the tile geometry and the shared-memory blocks whose size does not depend on the model, the
// row source as the kernel reads it, the dynamic tile hand-out with the rank / id prefetch, phase G (the gather),
// phase M (the sum of the 8 partial records), and the host side of an entry point (argument checks, launches).
//
// A CTA owns a tile of TS = 32 samples and gathers the tile's rows ONCE with cp.async into
//     X[s] = [ deep 38 x 8 | dense 13 | 1 (bias column) | 0 0 | pad ]     (row stride 324 floats = 81 x 16 B,
//            odd, so a warp's 32 rows are bank-conflict free for 128-bit reads; wide values in WV[g][s])
// Warp w owns id groups 5 w .. 5 w + 4 (tile columns 40 w .. 40 w + 39) in G, F and B1, and warp NKP - 1 also the
// dense | 1 | 0 0 block: each warp gathers exactly what it reads in F, so F waits for the warp's own copies only,
// not for the whole tile behind a CTA barrier.  A tower's kernel adds W1x (its first-layer weights in tile column
// order, followed in the scratch buffer by the tile counter), the partial records P and phases F, B1 and B2.
#pragma once
#include "deepfm_common.cuh"

namespace deepfm {

constexpr int TS = 32;        // samples per tile
constexpr int THREADS = 256;  // 8 warps
constexpr int NKP = 8;        // column parts (warps) of phases F / B1
constexpr int KPC = 40;       // tile columns per part = 5 id groups
constexpr int NCOL = 320;     // deep 304 | dense 13 | 1 | 0 0   (G <= 38)
constexpr int XS = 324;       // row stride: 320 + pad = 81 * 4 (odd number of 16 B quads: conflict-free 128-bit row reads)
constexpr int RS = 39;        // rank row stride (odd): Rt[s][g]
constexpr int MAXG = 38;
static_assert(NKP * KPC == NCOL && (NKP - 1) * KPC <= MAXG * D, "the last warp owns the dense block");
static_assert(MAXG == B200_DEEPFM_TILE_MAXG, "include/b200_deepfm.h");

// shared memory blocks of both towers (floats): X, the ranks, the wide values and the small parameters follow the
// tower's W1x and partial records; with a row source the ids come last
constexpr int SM_X = TS * XS;              // 10368
constexpr int SM_R = 2 * TS * RS;          // 2496   ranks Rt[buffer][s][g]: this tile's and the prefetched next tile's
constexpr int SM_WV = MAXG * TS;           // 1216   wide values WV[g][s]
constexpr int SM_SMALL = 128;              // w2 64 | b2 4 | w3 4 | wd 16, then the tower's own
constexpr int SM_U = TS * RS;              // 1248   table rows only: ids Ut[s][g] of the next tile, behind the rest

// b200_deepfm_rows_t as the kernel reads it (parameter space): the param offsets folded into the bases.
struct TileRows {
  const int64_t* uniq;
  const float* deep[MAXG];
  const float* wide[MAXG];
  long long deep_stride, wide_stride;
};

// Two units per call: two independent round-to-nearest FMAs (sm_90 has no packed fp32 FMA).
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// One thread's view of a CTA's tile loop: the dynamic tile hand-out and phase G.
//
// Tiles are handed out dynamically (one atomic per tile on a counter the prologue set to gridDim.x): with 1024 tiles
// on 296 resident CTAs a static round-robin leaves SMs with 8 tiles next to SMs with 6.  A CTA needs the index of its
// NEXT tile while it gathers the current one (rank prefetch), so two slots rotate: s_tile[k & 1] = tile of
// iteration k, written during iteration k - 2 (slot reuse) by thread 0.
//
// TABLE: the rows come straight from the tables' record slabs (TileRows) instead of bet_deep / bet_wide, which saves
// the step a separate pull kernel.  The id of a (sample, group) is one more dependent read between the rank and the
// row, so the ids of tile i + 1 are fetched right after the ranks of tile i + 1 land (end of G) and fly during the
// compute of tile i: G stays one round trip, and only a CTA's first tile pays rank -> id -> row back to back.
template <bool TABLE>
struct TileLoop {
  const b200_deepfm_args_t& a;
  const TileRows& rows;
  float* X;      // [TS][XS]
  float* WV;     // [G][TS] wide values
  int* Rt0;      // [2][TS][RS] ranks
  int* Ut;       // TABLE: [TS][RS] low words of the ids (< 2^31, direct-indexed)
  int* s_tile;   // [2] __shared__ tile slots
  int* counter;  // the tile counter behind W1x in the scratch buffer
  long long ntile;
  int lane, warp, g0, gl;  // this warp owns id groups g0 .. g0 + gl - 1

  __device__ __forceinline__ TileLoop(const b200_deepfm_args_t& a_, const TileRows& rows_, float* X_, float* WV_,
                                      int* Rt0_, int* Ut_, int* s_tile_, int* counter_)
      : a(a_), rows(rows_), X(X_), WV(WV_), Rt0(Rt0_), Ut(Ut_), s_tile(s_tile_), counter(counter_) {
    ntile = ((long long)a.B + TS - 1) / TS;
    lane = threadIdx.x & 31;
    warp = threadIdx.x >> 5;
    g0 = warp * (KPC / D);
    gl = max(0, min(a.G - g0, KPC / D));
  }

  // ranks of a tile: 4-byte cp.async, lane = sample, coalesced reads of inv (32 consecutive samples of one group)
  __device__ __forceinline__ void fetch_ranks(const long long tl, int* dst) const {
    long long b = tl * TS + lane;
    if (b >= a.B) b = a.B - 1;  // dead samples replay the last one, their results are masked
    for (int k = 0; k < gl; ++k) cp_async4(dst + lane * RS + g0 + k, a.inv + (long long)(g0 + k) * a.B + b);
  }
  // TABLE: the ids of a tile from its ranks, lane = sample; each lane reads the ranks its own copies wrote
  __device__ __forceinline__ void fetch_ids(const int* R) const {
    for (int k = 0; k < gl; ++k) {
      const int g = g0 + k;
      cp_async4(Ut + lane * RS + g, rows.uniq + (long long)g * a.B + R[lane * RS + g]);
    }
  }

  // The first two slots and the first tile's ranks (and ids); ends with a CTA barrier.
  __device__ __forceinline__ void start() const {
    if (threadIdx.x == 0) {
      s_tile[0] = (int)blockIdx.x;
      s_tile[1] = atomicAdd(counter, 1);
    }
    if ((long long)blockIdx.x < ntile) fetch_ranks(blockIdx.x, Rt0);
    cp_async_wait_all();
    if (TABLE && (long long)blockIdx.x < ntile) {
      fetch_ids(Rt0);
      cp_async_wait_all();
    }
    __syncthreads();
  }

  // After F's barrier: the tile of iteration iter + 2 into the slot of iteration iter (every thread has read it).
  __device__ __forceinline__ void hand_out(int iter) const {
    if (threadIdx.x == 0) s_tile[iter & 1] = atomicAdd(counter, 1);
  }

  // ---------------- G: gather tile b0 / TS once ----------------
  // Its ranks are already in Rt, rank buffer cur (prefetched while the previous tile was computed), so the gather is
  // ONE global round trip: the row copies of this tile and the rank prefetch of tile_next into buffer cur ^ 1 fly
  // together.  Each warp copies its own groups' rows and waits for its own copies only.
  __device__ __forceinline__ void gather(long long b0, bool live, int tile_next, const int* Rt, int cur) const {
    if (TABLE) {  // this tile's ids (fetched during the previous tile's compute) from every lane of the warp
      cp_async_wait_all();
      __syncwarp();
    }
    float* xrow = X + lane * XS;
    for (int k = 0; k < gl; ++k) {  // a lane pair copies one 32 B row: one request per row sector
      const int g = g0 + k;
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const int s = 16 * q + (lane >> 1), h = lane & 1;
        const float* src = TABLE ? rows.deep[g] + Ut[s * RS + g] * rows.deep_stride
                                 : a.bet_deep + ((long long)g * a.B + Rt[s * RS + g]) * D;
        cp_async16(X + s * XS + g * D + 4 * h, src + 4 * h);
      }
      cp_async4(WV + g * TS + lane, TABLE ? rows.wide[g] + Ut[lane * RS + g] * rows.wide_stride
                                          : a.bet_wide + (long long)g * a.B + Rt[lane * RS + g]);
    }
    if (tile_next < ntile) fetch_ranks(tile_next, Rt0 + (cur ^ 1) * (TS * RS));
    for (int g = g0 + gl; g < min(g0 + KPC / D, MAXG); ++g) {  // unused group columns (G < 38): zeros
      *reinterpret_cast<float4*>(xrow + g * D) = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(xrow + g * D + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    if (warp == NKP - 1) {  // tile columns 304..319: dense 13 | 1 | 0 | 0
      const float* dense = a.dense + (live ? b0 + lane : a.B - 1) * ND;
      for (int c = 0; c < ND; ++c) cp_async4(xrow + MAXG * D + c, dense + c);
      xrow[MAXG * D + ND] = 1.0f;
      xrow[MAXG * D + ND + 1] = 0.f;
      xrow[MAXG * D + ND + 2] = 0.f;
    }
    cp_async_wait_all();
    __syncwarp();  // (TABLE: also orders this tile's reads of Ut before the overwrite below)
    if (TABLE && tile_next < ntile) fetch_ids(Rt0 + (cur ^ 1) * (TS * RS));
  }
};

// ---------------- M: sum the 8 partial records P[kp][r][s] of RW floats into T[r][s] ----------------
// T aliases the first RW * TS floats of P; warp w sums records w, w + 8, ...  Ends with a CTA barrier.
template <int RW>
__device__ __forceinline__ void sum_partials(float* P, int warp, int lane) {
  constexpr int NR = (RW + NKP - 1) / NKP;
  float tsum[NR];
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    const int r = warp + NKP * i;
    float v = 0.f;
    if (r < RW) {
#pragma unroll
      for (int kp = 0; kp < NKP; ++kp) v += P[(kp * RW + r) * TS + lane];
    }
    tsum[i] = v;
  }
  __syncthreads();  // all partials read before T (aliasing P) is written
#pragma unroll
  for (int i = 0; i < NR; ++i) {
    const int r = warp + NKP * i;
    if (r < RW) P[r * TS + lane] = tsum[i];
  }
  __syncthreads();
}

// ---- host side of the entry points

// The checks of a tile tower `name` on top of check_common: at most 38 groups, a scratch buffer, and a row source in
// training only, with 16-byte aligned deep records.
inline int check_tile_args(const b200_deepfm_args_t* a, bool backward, const std::string& name) {
  if (check_common(a, backward)) return -1;
  if (a->G > MAXG) return fail(-1, ("the " + name + " holds at most 38 id groups").c_str());
  if (!a->scratch) return fail(-1, "null input");
  if (a->rows) {
    const b200_deepfm_rows_t* r = a->rows;
    if (!backward) return fail(-1, ("the forward-only " + name + " reads pulled rows only").c_str());
    if (!r->uniq || r->deep_stride < D || r->wide_stride < 1 || r->deep_param_off < 0 || r->wide_param_off < 0 ||
        r->deep_stride % 4 || r->deep_param_off % 4)
      return fail(-1, "bad row source");
    for (int g = 0; g < a->G; ++g)
      if (!r->deep_base[g] || !r->wide_base[g] || (reinterpret_cast<uintptr_t>(r->deep_base[g]) & 15))
        return fail(-1, "bad row source");
  }
  return 0;
}

inline TileRows tile_rows(const b200_deepfm_rows_t* r, int G) {
  TileRows rows{};
  rows.uniq = r->uniq;
  for (int g = 0; g < G; ++g) {
    rows.deep[g] = r->deep_base[g] + r->deep_param_off;
    rows.wide[g] = r->wide_base[g] + r->wide_param_off;
  }
  rows.deep_stride = r->deep_stride;
  rows.wide_stride = r->wide_stride;
  return rows;
}

// Launches the prep kernel of a tile tower on `grid` (its tile counter starts at `main_grid`).
using TilePrep = void (*)(dim3 grid, cudaStream_t st, const b200_deepfm_args_t& a, float* w1x, int main_grid);

// The launches of a tile tower's entry point, its arguments checked (check_tile_args): what = 1 prologue only (the
// prep kernel), 2 tile kernel only, 3 both.  Pulled is the tower's tile kernel <BACKWARD, false> and Table its
// <true, true>, which training takes when it has a row source; smem is their dynamic shared memory without the ids.
// The tile kernel runs 2 CTAs per SM (its __launch_bounds__), at most one per tile; `launches` counts the launches.
template <bool BACKWARD, auto Pulled, auto Table>
int launch_tile_tower(const b200_deepfm_args_t* args, void* stream, int what, size_t smem, TilePrep prep,
                      long long& launches) {
  cudaStream_t st = (cudaStream_t)stream;
  int n_sm;
  const int dev = current_device(&n_sm);
  b200_deepfm_args_t a = *args;
  if (!BACKWARD) { a.grads = nullptr; a.gsum_deep = nullptr; a.gsum_wide = nullptr; a.loss = nullptr; }
  float* w1x = a.scratch;  // W1x at the start of the scratch buffer, then the tile counter
  const long long ntile = ((long long)a.B + TS - 1) / TS;
  long long grid = (long long)n_sm * 2;
  if (grid > ntile) grid = ntile;
  if (what & 1) {
    prep(dim3(4, BACKWARD ? a.G : 1), st, a, w1x, (int)grid);
    launches += 1;
  }
  if (!(what & 2)) return launch_status();
  if (BACKWARD && args->rows) {
    const size_t smem_u = smem + SM_U * sizeof(int);
    max_dynamic_smem_once<Table>(dev, (int)smem_u);
    Table<<<(unsigned)grid, THREADS, smem_u, st>>>(a, w1x, tile_rows(args->rows, a.G));
  } else {
    max_dynamic_smem_once<Pulled>(dev, (int)smem);
    Pulled<<<(unsigned)grid, THREADS, smem, st>>>(a, w1x, TileRows{});
  }
  launches += 1;
  return launch_status();
}

}  // namespace deepfm
