// What the deepctr towers (deepctr_wdl_tower.cu, deepctr_deepfm_tower.cu) share: the 117-256-128-64 relu DNN of a
// 64-sample tile on 3xTF32 mma.sync (forward, and backward into a CTA's own weight-gradient partial), the stable
// counting sort of a table's occurrences by row, and the CTA-order sum of the partials.  Each tower keeps its own
// gather, logit, loss and table-gradient rule.
//
// Shared memory of a tile (floats): x [TILE][XS] (26 x 4 embedding columns, then the 13 numeric values; columns
// F .. XS-1 zero) | h1 [TILE][S1] | h2 [TILE][S2] | h3 [TILE][S3], the activations rewritten in place by their
// gradients in the backward.  A DNN layout L names the flat offsets, inside the tower's dense block D and inside its
// partial, of W0 [117, 256], b0, W1 [256, 128], b1, W2 [128, 64], b2 and wd [64] (the logit kernel).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "mma_tf32.cuh"

namespace deepctr {

constexpr int NF = 26, ND = 13, DIM = 4;
constexpr int NS = NF * DIM;  // 104 sparse columns of x
constexpr int F = NS + ND;    // 117
constexpr int N1 = 256, N2 = 128, N3 = 64;
constexpr int TILE = 64, THREADS = 256, WARPS = THREADS / 32;
constexpr int XS = 132, S1 = N1 + 4, S2 = N2 + 4, S3 = N3 + 4;  // row strides = 4 mod 32: conflict-free rows
static_assert(XS >= 128 && XS % 4 == 0, "x is read as 128 columns by dW0 = x^T dh1");
static_assert(THREADS == N1, "one thread per unit of h1 for db0");

// the sort: NCH chunks of samples per table, one CTA of SORT_THREADS per (chunk, table)
constexpr int NCH = 4, SORT_THREADS = 1024;

// ---- the DNN
// C = A B over M x N (M a multiple of 64, N of 8), K a multiple of 8: each warp unit is 64 rows x 8 columns (four
// m16n8k8 tiles sharing one B fragment); a(m, k), b(k, n) load the operands; epi(m, n, c) takes each result.
template <class LA, class LB, class Epi>
__device__ __forceinline__ void warp_gemm(int M, int N, int K, LA a, LB b, Epi epi) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
  const int nn = N / 8, units = (M / 64) * nn;
  for (int u = warp; u < units; u += WARPS) {
    const int m0 = (u / nn) * 64, n0 = (u % nn) * 8;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i) acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f;
    for (int k0 = 0; k0 < K; k0 += 8) {
      uint32_t bh[2], bl[2];
      deepfm::split(b(k0 + tig, n0 + gid), bh[0], bl[0]);
      deepfm::split(b(k0 + tig + 4, n0 + gid), bh[1], bl[1]);
#pragma unroll
      for (int mb = 0; mb < 4; ++mb) {
        const int r = m0 + 16 * mb + gid;
        uint32_t ah[4], al[4];
        deepfm::split(a(r, k0 + tig), ah[0], al[0]);
        deepfm::split(a(r + 8, k0 + tig), ah[1], al[1]);
        deepfm::split(a(r, k0 + tig + 4), ah[2], al[2]);
        deepfm::split(a(r + 8, k0 + tig + 4), ah[3], al[3]);
        deepfm::mma3(acc[mb], ah, al, bh, bl);
      }
    }
#pragma unroll
    for (int mb = 0; mb < 4; ++mb) {
      const int r = m0 + 16 * mb + gid, cc = n0 + 2 * tig;
      epi(r, cc, acc[mb][0]);
      epi(r, cc + 1, acc[mb][1]);
      epi(r + 8, cc, acc[mb][2]);
      epi(r + 8, cc + 1, acc[mb][3]);
    }
  }
}

// entry i of this CTA's partial: set on its first tile, added to after
__device__ __forceinline__ void add_part(float* p, float v, bool first) { __stcg(p, first ? v : __ldcg(p) + v); }

// h1 = relu(x W0 + b0), h2 = relu(h1 W1 + b1), h3 = relu(h2 W2 + b2); ends on a barrier
template <class L>
__device__ __forceinline__ void dnn_forward(const float* X, float* A1, float* A2, float* A3,
                                            const float* __restrict__ D) {
  warp_gemm(64, N1, 120, [&](int m, int k) { return X[m * XS + k]; },
            [&](int k, int c) { return k < F ? __ldg(D + L::W0 + k * N1 + c) : 0.f; },
            [&](int m, int c, float v) { A1[m * S1 + c] = fmaxf(v + __ldg(D + L::B0 + c), 0.f); });
  __syncthreads();
  warp_gemm(64, N2, N1, [&](int m, int k) { return A1[m * S1 + k]; },
            [&](int k, int c) { return __ldg(D + L::W1 + k * N2 + c); },
            [&](int m, int c, float v) { A2[m * S2 + c] = fmaxf(v + __ldg(D + L::B1 + c), 0.f); });
  __syncthreads();
  warp_gemm(64, N3, N2, [&](int m, int k) { return A2[m * S2 + k]; },
            [&](int k, int c) { return __ldg(D + L::W2 + k * N3 + c); },
            [&](int m, int c, float v) { A3[m * S3 + c] = fmaxf(v + __ldg(D + L::B2 + c), 0.f); });
  __syncthreads();
}

// From dz [TILE] (zero past the batch) back to x: the batch sums of db2, dW2, db1, dW1, db0 and dW0 into the CTA's
// partial `mine`, and dx of the 104 sparse columns, dx(m, c, v) per element.  Enter after a barrier that follows
// every read of h3 by the caller; the caller's barrier follows.
template <class L, class Dx>
__device__ __forceinline__ void dnn_backward(const float* X, float* A1, float* A2, float* A3, const float* dzs,
                                             const float* __restrict__ D, float* mine, bool first, Dx dx) {
  const int t = threadIdx.x;
  // dh3 = dz wd [h3 > 0], in place
  for (int i = t; i < TILE * N3; i += THREADS) {
    const int r = i / N3, c = i % N3;
    A3[r * S3 + c] = A3[r * S3 + c] > 0.f ? dzs[r] * __ldg(D + L::WD + c) : 0.f;
  }
  __syncthreads();
  if (t < N3) {
    float s = 0.f;
    for (int r = 0; r < TILE; ++r) s += A3[r * S3 + t];
    add_part(mine + L::B2 + t, s, first);
  }
  // dW2 = h2^T dh3
  warp_gemm(N2, N3, TILE, [&](int m, int k) { return A2[k * S2 + m]; }, [&](int k, int c) { return A3[k * S3 + c]; },
            [&](int m, int c, float v) { add_part(mine + L::W2 + m * N3 + c, v, first); });
  __syncthreads();
  // dh2 = (dh3 W2^T) [h2 > 0], in place
  warp_gemm(64, N2, N3, [&](int m, int k) { return A3[m * S3 + k]; },
            [&](int k, int c) { return __ldg(D + L::W2 + c * N3 + k); },
            [&](int m, int c, float v) { A2[m * S2 + c] = A2[m * S2 + c] > 0.f ? v : 0.f; });
  __syncthreads();
  if (t < N2) {
    float s = 0.f;
    for (int r = 0; r < TILE; ++r) s += A2[r * S2 + t];
    add_part(mine + L::B1 + t, s, first);
  }
  // dW1 = h1^T dh2
  warp_gemm(N1, N2, TILE, [&](int m, int k) { return A1[k * S1 + m]; }, [&](int k, int c) { return A2[k * S2 + c]; },
            [&](int m, int c, float v) { add_part(mine + L::W1 + m * N2 + c, v, first); });
  __syncthreads();
  // dh1 = (dh2 W1^T) [h1 > 0], in place
  warp_gemm(64, N1, N2, [&](int m, int k) { return A2[m * S2 + k]; },
            [&](int k, int c) { return __ldg(D + L::W1 + c * N2 + k); },
            [&](int m, int c, float v) { A1[m * S1 + c] = A1[m * S1 + c] > 0.f ? v : 0.f; });
  __syncthreads();
  {
    float s = 0.f;  // THREADS == N1: thread t owns db0[t]
    for (int r = 0; r < TILE; ++r) s += A1[r * S1 + t];
    add_part(mine + L::B0 + t, s, first);
  }
  // dW0 = x^T dh1 (x's columns past F are zero and not stored)
  warp_gemm(128, N1, TILE, [&](int m, int k) { return X[k * XS + m]; }, [&](int k, int c) { return A1[k * S1 + c]; },
            [&](int m, int c, float v) {
              if (m < F) add_part(mine + L::W0 + m * N1 + c, v, first);
            });
  // dx of the sparse columns = dh1 W0^T
  warp_gemm(64, NS, N1, [&](int m, int k) { return A1[m * S1 + k]; },
            [&](int k, int c) { return __ldg(D + L::W0 + c * N1 + k); }, dx);
}

// ---- the sort: a stable counting sort of each table's occurrences by row.  Rule::row(id) is the row an id reads;
// with Rule::kSkips it may be -1, an id with no occurrence.  hist: each CTA counts its sample chunk's ids per row of
// one table.  scatter: each CTA's cursors start at the row's offset plus the earlier chunks' counts; inside a chunk,
// warps take their turn in order and lanes of one row rank by lane.  perm[j] then lists, row by row, the samples that
// read the row in sample order, and offsets[j][ROWS] is the table's count of occurrences.
__device__ __forceinline__ void chunk_of(int64_t B, int c, int64_t* b0, int64_t* b1) {
  const int64_t ch = (B + NCH - 1) / NCH;
  *b0 = c * ch < B ? c * ch : B;
  *b1 = *b0 + ch < B ? *b0 + ch : B;
}

template <int ROWS, class Rule>
__device__ __forceinline__ void sort_hist(const int32_t* __restrict__ ids, int64_t B, int* __restrict__ counts) {
  __shared__ int h[ROWS];
  const int c = blockIdx.x, j = blockIdx.y, t = threadIdx.x;
  int64_t b0, b1;
  chunk_of(B, c, &b0, &b1);
  for (int i = t; i < ROWS; i += SORT_THREADS) h[i] = 0;
  __syncthreads();
  for (int64_t b = b0 + t; b < b1; b += SORT_THREADS) {
    const int r = Rule::row(__ldg(ids + j * B + b));
    if (!Rule::kSkips || r >= 0) atomicAdd(&h[r], 1);
  }
  __syncthreads();
  int* out = counts + ((size_t)j * NCH + c) * ROWS;
  for (int i = t; i < ROWS; i += SORT_THREADS) out[i] = h[i];
}

template <int ROWS, class Rule>
__device__ __forceinline__ void sort_scatter(const int32_t* __restrict__ ids, int64_t B,
                                             const int* __restrict__ counts, int* __restrict__ offsets,
                                             int* __restrict__ perm) {
  constexpr int ROWS_PER_THREAD = (ROWS + SORT_THREADS - 1) / SORT_THREADS;
  __shared__ int cur[ROWS];
  __shared__ int wsum[32];
  const int c = blockIdx.x, j = blockIdx.y, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  // row r's first position in perm[j]: the rows before it (an exclusive scan of the totals over rows), then the
  // earlier chunks' occurrences of r
  const int r0 = t * ROWS_PER_THREAD;
  const int* cj = counts + (size_t)j * NCH * ROWS;
  auto total = [&](int r, int upto) {  // occurrences of row r in chunks [0, upto)
    int s = 0;
    for (int cc = 0; cc < upto; ++cc) s += __ldg(cj + (size_t)cc * ROWS + r);
    return s;
  };
  int mine = 0;
  for (int r = r0; r < r0 + ROWS_PER_THREAD && r < ROWS; ++r) mine += total(r, NCH);
  int inc = mine;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int v = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += v;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    int v = wsum[lane], s = v;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += u;
    }
    wsum[lane] = s - v;
  }
  __syncthreads();
  int start = wsum[warp] + inc - mine;
  for (int r = r0; r < r0 + ROWS_PER_THREAD && r < ROWS; ++r) {
    cur[r] = start + total(r, c);
    if (c == 0) offsets[(size_t)j * (ROWS + 1) + r] = start;
    start += total(r, NCH);
  }
  if constexpr (Rule::kSkips) {  // the table ends at its count of occurrences, the last thread's inclusive scan
    if (c == 0 && t == SORT_THREADS - 1) offsets[(size_t)j * (ROWS + 1) + ROWS] = wsum[warp] + inc;
  } else {
    if (c == 0 && t == 0) offsets[(size_t)j * (ROWS + 1) + ROWS] = (int)B;
  }
  __syncthreads();
  int64_t b0, b1;
  chunk_of(B, c, &b0, &b1);
  for (int64_t base = b0; base < b1; base += SORT_THREADS) {
    const int64_t b = base + t;
    const bool valid = b < b1;
    const int key = valid ? Rule::row(__ldg(ids + j * B + b)) : -1;
    const bool take = valid && (!Rule::kSkips || key >= 0);
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int rank = __popc(peers & ((1u << lane) - 1u)), cnt = __popc(peers);
    for (int w = 0; w < SORT_THREADS / 32; ++w) {  // the warps in order: a stable sort
      if (warp == w) {
        int pos = 0;
        if (take) pos = cur[key] + rank;
        __syncwarp();
        if (take) {
          if (rank == 0) cur[key] += cnt;
          perm[(size_t)j * B + pos] = (int)b;
        }
      }
      __syncthreads();
    }
  }
}

// ---- entry i of the sum over `grid` CTAs' partials of q floats each, in CTA order
__device__ __forceinline__ float cta_order_sum(const float* parts, int q, int grid, int i) {
  float s = 0.f;
  for (int c = 0; c < grid; ++c) s += __ldcg(parts + (size_t)c * q + i);
  return s;
}

}  // namespace deepctr
