// xDeepFM tower (include/b200_deepfm.h: b200_deepfm_xdeepfm_*), the dense part of the dac_ctr xDeepFM model:
// Wide & Deep's logit (deepfm_tower2.cu, k_tower_tile<..., FM = false, CIN = true>) plus a two-layer Compressed
// Interaction Network over the deep rows X0[b] = [G fields x 8] (layer_size (128, 128), split_half, relu):
//     Z_k[b, d, i H_k + j] = X0[b, i, d] X_k[b, j, d],   C_k[b, h, d] = relu(sum_K W_k[h, K] Z_k[b, d, K] + b_k[h]),
//     X_1 = C_0[:, :64],  p = sum_d [C_0[:, 64:] | C_1],  cin logit = w_ex . p + b_ex,
// and the loss adds 1e-5 (|W_0|^2 + |W_1|^2).
//
// The CIN is compute-bound (2 x 128 x 8 x (G^2 + 64 G) FLOP per sample and pass), so its three contractions run
// on tensor cores as 3xTF32 mma.sync (mma_tf32.cuh): an fp32 operand is split hi + lo in registers and fp32
// accumulates.  Z is never stored: a lane forms its B fragment as the fp32 product X0 X_k from the tile in shared
// memory and splits that.  Launches of a training step:
//   prologue  Wide & Deep prep (deepfm_tower2.cu), then k_cin_prep: W_k into the two fragment-ordered A operands
//             (K padded: xdeepfm.cuh CinShape), the CIN gradients = 2e-5 W (0 for biases / w_ex / b_ex), loss += L2
//   main      k_cin_fwd     per 32-sample tile (tile_tower.cuh TileLoop: the tile's rows gathered once): C_k = W_k Z_k
//                           with warp w = channels 16w..16w+15 x 32 n-tiles (n-tile s = sample s, column = d);
//                           writes the CIN logit, p, X_1 and the ReLU masks (bits) to the scratch buffer
//             k_tower_tile  Wide & Deep + the CIN logit; writes dz
//             k_cin_data    per tile: dZ_1 = W_1^T dC_1 contracted into dX0 and dX_1 (shared-memory atomics), dC_0,
//                           dZ_0 = W_0^T dC_0 contracted into dX0 from both factors, then the per-unique-id sums
//                           of dX0 (deepfm_common.cuh dedup_red; the wide part is 0)
//             k_cin_weights dW_k = dC_k Z_k^T: one CTA per 128 x 128 output tile and batch slice, K split over
//                           the batch, dC and Z regenerated from dz, the masks, X0, X_1 and dC_0; one atomic per
//                           output per CTA; db_k, dw_ex and db_ex in the CTAs of the first output tile
// A direct channel's dC is dz w_ex[c] mask: the data pass folds w_ex into its A operand (W^T) and its B operand
// is mask ? dz : 0; the weight pass takes A = mask (exact in TF32, so two products instead of three), B = dz Z
// and scales the output by w_ex.
#include "mma_tf32.cuh"
#include "xdeepfm.cuh"

namespace {

using namespace deepfm;

entry::LaunchCount g_launches{0};

constexpr int X1S = CIN_HALF * D;  // 512: X_1 / dX_1 / dC_0 of one sample, [64][8]
constexpr int PS = CIN_P + 1;      // 193: p row stride in shared memory (odd: lane = sample reads are conflict-free)
constexpr int MW = 64;             // mask words per sample: 32 per layer
constexpr int DXS = MAXG * D;      // 304: dX0 / X0 row of one sample in shared memory
constexpr uint32_t TF32_ONE = 0x3f800000u;

// shared memory (floats): X | ranks | WV | then per kernel; with a row source the ids Ut come last
constexpr int SM_TILE = SM_X + SM_R + SM_WV;
constexpr size_t FWD_BYTES = (size_t)(SM_TILE + TS * X1S + TS * PS + TS * MW) * sizeof(float);
constexpr size_t DATA_BYTES = (size_t)(SM_TILE + 2 * TS * X1S + TS * DXS) * sizeof(float);
constexpr size_t WGT_BYTES = (size_t)(TS * DXS + TS * X1S + TS * MW + TS) * sizeof(float);
static_assert(TS * 32 + 2 * TS <= SM_WV, "the data pass keeps one layer's masks and dz hi / lo in WV");
static_assert(DATA_BYTES + SM_U * sizeof(int) <= 227 * 1024, "shared memory");

// ReLU mask bit of channel h, dim d in one layer's 32 words.  The forward stores the words as its ballots: word
// 4 (h / 16) + e with element e = 2 ((h / 8) % 2) + d % 2 of the accumulator, bit = lane = 4 (h % 8) + d / 2.
__device__ __forceinline__ uint32_t mask_bit(const uint32_t* w, int h, int d) {
  return (w[(h >> 4) * 4 + ((h >> 3) & 1) * 2 + (d & 1)] >> ((h & 7) * 4 + (d >> 1))) & 1u;
}

__device__ __forceinline__ float block_sum(float v, float* red) {  // all threads of a 256-thread block call it
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < THREADS / 32; ++w) s += red[w];
  return s;
}

// ---------------- prologue ----------------
// Reads params only.  Wf_k[k-step][m-tile 8][lane][4]: A fragment (a0..a3) of W_k for forward k-step ks and channel
// tile mt; Wb_k[m-tile][k-step 16][lane][4]: A fragment of W_k^T (rows = padded K, k = channel) for the data pass,
// direct channels scaled by their w_ex.  Padding is 0.
__global__ void __launch_bounds__(THREADS) k_cin_prep(b200_deepfm_args_t a, int cin_grid) {
  const int G = a.G;
  const CinLayout c = cin_layout(G);
  const CinShape s = cin_shape(G);
  const CinScratch sc = cin_scratch(G, a.B);
  const float* p = a.params;
  float* scr = a.scratch;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (tid < 2) reinterpret_cast<int*>(scr + sc.o_cnt)[tid] = cin_grid;
  auto w0 = [&](int h, int k) {  // W_0[h] at padded K = i Hp0 + j
    const int i = k / s.hp0, j = k - i * s.hp0;
    return (k < s.k0 && j < G) ? p[c.o_w0 + h * G * G + i * G + j] : 0.f;
  };
  const long long nf0 = (long long)CIN_H * s.k0, nb0 = (long long)CIN_H * s.k0b;
  for (long long q = tid; q < nf0 + (long long)CIN_H * s.k1; q += stride) {
    const bool l1 = q >= nf0;
    const long long r = l1 ? q - nf0 : q;
    const int e = (int)(r & 3), lane = (int)((r >> 2) & 31), mt = (int)((r >> 7) & 7), ks = (int)(r >> 10);
    const int h = 16 * mt + (lane >> 2) + 8 * (e & 1), k = 8 * ks + (lane & 3) + 4 * (e >> 1);
    scr[sc.o_wf0 + q] = l1 ? p[c.o_w1 + h * s.k1 + k] : w0(h, k);
  }
  for (long long q = tid; q < nb0 + (long long)CIN_H * s.k1; q += stride) {
    const bool l1 = q >= nb0;
    const long long r = l1 ? q - nb0 : q;
    const int e = (int)(r & 3), lane = (int)((r >> 2) & 31), ks = (int)((r >> 7) & 15), mt = (int)(r >> 11);
    const int k = 16 * mt + (lane >> 2) + 8 * (e & 1), h = 8 * ks + (lane & 3) + 4 * (e >> 1);
    scr[sc.o_wb0 + q] = l1 ? p[c.o_w1 + h * s.k1 + k] * p[c.o_wex + CIN_HALF + h]
                           : w0(h, k) * (h < CIN_HALF ? 1.f : p[c.o_wex + h - CIN_HALF]);
  }
  if (a.grads == nullptr) return;
  float r2 = 0.f;
  for (long long i = c.o_w0 + tid; i < c.l.total; i += stride) {
    const bool filter = i < c.o_b0 || (i >= c.o_w1 && i < c.o_b1);
    const float w = p[i];
    a.grads[i] = filter ? 2.f * CIN_L2 * w : 0.f;
    if (filter) r2 = fmaf(w, w, r2);
  }
  __shared__ float red[THREADS / 32];
  r2 = block_sum(r2, red);
  if (threadIdx.x == 0) atomicAdd(a.loss, CIN_L2 * r2);  // after the Wide & Deep prep zeroed it (same stream)
}

// ---------------- forward ----------------
// One layer of a tile: acc[s] = the 16 x 8 block (channels 16 warp .., dims of sample s) of W_k Z_k.  The A fragment
// of k-step ks + 1 is loaded while k-step ks computes.
template <int LAYER>
__device__ __forceinline__ void cin_fwd_layer(const float* __restrict__ wf, int nks, int hp, const float* X,
                                              const float* X1s, float (&acc)[TS][4], int warp, int lane) {
  const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int s = 0; s < TS; ++s) acc[s][0] = acc[s][1] = acc[s][2] = acc[s][3] = 0.f;
  const float4* ap = reinterpret_cast<const float4*>(wf) + warp * 32 + lane;
  float4 an = __ldg(ap);
#pragma unroll 1
  for (int ks = 0; ks < nks; ++ks) {
    const float4 av = an;
    if (ks + 1 < nks) an = __ldg(ap + (ks + 1) * 256);
    uint32_t ah[4], al[4];
    split(av.x, ah[0], al[0]);
    split(av.y, ah[1], al[1]);
    split(av.z, ah[2], al[2]);
    split(av.w, ah[3], al[3]);
    const int i = (8 * ks) / hp, j = 8 * ks - i * hp + tig;
    const float* x0 = X + i * D + gid;
    const float* xk = (LAYER == 0 ? X : X1s) + j * D + gid;
    constexpr int xks = LAYER == 0 ? XS : X1S;
#pragma unroll
    for (int s = 0; s < TS; ++s) {
      const float f = x0[s * XS];
      uint32_t bh[2], bl[2];
      split(f * xk[s * xks], bh[0], bl[0]);
      split(f * xk[s * xks + 4 * D], bh[1], bl[1]);
      mma3(acc[s], ah, al, bh, bl);
    }
  }
}

// Bias, ReLU (mask bits by ballot), then X_1 (layer 0, channels < 64) or p (the direct channels, summed over d).
template <int LAYER>
__device__ __forceinline__ void cin_fwd_epilogue(float (&acc)[TS][4], const float* bias, float* X1s, float* P,
                                                 uint32_t* Ms, int warp, int lane) {
  const int gid = lane >> 2, tig = lane & 3;
  const int h0 = 16 * warp + gid;
  const float bz0 = __ldg(bias + h0), bz1 = __ldg(bias + h0 + 8);
#pragma unroll
  for (int s = 0; s < TS; ++s) {
    float v[4] = {acc[s][0] + bz0, acc[s][1] + bz0, acc[s][2] + bz1, acc[s][3] + bz1};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const unsigned m = __ballot_sync(0xffffffffu, v[e] > 0.f);
      if (lane == 0) Ms[s * MW + LAYER * 32 + warp * 4 + e] = m;
      v[e] = fmaxf(v[e], 0.f);
    }
    if (LAYER == 0 && warp < 4) {
      *reinterpret_cast<float2*>(X1s + s * X1S + h0 * D + 2 * tig) = make_float2(v[0], v[1]);
      *reinterpret_cast<float2*>(X1s + s * X1S + (h0 + 8) * D + 2 * tig) = make_float2(v[2], v[3]);
    } else {
      float p0 = v[0] + v[1], p1 = v[2] + v[3];
      p0 += __shfl_xor_sync(0xffffffffu, p0, 1);
      p1 += __shfl_xor_sync(0xffffffffu, p1, 1);
      p0 += __shfl_xor_sync(0xffffffffu, p0, 2);
      p1 += __shfl_xor_sync(0xffffffffu, p1, 2);
      const int base = LAYER == 0 ? -CIN_HALF : CIN_HALF;  // direct_0 -> p[0..63], direct_1 -> p[64..191]
      if (tig == 0) {
        P[s * PS + base + h0] = p0;
        P[s * PS + base + h0 + 8] = p1;
      }
    }
  }
}

template <bool BACKWARD, bool TABLE>
__global__ void __launch_bounds__(THREADS, 1) k_cin_fwd(b200_deepfm_args_t a, const __grid_constant__ TileRows rows) {
  extern __shared__ __align__(16) float smem[];
  float* X = smem;                                    // [TS][XS] the tile (X0 = its deep columns)
  int* Rt0 = reinterpret_cast<int*>(X + SM_X);        // [2][TS][RS]
  float* WV = reinterpret_cast<float*>(Rt0 + SM_R);   // wide values (unused here)
  float* X1s = WV + SM_WV;                            // [TS][64][8]
  float* P = X1s + TS * X1S;                          // [TS][PS]
  uint32_t* Ms = reinterpret_cast<uint32_t*>(P + TS * PS);  // [TS][MW]
  int* Ut = reinterpret_cast<int*>(Ms + TS * MW);     // TABLE: ids
  const int G = a.G, B = a.B;
  const CinLayout c = cin_layout(G);
  const CinShape sh = cin_shape(G);
  const CinScratch sc = cin_scratch(G, B);
  float* scr = a.scratch;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  __shared__ int s_tile[2];
  const TileLoop<TABLE> tl(a, rows, X, WV, Rt0, Ut, s_tile, reinterpret_cast<int*>(scr + sc.o_cnt));
  tl.start();
  int cur = 0;
  float acc[TS][4];
  for (int iter = 0;; ++iter, cur ^= 1) {
    const int tile = s_tile[iter & 1], tile_next = s_tile[(iter + 1) & 1];
    if (tile >= tl.ntile) break;
    const long long b0 = (long long)tile * TS;
    tl.gather(b0, b0 + lane < B, tile_next, Rt0 + cur * (TS * RS), cur);
    __syncthreads();  // every warp's rows
    tl.hand_out(iter);
    cin_fwd_layer<0>(scr + sc.o_wf0, sh.k0 / 8, sh.hp0, X, X1s, acc, warp, lane);
    cin_fwd_epilogue<0>(acc, a.params + c.o_b0, X1s, P, Ms, warp, lane);
    __syncthreads();  // X_1 complete
    cin_fwd_layer<1>(scr + sc.o_wf1, sh.k1 / 8, CIN_HALF, X, X1s, acc, warp, lane);
    cin_fwd_epilogue<1>(acc, a.params + c.o_b1, X1s, P, Ms, warp, lane);
    __syncthreads();  // p complete
    if (warp == 0 && b0 + lane < B) {
      float v = __ldg(a.params + c.o_bex);
      for (int k = 0; k < CIN_P; ++k) v = fmaf(__ldg(a.params + c.o_wex + k), P[lane * PS + k], v);
      scr[sc.o_logit + b0 + lane] = v;
    }
    if (BACKWARD) {  // what the backward regenerates dC and Z from
      const int n = (int)min((long long)TS, B - b0);
      for (int i = t; i < n * CIN_P; i += THREADS) scr[sc.o_p + b0 * CIN_P + i] = P[(i / CIN_P) * PS + i % CIN_P];
      uint32_t* mg = reinterpret_cast<uint32_t*>(scr + sc.o_mask) + b0 * MW;
      for (int i = t; i < n * MW; i += THREADS) mg[i] = Ms[i];
      float4* xg = reinterpret_cast<float4*>(scr + sc.o_x1 + b0 * X1S);
      const float4* xs = reinterpret_cast<const float4*>(X1s);
      for (int i = t; i < n * (X1S / 4); i += THREADS) xg[i] = xs[i];
    }
    __syncthreads();  // X / P / X_1 are rewritten by the next tile
  }
}

// ---------------- backward, data ----------------
// One layer's dZ^T block of m-tile mt: acc[s] = rows K = 16 mt + (gid, gid + 8) x dims of sample s, reduced over the
// 128 channels.  B (channel h, dim d of sample s): h < 64 of layer 0: dC_0 (Y, split); else mask ? dz : 0.
template <int LAYER>
__device__ __forceinline__ void cin_data_tile(const float* __restrict__ wb, int mt, const float* Y, const uint32_t* Mk,
                                              const float* dzh, const float* dzl, float (&acc)[TS][4], int lane) {
  const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int s = 0; s < TS; ++s) acc[s][0] = acc[s][1] = acc[s][2] = acc[s][3] = 0.f;
  const float4* ap = reinterpret_cast<const float4*>(wb) + mt * 16 * 32 + lane;
  float4 an = __ldg(ap);
#pragma unroll 1
  for (int ks = 0; ks < CIN_H / 8; ++ks) {
    const float4 av = an;
    if (ks + 1 < CIN_H / 8) an = __ldg(ap + (ks + 1) * 32);
    uint32_t ah[4], al[4];
    split(av.x, ah[0], al[0]);
    split(av.y, ah[1], al[1]);
    split(av.z, ah[2], al[2]);
    split(av.w, ah[3], al[3]);
    const int h = 8 * ks + tig;
    if (LAYER == 0 && ks < CIN_HALF / 8) {
#pragma unroll
      for (int s = 0; s < TS; ++s) {
        uint32_t bh[2], bl[2];
        split(Y[s * X1S + h * D + gid], bh[0], bl[0]);
        split(Y[s * X1S + (h + 4) * D + gid], bh[1], bl[1]);
        mma3(acc[s], ah, al, bh, bl);
      }
    } else {
#pragma unroll
      for (int s = 0; s < TS; ++s) {
        const uint32_t zh = __float_as_uint(dzh[s]), zl = __float_as_uint(dzl[s]);
        const uint32_t m0 = mask_bit(Mk + s * 32, h, gid), m1 = mask_bit(Mk + s * 32, h + 4, gid);
        const uint32_t bh[2] = {m0 ? zh : 0u, m1 ? zh : 0u}, bl[2] = {m0 ? zl : 0u, m1 ? zl : 0u};
        mma3(acc[s], ah, al, bh, bl);
      }
    }
  }
}

template <bool TABLE>
__global__ void __launch_bounds__(THREADS, 1) k_cin_data(b200_deepfm_args_t a, const __grid_constant__ TileRows rows) {
  extern __shared__ __align__(16) float smem[];
  float* X = smem;
  int* Rt0 = reinterpret_cast<int*>(X + SM_X);
  float* WV = reinterpret_cast<float*>(Rt0 + SM_R);
  uint32_t* Mk = reinterpret_cast<uint32_t*>(WV);     // [TS][32] one layer's masks (WV is free after the gather)
  float* dzh = WV + TS * 32;                          // [TS] dz split hi / lo
  float* dzl = dzh + TS;
  float* X1s = WV + SM_WV;                            // [TS][64][8]
  float* dX1 = X1s + TS * X1S;                        // [TS][64][8], then dC_0's first half
  float* dX0 = dX1 + TS * X1S;                        // [TS][DXS]
  int* Ut = reinterpret_cast<int*>(dX0 + TS * DXS);
  const int G = a.G, B = a.B;
  const CinShape sh = cin_shape(G);
  const CinScratch sc = cin_scratch(G, B);
  const float* scr = a.scratch;
  const uint32_t* mg = reinterpret_cast<const uint32_t*>(scr + sc.o_mask);
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, gid = lane >> 2, tig = lane & 3;
  __shared__ int s_tile[2];
  const TileLoop<TABLE> tl(a, rows, X, WV, Rt0, Ut, s_tile, reinterpret_cast<int*>(a.scratch + sc.o_cnt) + 1);
  tl.start();
  int cur = 0;
  float acc[TS][4];
  for (int iter = 0;; ++iter, cur ^= 1) {
    const int tile = s_tile[iter & 1], tile_next = s_tile[(iter + 1) & 1];
    if (tile >= tl.ntile) break;
    const long long b0 = (long long)tile * TS;
    const bool live = b0 + lane < B;
    int* Rt = Rt0 + cur * (TS * RS);
    tl.gather(b0, live, tile_next, Rt, cur);
    __syncthreads();  // every warp's copies into WV have landed before the masks overwrite it
    {  // X_1, layer 1's masks and dz of the tile (dead samples read the last one, their dz is 0); dX_1 = dX0 = 0
      const float4* xg = reinterpret_cast<const float4*>(scr + sc.o_x1);
      for (int i = t; i < TS * (X1S / 4); i += THREADS) {
        const long long b = min(b0 + i / (X1S / 4), (long long)B - 1);
        reinterpret_cast<float4*>(X1s)[i] = xg[b * (X1S / 4) + i % (X1S / 4)];
        reinterpret_cast<float4*>(dX1)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      for (int i = t; i < TS * DXS; i += THREADS) dX0[i] = 0.f;
      for (int i = t; i < TS * 32; i += THREADS) Mk[i] = mg[min(b0 + i / 32, (long long)B - 1) * MW + 32 + i % 32];
      if (t < TS) {
        uint32_t hi, lo;
        split(b0 + t < B ? scr[sc.o_dz + b0 + t] : 0.f, hi, lo);
        dzh[t] = __uint_as_float(hi);
        dzl[t] = __uint_as_float(lo);
      }
    }
    __syncthreads();
    tl.hand_out(iter);
    // layer 1: K = i 64 + j, both rows of an m-tile in the same i
#pragma unroll 1
    for (int mt = warp; mt < sh.k1 / 16; mt += THREADS / 32) {
      cin_data_tile<1>(scr + sc.o_wb1, mt, nullptr, Mk, dzh, dzl, acc, lane);
      const int r0 = 16 * mt + gid, i = r0 / CIN_HALF, j0 = r0 % CIN_HALF, j1 = j0 + 8, d0 = 2 * tig, d1 = d0 + 1;
#pragma unroll
      for (int s = 0; s < TS; ++s) {
        const float* x1 = X1s + s * X1S;
        const float* x0 = X + s * XS + i * D;
        float u0 = fmaf(acc[s][0], x1[j0 * D + d0], acc[s][2] * x1[j1 * D + d0]);
        float u1 = fmaf(acc[s][1], x1[j0 * D + d1], acc[s][3] * x1[j1 * D + d1]);
        for (int o = 4; o < 32; o <<= 1) {
          u0 += __shfl_xor_sync(0xffffffffu, u0, o);
          u1 += __shfl_xor_sync(0xffffffffu, u1, o);
        }
        if (gid == 0) {
          atomicAdd(dX0 + s * DXS + i * D + d0, u0);
          atomicAdd(dX0 + s * DXS + i * D + d1, u1);
        }
        const float xa = x0[d0], xb = x0[d1];
        float* dx1 = dX1 + s * X1S;
        atomicAdd(dx1 + j0 * D + d0, acc[s][0] * xa);
        atomicAdd(dx1 + j0 * D + d1, acc[s][1] * xb);
        atomicAdd(dx1 + j1 * D + d0, acc[s][2] * xa);
        atomicAdd(dx1 + j1 * D + d1, acc[s][3] * xb);
      }
    }
    __syncthreads();
    for (int i = t; i < TS * 32; i += THREADS) Mk[i] = mg[min(b0 + i / 32, (long long)B - 1) * MW + i % 32];
    __syncthreads();
    {  // dC_0's first half = dX_1 masked by layer 0, kept for the weight pass
      float* dg = a.scratch + sc.o_dc0;
      for (int i = t; i < TS * X1S; i += THREADS) {
        const int s = i / X1S, r = i % X1S;
        const float v = mask_bit(Mk + s * 32, r / D, r % D) ? dX1[i] : 0.f;
        dX1[i] = v;
        if (b0 + s < B) dg[(b0 + s) * X1S + r] = v;
      }
    }
    __syncthreads();
    // layer 0: K = i Hp0 + j; rows of one m-tile may lie in two i; padding (j >= G, K >= k0) has W = 0 and is skipped
#pragma unroll 1
    for (int mt = warp; mt < sh.k0b / 16; mt += THREADS / 32) {
      cin_data_tile<0>(scr + sc.o_wb0, mt, dX1, Mk, dzh, dzl, acc, lane);
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        const int r = 16 * mt + gid + 8 * half, i = r / sh.hp0, j = r - i * sh.hp0;
        if (r >= sh.k0 || j >= G) continue;
#pragma unroll
        for (int s = 0; s < TS; ++s) {
          const float* x0 = X + s * XS;
          float* dx0 = dX0 + s * DXS;
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int d = 2 * tig + e;
            const float v = acc[s][2 * half + e];
            atomicAdd(dx0 + i * D + d, v * x0[j * D + d]);
            atomicAdd(dx0 + j * D + d, v * x0[i * D + d]);
          }
        }
      }
    }
    __syncthreads();
    // the rows' gradients, reduced per unique id (warp w: the tile's groups 5w .. 5w + 4)
#pragma unroll 1
    for (int gi = 0; gi < KPC / D; ++gi) {
      const int g = warp * (KPC / D) + gi;
      if (g >= G) break;  // warp-uniform
      float x[D + 1];
#pragma unroll
      for (int d = 0; d < D; ++d) x[d] = dX0[lane * DXS + g * D + d];
      x[D] = 0.f;
      dedup_red(x, Rt[lane * RS + g], live, lane, a, g);
    }
    __syncthreads();  // the next tile's gather rewrites X, WV and the ranks
  }
}

// ---------------- backward, weights ----------------
// CTA (x, y): output tile x (layer 0's k0 / 128 tiles, then layer 1's) over the tiles [y per, (y + 1) per) of the
// batch.  Warp (wm = w % 4, wn = w / 4): channels 32 wm .. + 31 (2 m-tiles) x K columns 64 wn .. + 63 (8 n-tiles);
// one k-step per sample (k = d).
// The tensor cores add into their fp32 accumulator without rounding to nearest, which drifts when many terms of one
// sign meet (identical rows in every sample), so the mma accumulator covers one tile (32 k-steps) and the CTA's
// total over its tiles is kept in a second set of registers with ordinary fp32 adds.
template <bool TABLE>
__global__ void __launch_bounds__(THREADS, 1) k_cin_weights(b200_deepfm_args_t a, const __grid_constant__ TileRows rows,
                                                            int nb0, int per) {
  extern __shared__ __align__(16) float smem[];
  float* X0s = smem;                                          // [TS][DXS]
  float* Y = X0s + TS * DXS;                                  // [TS][64][8]: X_1 (layer 1) or dC_0 (layer 0)
  uint32_t* Ms = reinterpret_cast<uint32_t*>(Y + TS * X1S);  // [TS][MW]
  float* dzs = reinterpret_cast<float*>(Ms + TS * MW);        // [TS]
  const int G = a.G, B = a.B;
  const CinLayout c = cin_layout(G);
  const CinShape sh = cin_shape(G);
  const CinScratch sc = cin_scratch(G, B);
  const float* scr = a.scratch;
  const float* wex = a.params + c.o_wex;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, gid = lane >> 2, tig = lane & 3;
  const int wm = warp & 3, wn = warp >> 2;
  const bool l1 = (int)blockIdx.x >= nb0;
  const int kb = (l1 ? (int)blockIdx.x - nb0 : (int)blockIdx.x) * 128 + 64 * wn;
  const int hp = l1 ? CIN_HALF : sh.hp0, kend = l1 ? sh.k1 : sh.k0;
  const bool real_a = !l1 && wm < 2;  // layer 0, channels < 64: dC_0 of the data pass; else A = mask, B = dz Z
  int ci[8], cj[8];                   // per n-tile: X0 column i D and X_k column j D of this lane's K, or ci = -1
#pragma unroll
  for (int ni = 0; ni < 8; ++ni) {
    const int k = kb + 8 * ni + gid, i = k / hp, j = k - i * hp;
    ci[ni] = (k < kend && j < (l1 ? CIN_HALF : G)) ? i * D : -1;
    cj[ni] = j * D;
  }
  float acc[2][8][4], tot[2][8][4];
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni) tot[mi][ni][0] = tot[mi][ni][1] = tot[mi][ni][2] = tot[mi][ni][3] = 0.f;
  float sb = 0.f, sx = 0.f;  // x == 0: db of channel t % 128 of layer t / 128; dw_ex[t] (t < 192) / db_ex (t == 192)
  const long long ntile = ((long long)B + TS - 1) / TS;
  const long long t0 = (long long)blockIdx.y * per, t1 = min(ntile, t0 + per);
  const float* yg = scr + (l1 ? sc.o_x1 : sc.o_dc0);
  const uint32_t* mg = reinterpret_cast<const uint32_t*>(scr + sc.o_mask);
  for (long long tile = t0; tile < t1; ++tile) {
    const long long b0 = tile * TS;
    __syncthreads();  // the previous tile is consumed
    for (int i = t; i < G * TS * 2; i += THREADS) {  // X0: (group, sample, half row); dead samples 0
      const int g = i / (2 * TS), s = (i >> 1) & (TS - 1), q = i & 1;
      const long long b = b0 + s;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (b < B) {
        const int r = a.inv[(long long)g * B + b];
        const float* src = TABLE ? rows.deep[g] + rows.uniq[(long long)g * B + r] * rows.deep_stride
                                 : a.bet_deep + ((long long)g * B + r) * D;
        v = *reinterpret_cast<const float4*>(src + 4 * q);
      }
      *reinterpret_cast<float4*>(X0s + s * DXS + g * D + 4 * q) = v;
    }
    for (int i = t; i < TS * (X1S / 4); i += THREADS) {
      const long long b = b0 + i / (X1S / 4);
      reinterpret_cast<float4*>(Y)[i] = b < B ? reinterpret_cast<const float4*>(yg)[b * (X1S / 4) + i % (X1S / 4)]
                                              : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    for (int i = t; i < TS * MW; i += THREADS) Ms[i] = b0 + i / MW < B ? mg[b0 * MW + i] : 0u;
    if (t < TS) dzs[t] = b0 + t < B ? scr[sc.o_dz + b0 + t] : 0.f;
    __syncthreads();
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) acc[mi][ni][0] = acc[mi][ni][1] = acc[mi][ni][2] = acc[mi][ni][3] = 0.f;
#pragma unroll 1
    for (int s = 0; s < TS; ++s) {
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int mi = 0; mi < 2; ++mi) {
        const int h = 32 * wm + 16 * mi + gid;
        if (real_a) {
          const float* yr = Y + s * X1S;
          split(yr[h * D + tig], ah[mi][0], al[mi][0]);
          split(yr[(h + 8) * D + tig], ah[mi][1], al[mi][1]);
          split(yr[h * D + tig + 4], ah[mi][2], al[mi][2]);
          split(yr[(h + 8) * D + tig + 4], ah[mi][3], al[mi][3]);
        } else {
          const uint32_t* mw = Ms + s * MW + (l1 ? 32 : 0);
          ah[mi][0] = mask_bit(mw, h, tig) ? TF32_ONE : 0u;
          ah[mi][1] = mask_bit(mw, h + 8, tig) ? TF32_ONE : 0u;
          ah[mi][2] = mask_bit(mw, h, tig + 4) ? TF32_ONE : 0u;
          ah[mi][3] = mask_bit(mw, h + 8, tig + 4) ? TF32_ONE : 0u;
        }
      }
      const float scale = real_a ? 1.f : dzs[s];
      const float* x0 = X0s + s * DXS;
      const float* xk = l1 ? Y + s * X1S : x0;
#pragma unroll
      for (int ni = 0; ni < 8; ++ni) {
        uint32_t bh[2] = {0u, 0u}, bl[2] = {0u, 0u};
        if (ci[ni] >= 0) {
          split(scale * (x0[ci[ni] + tig] * xk[cj[ni] + tig]), bh[0], bl[0]);
          split(scale * (x0[ci[ni] + tig + 4] * xk[cj[ni] + tig + 4]), bh[1], bl[1]);
        }
#pragma unroll
        for (int mi = 0; mi < 2; ++mi) {
          if (real_a) {
            mma3(acc[mi][ni], ah[mi], al[mi], bh, bl);
          } else {
            mma_tf32(acc[mi][ni], ah[mi], bl);
            mma_tf32(acc[mi][ni], ah[mi], bh);
          }
        }
      }
    }
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int ni = 0; ni < 8; ++ni)
#pragma unroll
        for (int e = 0; e < 4; ++e) tot[mi][ni][e] += acc[mi][ni][e];
    if (blockIdx.x == 0) {  // db_0, db_1, dw_ex, db_ex over this tile
      if (t < CIN_HALF) {
        for (int s = 0; s < TS; ++s)
          for (int d = 0; d < D; ++d) sb += Y[s * X1S + t * D + d];
      } else {
        const int h = t % CIN_H, layer = t / CIN_H;
        for (int s = 0; s < TS; ++s) {
          int n = 0;
          for (int d = 0; d < D; ++d) n += mask_bit(Ms + s * MW + 32 * layer, h, d);
          sb = fmaf(dzs[s], (float)n, sb);
        }
      }
      if (t < CIN_P) {
        const float* pg = scr + sc.o_p;
        for (int s = 0; s < TS && b0 + s < B; ++s) sx = fmaf(dzs[s], pg[(b0 + s) * CIN_P + t], sx);
      } else if (t == CIN_P) {
        for (int s = 0; s < TS; ++s) sx += dzs[s];
      }
    }
  }
  // one atomic per output: W_k's rows scaled by the w_ex their dC carried
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int ni = 0; ni < 8; ++ni)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int h = 32 * wm + 16 * mi + gid + 8 * (e >> 1), k = kb + 8 * ni + 2 * tig + (e & 1);
        if (k >= kend) continue;
        const int i = k / hp, j = k - i * hp;
        if (l1) {
          atomicAdd(a.grads + c.o_w1 + h * sh.k1 + k, tot[mi][ni][e] * __ldg(wex + CIN_HALF + h));
        } else if (j < G) {
          const float f = h < CIN_HALF ? 1.f : __ldg(wex + h - CIN_HALF);
          atomicAdd(a.grads + c.o_w0 + h * G * G + i * G + j, tot[mi][ni][e] * f);
        }
      }
  if (blockIdx.x == 0) {
    if (t < CIN_HALF) atomicAdd(a.grads + c.o_b0 + t, sb);
    else if (t < CIN_H) atomicAdd(a.grads + c.o_b0 + t, sb * __ldg(wex + t - CIN_HALF));
    else atomicAdd(a.grads + c.o_b1 + t - CIN_H, sb * __ldg(wex + CIN_HALF + t - CIN_H));
    if (t < CIN_P) atomicAdd(a.grads + c.o_wex + t, sx);
    else if (t == CIN_P) atomicAdd(a.grads + c.o_bex, sx);
  }
}

// ---------------- host ----------------
// what: 1 = prologue only (the Wide & Deep prep, k_cin_prep), 2 = main only (k_cin_fwd, the tile kernel and, in
// training, k_cin_data and k_cin_weights), 3 = both.
template <bool BACKWARD>
int launch(const b200_deepfm_args_t* args, void* stream, int what = 3) {
  if (check_tile_args(args, BACKWARD, "xDeepFM tile tower")) return -1;
  if (args->G < 2) return E::fail(-1, "the xDeepFM tile tower needs at least 2 id groups");
  cudaStream_t st = (cudaStream_t)stream;
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int n_sm = d.sms;
  b200_deepfm_args_t a = *args;
  if (!BACKWARD) { a.grads = nullptr; a.gsum_deep = nullptr; a.gsum_wide = nullptr; a.loss = nullptr; }
  const long long ntile = ((long long)a.B + TS - 1) / TS;
  const int cin_grid = (int)(ntile < n_sm ? ntile : n_sm);  // one CTA per SM: the tile kernels take 150-230 KB
  if (what & 1) {
    if (int rc = launch_xdeepfm_tile<BACKWARD>(args, stream, 1, g_launches)) return rc;
    k_cin_prep<<<2 * n_sm, THREADS, 0, st>>>(a, cin_grid);
    if (int rc = E::launched("k_cin_prep", g_launches)) return rc;
  }
  if (!(what & 2)) return 0;
  const bool table = BACKWARD && args->rows;
  const TileRows rows = table ? tile_rows(args->rows, a.G) : TileRows{};
  const size_t u = table ? SM_U * sizeof(int) : 0;
  if (table) {
    if (int rc = E::raise_smem_limit(k_cin_fwd<true, true>, FWD_BYTES + u)) return rc;
    k_cin_fwd<true, true><<<cin_grid, THREADS, FWD_BYTES + u, st>>>(a, rows);
  } else {
    if (int rc = E::raise_smem_limit(k_cin_fwd<BACKWARD, false>, FWD_BYTES)) return rc;
    k_cin_fwd<BACKWARD, false><<<cin_grid, THREADS, FWD_BYTES, st>>>(a, rows);
  }
  if (int rc = E::launched("k_cin_fwd", g_launches)) return rc;
  if (int rc = launch_xdeepfm_tile<BACKWARD>(args, stream, 2, g_launches)) return rc;
  if (!BACKWARD) return 0;
  const CinShape sh = cin_shape(a.G);
  const int nb0 = (sh.k0 + 127) / 128, nb = nb0 + (sh.k1 + 127) / 128;
  const long long per = (ntile + (4LL * n_sm / nb) - 1) / max(1LL, 4LL * n_sm / nb);  // about 4 waves
  const unsigned ny = (unsigned)((ntile + per - 1) / per);
  if (table) {
    if (int rc = E::raise_smem_limit(k_cin_data<true>, DATA_BYTES + u)) return rc;
    k_cin_data<true><<<cin_grid, THREADS, DATA_BYTES + u, st>>>(a, rows);
    if (int rc = E::launched("k_cin_data", g_launches)) return rc;
    if (int rc = E::raise_smem_limit(k_cin_weights<true>, WGT_BYTES)) return rc;
    k_cin_weights<true><<<dim3(nb, ny), THREADS, WGT_BYTES, st>>>(a, rows, nb0, (int)per);
  } else {
    if (int rc = E::raise_smem_limit(k_cin_data<false>, DATA_BYTES)) return rc;
    k_cin_data<false><<<cin_grid, THREADS, DATA_BYTES, st>>>(a, rows);
    if (int rc = E::launched("k_cin_data", g_launches)) return rc;
    if (int rc = E::raise_smem_limit(k_cin_weights<false>, WGT_BYTES)) return rc;
    k_cin_weights<false><<<dim3(nb, ny), THREADS, WGT_BYTES, st>>>(a, rows, nb0, (int)per);
  }
  return E::launched("k_cin_weights", g_launches);
}

}  // namespace

extern "C" {

size_t b200_deepfm_xdeepfm_param_count(int G) { return G < 1 ? 0 : (size_t)cin_layout(G).l.total; }

size_t b200_deepfm_xdeepfm_scratch_floats(int G, int B) {
  return G < 1 || B < 1 ? 0 : (size_t)cin_scratch(G, B).total;
}

int64_t b200_deepfm_xdeepfm_launch_count(void) { return g_launches.load(); }

int b200_deepfm_xdeepfm_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream);
}

int b200_deepfm_xdeepfm_tile_prologue(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 1);
}

int b200_deepfm_xdeepfm_tile_main(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 2);
}

int b200_deepfm_xdeepfm_forward_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<false>(args, stream);
}

}  // extern "C"
