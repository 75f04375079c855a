// Deep & Cross Network tower, tile version (include/b200_deepfm.h: b200_deepfm_dcn_*), the dense part of the dac_ctr
// DCN model: logit = sum(wide) + w_dense . dense + w_out . [relu(W2 relu(W1 x0 + b1) + b2) | x_2] with a two-layer
// CrossNet ("vector" parameterization) x_{l+1} = x0 (x_l . w_l) + b_l + x_l over x0 = [dense | deep], and the loss
// adds 1e-5 (|w_0|^2 + |w_1|^2).
//
// The cross network needs no second pass over the rows.  With a = x0.w0, c = x0.w1, e = x0.w_out_cross,
// beta = b0.w1 and gamma = w_out_cross.(b0 + b1), the recursion unrolls to
//     x_2 = x0 ((1 + a)(1 + c) + beta) + b0 + b1,   cross logit = ((1 + a)(1 + c) + beta) e + gamma,
// so a, c and e are three more units of the first-layer contraction, beta / gamma come from the prologue and
// the rest is per-sample arithmetic.  With g = d loss / d logit and K = (1 + a)(1 + c) + beta:
//     d/da = g (1 + c) e,  d/dc = g (1 + a) e,  d/de = g K          (the three extra units of dZ)
//     d x0 = dh1 W1 + d/da w0 + d/dc w1 + d/de w_out_cross           (the same dZ . W1x^T as the DNN alone)
//     d w0 = sum d/da x0,  d w1 = sum d/dc x0 + b0 sum g e,  d w_out_cross = sum d/de x0 + (b0 + b1) sum g
//     d b0 = w1 sum g e + w_out_cross sum g,  d b1 = w_out_cross sum g,  + 2e-5 w_l (L2, written by the prologue)
// The dZ^T X contraction gives the sums over x0; the two batch sums sum g e and sum g ride along with the small
// gradients, and each CTA folds its own share of the rank-1 terms into the atomics it makes anyway.
//
// The tile machinery is tile_tower.cuh's, shared with the DeepFM tile tower (deepfm_tower2.cu): 32-sample tiles
// gathered once into shared memory with cp.async (pulled bet_* rows, or TABLE: straight from the record slabs with
// the next tile's ids prefetched), tiles handed out dynamically, phases G and M, the argument checks and the
// launches; this file adds phases F / B1 / B2 with the same warp roles, 2 CTAs per SM.  The units of W1x are
//     [ a c e 0 | h1 0 .. 15 ]   (row stride 20 floats = 5 x 16 B; unit 3 has weight 0)
// and the FM sums of DeepFM are gone: their shared-memory and register room holds the three cross units.
#include "tile_tower.cuh"

namespace {

using namespace deepfm;

constexpr int NX = 4;             // cross quad of a W1x row / of dZ: a c e | 0 (W1x) or g e (state record)
constexpr int UP = NX + H1;       // 20 units per W1x row
constexpr int RW = UP;            // partial record: a c e lin | h[16]
constexpr float L2 = 1e-5f;       // CrossNet l2_reg
// per-sample backward state record: da dc de | g e | then deepfm_common's record (dh1 16 | a1 16 | dh2 4 | h2 4 | dz)
constexpr int DSTATE = NX + STATE;  // 48
constexpr int NSMALL_X = NSMALL + 2;  // + sum g e, sum g
constexpr int SPART = 2;              // threads per small gradient (174 threads, 16 samples each)
constexpr int SPLEN = TS / SPART;
static_assert(DSTATE % 4 == 0 && SPART * NSMALL_X <= THREADS, "state record / small gradients");

long long g_launches = 0;

// shared memory carve-up (floats)
constexpr int SM_W1X = NCOL * UP;          // 6400
constexpr int SM_P = NKP * RW * TS;        // 5120   partial records [kp][r][s]; reused as T[r][s] + M[s][DSTATE]
constexpr size_t SMEM_BYTES = (size_t)(SM_W1X + SM_X + SM_P + SM_R + SM_WV + SM_SMALL) * sizeof(float);
static_assert(RW * TS + DSTATE * TS <= SM_P, "T and the state records share P");
// scratch: W1x [NCOL][UP] | tile counter | beta | gamma | pad
constexpr int SCR_CNT = SM_W1X, SCR_BETA = SM_W1X + 1, SCR_GAMMA = SM_W1X + 2;
static_assert(SM_W1X + 16 == B200_DEEPFM_DCN_SCRATCH, "include/b200_deepfm.h");

// the flat parameter layout of include/b200_deepfm.h: DeepFM's up to w_out, whose first 4 floats stand where
// DeepFM's w3 does (so deepfm_common's small gradients address them unchanged), then the cross parameters
struct DcnLayout {
  Layout l;  // l.o_w3 = w_out, l.total = the whole buffer
  int o_wc, o_cw, o_cb;  // w_out's cross part [in], cross kernels w0 | w1 [2][in], cross biases b0 | b1 [2][in]
};
__host__ __device__ inline DcnLayout dcn_layout(int G) {
  DcnLayout d;
  d.l = layout(G);
  d.o_wc = d.l.o_w3 + H2;
  d.o_cw = d.o_wc + d.l.in;
  d.o_cb = d.o_cw + 2 * d.l.in;
  d.l.total = d.o_cb + 2 * d.l.in;
  return d;
}

// Tile column c -> index into x0 = [dense 13 | deep 8G], or -1 (the constant-1 column, padding)
__host__ __device__ inline int x0_of_col(int G, int c) {
  if (c < G * D) return ND + c;
  if (c >= MAXG * D && c < MAXG * D + ND) return c - MAXG * D;
  return -1;
}

// Unit u of tile column c of W1x -> index into the flat parameter / gradient layout, or -1 (weight 0)
__host__ __device__ inline int w1x_src(const DcnLayout& d, int G, int c, int u) {
  const int i = x0_of_col(G, c);
  if (u >= NX) {
    const int j = u - NX;
    if (i >= 0) return d.l.o_w1 + j * d.l.in + i;
    return c == MAXG * D + ND ? d.l.o_b1 + j : -1;
  }
  if (i < 0 || u == 3) return -1;
  return u == 0 ? d.o_cw + i : (u == 1 ? d.o_cw + d.l.in + i : d.o_wc + i);
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

// Prologue: W1 and the cross weights in tile column order, the tile counter, beta and gamma; the gradients start at
// the L2 term's (2e-5 w_l on the cross kernels, 0 elsewhere) and the loss at 1e-5 (|w0|^2 + |w1|^2); the live
// rows of the per-unique-id sums are zeroed.
__global__ void __launch_bounds__(THREADS) k_dcn_prep(b200_deepfm_args_t a, float* w1x, int main_grid) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const DcnLayout d = dcn_layout(a.G);
  const float* p = a.params;
  if (blockIdx.y == 0) {
    if (tid == 0) reinterpret_cast<int*>(w1x + SCR_CNT)[0] = main_grid;
    for (long long i = tid; i < (long long)NCOL * UP; i += stride) {
      const int c = (int)(i / UP), u = (int)(i - (long long)c * UP);
      const int src = w1x_src(d, a.G, c, u);
      w1x[i] = src >= 0 ? p[src] : 0.f;
    }
    if (a.grads)
      for (long long i = tid; i < d.l.total; i += stride)
        a.grads[i] = i >= d.o_cw && i < d.o_cb ? 2.f * L2 * p[i] : 0.f;
  }
  zero_step_outputs(a, 0);  // the loss and the live per-unique-id rows (the gradients are written above)
  if (blockIdx.x == 0 && blockIdx.y == 0) {
    __shared__ float red[THREADS / 32];
    const int n = d.l.in;
    float be = 0.f, ga = 0.f, r = 0.f;
    for (int i = threadIdx.x; i < n; i += THREADS) {
      const float w0 = p[d.o_cw + i], w1 = p[d.o_cw + n + i], b0 = p[d.o_cb + i], b1 = p[d.o_cb + n + i];
      be = fmaf(b0, w1, be);
      ga = fmaf(p[d.o_wc + i], b0 + b1, ga);
      r = fmaf(w0, w0, fmaf(w1, w1, r));
    }
    be = block_sum(be, red);
    ga = block_sum(ga, red);
    r = block_sum(r, red);
    if (threadIdx.x == 0) {
      w1x[SCR_BETA] = be;
      w1x[SCR_GAMMA] = ga;
      if (a.loss) *a.loss = L2 * r;  // after zero_step_outputs' 0 in this same thread
    }
  }
}

// One sample's share of small gradient o (0 <= o < NSMALL_X): deepfm_common's 85, then g e and g.
__device__ __forceinline__ float dcn_small_grad(int o, const float* m, const float* dense) {
  if (o < NSMALL) return small_grad(o, m + NX, dense);
  return o == NSMALL ? m[3] : m[NX + ST_DZ];
}

template <bool BACKWARD, bool TABLE>
__global__ void __launch_bounds__(THREADS, 2) k_dcn_tile(b200_deepfm_args_t a, const float* __restrict__ w1x_g,
                                                         const __grid_constant__ TileRows rows) {
  extern __shared__ __align__(16) float smem[];
  float* W1x = smem;                 // [NCOL][UP]
  float* X = W1x + SM_W1X;           // [TS][XS]
  float* P = X + SM_X;               // [NKP][RW][TS], later T[RW][TS] and Mst[TS][DSTATE]
  int* Rt0 = reinterpret_cast<int*>(P + SM_P);  // [2][TS][RS] ranks
  float* WV = reinterpret_cast<float*>(Rt0 + SM_R);  // [G][TS] wide values
  float* small = WV + SM_WV;
  float* s_w2 = small;        // [H2][H1]
  float* s_b2 = small + 64;   // [H2]
  float* s_w3 = small + 68;   // [H2]  (w_out's DNN part)
  float* s_wd = small + 72;   // [ND]
  float* s_bg = small + 88;   // beta, gamma
  int* Ut = reinterpret_cast<int*>(small + SM_SMALL);  // TABLE: [TS][RS] low words of the ids (< 2^31, direct-indexed)
  float* T = P;                          // [RW][TS] summed records
  float* Mst = P + RW * TS;              // [TS][DSTATE] per-sample backward state for B2 (16 B aligned)

  const DcnLayout dl = dcn_layout(a.G);
  const Layout& l = dl.l;
  const int B = a.B, G = a.G;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  {
    const float4* src = reinterpret_cast<const float4*>(w1x_g);
    float4* dst = reinterpret_cast<float4*>(W1x);
    for (int i = t; i < SM_W1X / 4; i += THREADS) dst[i] = src[i];
    for (int i = t; i < H2 * H1; i += THREADS) s_w2[i] = a.params[l.o_w2 + i];
    if (t < H2) { s_b2[t] = a.params[l.o_b2 + t]; s_w3[t] = a.params[l.o_w3 + t]; }
    if (t < ND) s_wd[t] = a.params[l.o_wd + t];
    if (t < 2) s_bg[t] = w1x_g[SCR_BETA + t];
  }
  // B2 accumulators, persistent over the CTA's tiles: thread t owns tile column t (19 units) and, of the remaining
  // 64 columns, column 256 + t%64 x DNN units 4*(t/64) .. +3 and cross unit t/64 (t/64 < 3)
  float2 acc0[H1 / 2], acc1[2], accx;
  float acce = 0.f, accx1 = 0.f;
  float sacc = 0.f;  // threads t < SPART * NSMALL_X: half of one small output
#pragma unroll
  for (int j = 0; j < H1 / 2; ++j) acc0[j] = make_float2(0.f, 0.f);
  acc1[0] = acc1[1] = accx = make_float2(0.f, 0.f);
  float loss_acc = 0.f;
  __syncthreads();

  __shared__ int s_tile[2];
  const TileLoop<TABLE> tl(a, rows, X, WV, Rt0, Ut, s_tile, reinterpret_cast<int*>(const_cast<float*>(w1x_g) + SCR_CNT));
  tl.start();
  int cur = 0;
  for (int iter = 0;; ++iter, cur ^= 1) {
    const int tile = s_tile[iter & 1], tile_next = s_tile[(iter + 1) & 1];
    if (tile >= tl.ntile) break;
    const long long b0 = (long long)tile * TS;
    int* Rt = Rt0 + cur * (TS * RS);
    const bool live = b0 + lane < B;
    tl.gather(b0, live, tile_next, Rt, cur);
    // ---------------- F: partial H1 / a c e / linear term over this warp's 40 columns ----------------
    {
      float2 h2[H1 / 2], hx = make_float2(0.f, 0.f);
#pragma unroll
      for (int j = 0; j < H1 / 2; ++j) h2[j] = make_float2(0.f, 0.f);
      float he = 0.f, lin = 0.f;
      const float* xrow = X + lane * XS;
      const int c0 = warp * KPC;
#pragma unroll
      for (int gi = 0; gi < KPC / D; ++gi) {
        const int c = c0 + gi * D;
        const float4 xa = *reinterpret_cast<const float4*>(xrow + c);
        const float4 xb = *reinterpret_cast<const float4*>(xrow + c + 4);
        const float xv[D] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        const int g = c / D;
        if (g < G) {  // an embedding group: the wide value
          lin += WV[g * TS + lane];
        } else if (c == MAXG * D) {  // dense columns 304..311 and (next chunk) 312..316: the linear part
#pragma unroll
          for (int d = 0; d < D; ++d) lin = fmaf(s_wd[d], xv[d], lin);
        } else if (c == MAXG * D + D) {
#pragma unroll
          for (int d = 0; d < ND - D; ++d) lin = fmaf(s_wd[D + d], xv[d], lin);
        }
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const float4* w4 = reinterpret_cast<const float4*>(W1x + (c + d) * UP);
          const float2 xx = make_float2(xv[d], xv[d]);
          const float4 wx = w4[0];
          hx = ffma2(make_float2(wx.x, wx.y), xx, hx);
          he = fmaf(wx.z, xv[d], he);
#pragma unroll
          for (int qd = 0; qd < 4; ++qd) {
            const float4 w = w4[1 + qd];
            h2[2 * qd] = ffma2(make_float2(w.x, w.y), xx, h2[2 * qd]);
            h2[2 * qd + 1] = ffma2(make_float2(w.z, w.w), xx, h2[2 * qd + 1]);
          }
        }
      }
      float* mine = P + (warp * RW) * TS + lane;
      mine[0] = hx.x;
      mine[TS] = hx.y;
      mine[2 * TS] = he;
      mine[3 * TS] = lin;
#pragma unroll
      for (int j = 0; j < H1 / 2; ++j) {
        mine[(NX + 2 * j) * TS] = h2[j].x;
        mine[(NX + 2 * j + 1) * TS] = h2[j].y;
      }
    }
    __syncthreads();
    tl.hand_out(iter);
    sum_partials<RW>(P, warp, lane);
    // every warp: the per-sample tail (lane = sample)
    float hpre[H1], zero8[D];
#pragma unroll
    for (int j = 0; j < H1; ++j) hpre[j] = T[(NX + j) * TS + lane];
#pragma unroll
    for (int d = 0; d < D; ++d) zero8[d] = 0.f;
    const float xa = T[lane], xc = T[TS + lane], xe = T[2 * TS + lane], lin = T[3 * TS + lane];
    float a1[H1], h2[H2];
    // forward_tail with zero FM sums: lin + w3 . h2
    const float K = fmaf(1.f + xa, 1.f + xc, s_bg[0]);
    const float z = forward_tail(hpre, zero8, 0.f, lin, s_w2, s_b2, s_w3, a1, h2) + fmaf(K, xe, s_bg[1]);
    if (warp == 0 && live && a.logits != nullptr) a.logits[b0 + lane] = z;
    if (BACKWARD) {
      const long long bb = live ? b0 + lane : B - 1;
      float dz, dh2[H2], dh1[H1];
      const float lb = backward_tail(z, a.labels[bb], live, B, hpre, h2, s_w2, s_w3, dz, dh2, dh1);
      if (warp == 0 && live) loss_acc += lb;
      const float ge = dz * xe;
      const float da = ge * (1.f + xc), dc = ge * (1.f + xa), de = dz * K;
      if (warp == 0) {
        float* m = Mst + lane * DSTATE;
        *reinterpret_cast<float4*>(m) = make_float4(da, dc, de, ge);
        store_state(m + NX, dh1, a1, dh2, h2, dz);
      }
      __syncthreads();  // Mst complete; B1 writes no shared memory, so each warp runs B1 and B2 back to back
      // ---------------- B1: d loss / d embedding rows of this warp's groups, reduced per unique id ----------------
#pragma unroll 1
      for (int gi = 0; gi < KPC / D; ++gi) {
        const int g = warp * (KPC / D) + gi;
        if (g >= G) break;  // warp-uniform
        const int c = g * D;
        float x[D + 1];
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const float4* w4 = reinterpret_cast<const float4*>(W1x + (c + d) * UP);
          const float4 wx = w4[0];
          float2 dt2 = ffma2(make_float2(wx.x, wx.y), make_float2(da, dc), make_float2(wx.z * de, 0.f));
#pragma unroll
          for (int qd = 0; qd < 4; ++qd) {
            const float4 w = w4[1 + qd];
            dt2 = ffma2(make_float2(w.x, w.y), make_float2(dh1[4 * qd + 0], dh1[4 * qd + 1]), dt2);
            dt2 = ffma2(make_float2(w.z, w.w), make_float2(dh1[4 * qd + 2], dh1[4 * qd + 3]), dt2);
          }
          x[d] = dt2.x + dt2.y;
        }
        x[D] = dz;  // wide row gradient
        dedup_red(x, Rt[lane * RS + g], live, lane, a, g);
      }
      // ---------------- B2: parameter gradients, accumulated over the CTA's tiles ----------------
      {
        const int c1 = 256 + (t & 63), jsel = t >> 6;
#pragma unroll 4
        for (int s = 0; s < TS; ++s) {
          const float4* d4 = reinterpret_cast<const float4*>(Mst + s * DSTATE);
          const float4 qx = d4[0], q0 = d4[1], q1 = d4[2], q2 = d4[3], q3 = d4[4];
          const float dh[H1] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
          const float x0 = X[s * XS + t], x1 = X[s * XS + c1];
          const float4 dq = jsel == 0 ? q0 : (jsel == 1 ? q1 : (jsel == 2 ? q2 : q3));
          const float dxs = jsel == 0 ? qx.x : (jsel == 1 ? qx.y : (jsel == 2 ? qx.z : 0.f));
          const float2 xx0 = make_float2(x0, x0), xx1 = make_float2(x1, x1);
#pragma unroll
          for (int j = 0; j < H1 / 2; ++j) acc0[j] = ffma2(make_float2(dh[2 * j], dh[2 * j + 1]), xx0, acc0[j]);
          accx = ffma2(make_float2(qx.x, qx.y), xx0, accx);
          acce = fmaf(qx.z, x0, acce);
          acc1[0] = ffma2(make_float2(dq.x, dq.y), xx1, acc1[0]);
          acc1[1] = ffma2(make_float2(dq.z, dq.w), xx1, acc1[1]);
          accx1 = fmaf(dxs, x1, accx1);
        }
        if (t < SPART * NSMALL_X) {  // output t % NSMALL_X over half of the samples
          const int o = t % NSMALL_X, s0 = (t / NSMALL_X) * SPLEN;
          for (int s = s0; s < s0 + SPLEN; ++s) sacc += dcn_small_grad(o, Mst + s * DSTATE, X + s * XS + MAXG * D);
        }
      }
    }
    __syncthreads();  // X / R / P are rewritten by the next tile's gather
  }
  if (BACKWARD) {
    if (t < SPART * NSMALL_X) P[t] = sacc;  // P is free: every thread has left the tile loop
    __syncthreads();
    if (t < NSMALL) atomicAdd(a.grads + small_grad_offset(l, t), P[t] + P[NSMALL_X + t]);
    // this CTA's sum g e and sum g, and its share of the rank-1 terms of w1, w_out_cross, b0, b1
    const float ge = P[NSMALL] + P[NSMALL_X + NSMALL], gs = P[NSMALL + 1] + P[NSMALL_X + NSMALL + 1];
    const int n = l.in;
    auto cross_rank1 = [&](int i, float& gw1, float& gwc) {  // x0 index i: the b0 / b1 gradients, and the
      const float* p = a.params;                             // rank-1 parts of w1 / w_out_cross
      const float w1 = p[dl.o_cw + n + i], wc = p[dl.o_wc + i], b0 = p[dl.o_cb + i], b1 = p[dl.o_cb + n + i];
      atomicAdd(a.grads + dl.o_cb + i, fmaf(w1, ge, wc * gs));
      atomicAdd(a.grads + dl.o_cb + n + i, wc * gs);
      gw1 = b0 * ge;
      gwc = (b0 + b1) * gs;
    };
#pragma unroll
    for (int j = 0; j < H1; ++j) {
      const int dst = w1x_src(dl, G, t, NX + j);
      if (dst >= 0) atomicAdd(a.grads + dst, (j & 1) ? acc0[j >> 1].y : acc0[j >> 1].x);
    }
    const int i0 = x0_of_col(G, t);
    if (i0 >= 0) {
      float gw1, gwc;
      cross_rank1(i0, gw1, gwc);
      atomicAdd(a.grads + dl.o_cw + i0, accx.x);
      atomicAdd(a.grads + dl.o_cw + n + i0, accx.y + gw1);
      atomicAdd(a.grads + dl.o_wc + i0, acce + gwc);
    }
    const int c1 = 256 + (t & 63), jsel = t >> 6;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dst = w1x_src(dl, G, c1, NX + jsel * 4 + j);
      if (dst >= 0) atomicAdd(a.grads + dst, (j & 1) ? acc1[j >> 1].y : acc1[j >> 1].x);
    }
    const int i1 = x0_of_col(G, c1);
    if (i1 >= 0) {
      float gw1 = 0.f, gwc = 0.f;
      if (jsel == 3) cross_rank1(i1, gw1, gwc);  // the thread of column c1 without a cross unit adds the biases
      const float b0 = a.params[dl.o_cb + i1], b1 = a.params[dl.o_cb + n + i1];
      if (jsel == 0) atomicAdd(a.grads + dl.o_cw + i1, accx1);
      if (jsel == 1) atomicAdd(a.grads + dl.o_cw + n + i1, accx1 + b0 * ge);
      if (jsel == 2) atomicAdd(a.grads + dl.o_wc + i1, accx1 + (b0 + b1) * gs);
    }
    if (warp == 0) add_warp_loss(loss_acc, a.loss, B, lane == 0);
  }
}

void prep(dim3 grid, cudaStream_t st, const b200_deepfm_args_t& a, float* w1x, int main_grid) {
  k_dcn_prep<<<grid, THREADS, 0, st>>>(a, w1x, main_grid);
}

// what: 1 = prologue only (k_dcn_prep), 2 = tile kernel only, 3 = both
template <bool BACKWARD>
int launch(const b200_deepfm_args_t* args, void* stream, int what = 3) {
  if (check_tile_args(args, BACKWARD, "DCN tile tower")) return -1;
  return launch_tile_tower<BACKWARD, k_dcn_tile<BACKWARD, false>, k_dcn_tile<true, true>>(args, stream, what, SMEM_BYTES,
                                                                                          prep, g_launches);
}

}  // namespace

extern "C" {

size_t b200_deepfm_dcn_param_count(int G) { return G < 1 ? 0 : (size_t)dcn_layout(G).l.total; }

int64_t b200_deepfm_dcn_launch_count(void) { return g_launches; }

int b200_deepfm_dcn_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream);
}

int b200_deepfm_dcn_tile_prologue(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 1);
}

int b200_deepfm_dcn_tile_main(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 2);
}

int b200_deepfm_dcn_forward_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<false>(args, stream);
}

}  // extern "C"
