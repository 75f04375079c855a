// DeepFM tower, tile version (include/b200_deepfm.h: b200_deepfm_fwd_bwd_tile / b200_deepfm_forward_tile), and the
// Wide & Deep tower (b200_deepfm_wide_deep_*) as its instances without the FM term (k_tower_tile<..., FM = false>), and
// xDeepFM's Wide & Deep part (b200_deepfm_xdeepfm_*, k_tower_tile<..., FM = false, CIN = true>).
//
// Round 1's tower gathered every embedding row three times (forward, backward, parameter-gradient
// kernel) with one dependent global gather chain per lane at low occupancy, most of the
// step.  Here a CTA owns a tile of 32 samples and gathers the tile's 38 x 32 rows ONCE, with
// cp.async (16 B, L2 -> shared memory, no registers held while in flight), into X (tile_tower.cuh: the tile
// design this tower shares with dcn_tower.cu), and everything else -- H1 = X W1x, the FM sums, the per-sample
// middle, dX = dH1 W1x^T + FM term with the per-unique-id reduction, dW1x += dH1^T X and the small gradients --
// runs out of shared memory:
//   G  gather             warp = the 5 id groups it reads in F (and the last warp the dense block), a lane pair
//                         per 32 B row; F waits for the warp's own copies only (no CTA barrier between G and F)
//   F  forward            warp = 40 tile columns (5 id groups), lane = sample: 16 accumulators + FM partials
//   M  middle             partial records summed through shared memory; every warp redoes the tiny
//                         per-sample MLP tail (it needs dh1 / dz / FM sums in registers for B1 anyway)
//   B1 embedding grads    warp = its 5 groups, lane = sample; equal rows of a warp combine up a tree
//                         (warp-level id dedup), one vector red per distinct row
//   B2 parameter grads    thread = tile column t x 16 hidden units + 4 hidden units of column 256 + t % 64
//                         (all 8 warps busy), accumulated in registers across the CTA's tiles, one atomic
//                         per output per CTA at the end; B1 writes no shared memory, so a warp goes from its
//                         B1 straight into B2 (no barrier between them).  The 85 small gradients run on 255
//                         threads, 3 per output over 11 samples each.
// W1 is presented in TILE COLUMN ORDER (W1x[c][j]: deep columns first, then dense, then b1 as the weight
// of the constant-1 column) by the prep kernel, so the bias needs no special case and every CTA loads it
// with straight 16-byte copies.  fp32 SIMT: the step has 1 GFLOP of first-layer work, and the kernel waits on
// the gather round trip and on its per-tile phases and barriers, not on FMA throughput (DESIGN.md section 10:
// a 3xTF32 mma.sync version of F / B1 / B2 measured slower).
#include "xdeepfm.cuh"

namespace {

using namespace deepfm;

constexpr int RW = H1 + D + 2;  // partial record: h[16] | s[8] | q | lin
constexpr int SPART = 3;                       // threads per small gradient (255 threads, 11 samples each)
constexpr int SPLEN = (TS + SPART - 1) / SPART;

long long g_launches = 0;

// shared memory carve-up (floats)
constexpr int SM_W1X = NCOL * H1;          // 5120
constexpr int SM_P = NKP * RW * TS;        // 6656   partial records [kp][r][s]; reused as T[r][s] + M[s][STATE]
constexpr size_t SMEM_BYTES = (size_t)(SM_W1X + SM_X + SM_P + SM_R + SM_WV + SM_SMALL) * sizeof(float);

// Tile column c of W1x -> index into the flat parameter / gradient layout, or -1 (padding).
__host__ __device__ inline int w1x_src(const Layout& l, int G, int c, int j) {
  const int ndeep = G * D;
  if (c < ndeep) return l.o_w1 + j * l.in + ND + c;
  if (c >= MAXG * D && c < MAXG * D + ND) return l.o_w1 + j * l.in + (c - MAXG * D);
  if (c == MAXG * D + ND) return l.o_b1 + j;
  return -1;
}

__global__ void __launch_bounds__(256) k_tile_prep(b200_deepfm_args_t a, int n_params, float* w1x, int main_grid) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {  // the dynamic tile counter and W1 in tile column order
    if (tid == 0) reinterpret_cast<int*>(w1x + NCOL * H1)[0] = main_grid;
    const Layout l = layout(a.G);
    for (long long i = tid; i < (long long)NCOL * H1; i += stride) {
      const int c = (int)(i / H1), j = (int)(i - (long long)c * H1);
      const int src = w1x_src(l, a.G, c, j);
      w1x[i] = src >= 0 ? a.params[src] : 0.f;
    }
  }
  zero_step_outputs(a, n_params);
}

// FM = false is the Wide & Deep model (b200_deepfm_wide_deep_*): DeepFM without its FM term, so F does not sum the
// FM partials (their records stay 0), the tail gets zero FM sums and B1's row gradient is the DNN's alone.
// CIN (with FM = false) is xDeepFM: the CIN forward (xdeepfm_cin.cu) left each sample's CIN logit in the scratch
// buffer, the tail adds it to z, and training stores dz there for the CIN's backward.
template <bool BACKWARD, bool TABLE, bool FM, bool CIN = false>
__global__ void __launch_bounds__(THREADS, 2) k_tower_tile(b200_deepfm_args_t a, const float* __restrict__ w1x_g,
                                                           const __grid_constant__ TileRows rows) {
  extern __shared__ __align__(16) float smem[];
  float* W1x = smem;                 // [NCOL][16]
  float* X = W1x + SM_W1X;           // [TS][XS]
  float* P = X + SM_X;               // [NKP][RW][TS], later T[RW][TS] and Mst[TS][STATE]
  int* Rt0 = reinterpret_cast<int*>(P + SM_P);  // [2][TS][RS] ranks
  float* WV = reinterpret_cast<float*>(Rt0 + SM_R);  // [G][TS] wide values
  float* small = WV + SM_WV;
  float* s_w2 = small;        // [H2][H1]
  float* s_b2 = small + 64;   // [H2]
  float* s_w3 = small + 68;   // [H2]
  float* s_wd = small + 72;   // [ND]
  int* Ut = reinterpret_cast<int*>(small + SM_SMALL);  // TABLE: [TS][RS] low words of the ids (< 2^31, direct-indexed)
  float* T = P;                          // [RW][TS] summed records (first RW*TS floats of P)
  float* Mst = P + RW * TS + 64;         // [TS][STATE] per-sample backward state for B2 (after T, 16 B aligned)

  const Layout l = layout(a.G);
  const int B = a.B, G = a.G;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  {
    const float4* src = reinterpret_cast<const float4*>(w1x_g);
    float4* dst = reinterpret_cast<float4*>(W1x);
    for (int i = t; i < SM_W1X / 4; i += THREADS) dst[i] = src[i];
    for (int i = t; i < H2 * H1; i += THREADS) s_w2[i] = a.params[l.o_w2 + i];
    if (t < H2) { s_b2[t] = a.params[l.o_b2 + t]; s_w3[t] = a.params[l.o_w3 + t]; }
    if (t < ND) s_wd[t] = a.params[l.o_wd + t];
  }
  // B2 accumulators, persistent over the CTA's tiles, all 8 warps busy: thread t owns tile column t (16 hidden
  // units) and, of the remaining 64 columns, column 256 + t%64 x hidden units 4*(t/64) .. +3
  float2 acc0[H1 / 2], acc1[2];
  float sacc = 0.f;  // threads t < SPART * NSMALL: a third of one small output
#pragma unroll
  for (int j = 0; j < H1 / 2; ++j) acc0[j] = make_float2(0.f, 0.f);
  acc1[0] = acc1[1] = make_float2(0.f, 0.f);
  float loss_acc = 0.f;
  __syncthreads();

  __shared__ int s_tile[2];
  const TileLoop<TABLE> tl(a, rows, X, WV, Rt0, Ut, s_tile, reinterpret_cast<int*>(const_cast<float*>(w1x_g) + SM_W1X));
  tl.start();
  int cur = 0;
  for (int iter = 0;; ++iter, cur ^= 1) {
    const int tile = s_tile[iter & 1], tile_next = s_tile[(iter + 1) & 1];
    if (tile >= tl.ntile) break;
    const long long b0 = (long long)tile * TS;
    int* Rt = Rt0 + cur * (TS * RS);
    const bool live = b0 + lane < B;
    tl.gather(b0, live, tile_next, Rt, cur);
    // ---------------- F: partial H1 / FM sums over this warp's 40 columns ----------------
    {
      float2 h2[H1 / 2];
#pragma unroll
      for (int j = 0; j < H1 / 2; ++j) h2[j] = make_float2(0.f, 0.f);
      float sd[D], q = 0.f, lin = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) sd[d] = 0.f;
      const float* xrow = X + lane * XS;
      const int c0 = warp * KPC;
#pragma unroll
      for (int gi = 0; gi < KPC / D; ++gi) {
        const int c = c0 + gi * D;
        const float4 xa = *reinterpret_cast<const float4*>(xrow + c);
        const float4 xb = *reinterpret_cast<const float4*>(xrow + c + 4);
        const float xv[D] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        const int g = c / D;
        if (g < G) {  // an embedding group: FM sums + the wide value
          if constexpr (FM) {
#pragma unroll
            for (int d = 0; d < D; ++d) { sd[d] += xv[d]; q = fmaf(xv[d], xv[d], q); }
          }
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
          const float4* w4 = reinterpret_cast<const float4*>(W1x + (c + d) * H1);
          const float2 xx = make_float2(xv[d], xv[d]);
#pragma unroll
          for (int qd = 0; qd < 4; ++qd) {  // two hidden units per ffma2 call
            const float4 w = w4[qd];
            h2[2 * qd] = ffma2(make_float2(w.x, w.y), xx, h2[2 * qd]);
            h2[2 * qd + 1] = ffma2(make_float2(w.z, w.w), xx, h2[2 * qd + 1]);
          }
        }
      }
      float* mine = P + (warp * RW) * TS + lane;
#pragma unroll
      for (int j = 0; j < H1 / 2; ++j) {
        mine[(2 * j) * TS] = h2[j].x;
        mine[(2 * j + 1) * TS] = h2[j].y;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) mine[(H1 + d) * TS] = sd[d];
      mine[(H1 + D) * TS] = q;
      mine[(H1 + D + 1) * TS] = lin;
    }
    __syncthreads();
    tl.hand_out(iter);
    sum_partials<RW>(P, warp, lane);
    // every warp: the per-sample tail (lane = sample)
    float hpre[H1], sd[D];
#pragma unroll
    for (int j = 0; j < H1; ++j) hpre[j] = T[j * TS + lane];
#pragma unroll
    for (int d = 0; d < D; ++d) sd[d] = FM ? T[(H1 + d) * TS + lane] : 0.f;
    const float q = FM ? T[(H1 + D) * TS + lane] : 0.f, lin = T[(H1 + D + 1) * TS + lane];
    float a1[H1], h2[H2];
    float z = forward_tail(hpre, sd, q, lin, s_w2, s_b2, s_w3, a1, h2);  // FM = false: lin + w3 . h2
    if constexpr (CIN) z += a.scratch[cin_scratch(G, B).o_logit + (live ? b0 + lane : B - 1)];
    if (warp == 0 && live && a.logits != nullptr) a.logits[b0 + lane] = z;
    float dz = 0.f, dh1[H1];
    if (BACKWARD) {
      // The backward tail, the state record store and the dedup tree below are deepfm_common.cuh's backward_tail,
      // store_state and dedup_red written out: called as helpers they change this kernel's register allocation
      // (more spills in the training instances), so here they stay inline.
      const long long bb = live ? b0 + lane : B - 1;
      const float y = a.labels[bb];
      const float lb = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));  // BCE with logits
      if (warp == 0 && live) loss_acc += lb;
      const float pr = 1.f / (1.f + expf(-z));
      dz = live ? (pr - y) / (float)B : 0.f;
      if constexpr (CIN) {
        if (warp == 0 && live) a.scratch[cin_scratch(G, B).o_dz + b0 + lane] = dz;
      }
      float dh2[H2];
#pragma unroll
      for (int k = 0; k < H2; ++k) dh2[k] = h2[k] > 0.f ? dz * s_w3[k] : 0.f;
#pragma unroll
      for (int j = 0; j < H1; ++j) {
        float accv = 0.f;
#pragma unroll
        for (int k = 0; k < H2; ++k) accv = fmaf(s_w2[k * H1 + j], dh2[k], accv);
        dh1[j] = hpre[j] > 0.f ? accv : 0.f;
      }
      // backward state for B2 (T's region is not overwritten: Mst lies behind it)
      if (warp == 0) {
        float4* m4 = reinterpret_cast<float4*>(Mst + lane * STATE);
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) m4[qd] = make_float4(dh1[4 * qd], dh1[4 * qd + 1], dh1[4 * qd + 2], dh1[4 * qd + 3]);
#pragma unroll
        for (int qd = 0; qd < 4; ++qd) m4[4 + qd] = make_float4(a1[4 * qd], a1[4 * qd + 1], a1[4 * qd + 2], a1[4 * qd + 3]);
        m4[8] = make_float4(dh2[0], dh2[1], dh2[2], dh2[3]);
        m4[9] = make_float4(h2[0], h2[1], h2[2], h2[3]);
        m4[10] = make_float4(dz, 0.f, 0.f, 0.f);
      }
      __syncthreads();  // Mst complete; B1 writes no shared memory, so each warp runs B1 and B2 back to back
      // ---------------- B1: d loss / d embedding rows of this warp's groups, reduced per unique id ----------------
      const float* xrow = X + lane * XS;
#pragma unroll 1
      for (int gi = 0; gi < KPC / D; ++gi) {
        const int g = warp * (KPC / D) + gi;
        if (g >= G) break;  // warp-uniform
        const int c = g * D;
        const float4 xa = *reinterpret_cast<const float4*>(xrow + c);  // the group's row: the FM term (unused without)
        const float4 xb = *reinterpret_cast<const float4*>(xrow + c + 4);
        const float ev[D] = {xa.x, xa.y, xa.z, xa.w, xb.x, xb.y, xb.z, xb.w};
        float x[D + 1];
#pragma unroll
        for (int d = 0; d < D; ++d) {
          const float4* w4 = reinterpret_cast<const float4*>(W1x + (c + d) * H1);
          float2 dt2 = make_float2(0.f, 0.f);
#pragma unroll
          for (int qd = 0; qd < 4; ++qd) {
            const float4 w = w4[qd];
            dt2 = ffma2(make_float2(w.x, w.y), make_float2(dh1[4 * qd + 0], dh1[4 * qd + 1]), dt2);
            dt2 = ffma2(make_float2(w.z, w.w), make_float2(dh1[4 * qd + 2], dh1[4 * qd + 3]), dt2);
          }
          if constexpr (FM)
            x[d] = fmaf(dz, sd[d] - ev[d], dt2.x + dt2.y);
          else
            x[d] = dt2.x + dt2.y;
        }
        x[D] = dz;  // wide row gradient
        // warp-level id dedup (dedup_red): lanes hitting the same row combine pairwise up a tree threaded through
        // the peer mask (pointer doubling): ceil(log2(max multiplicity)) rounds for the whole warp
        const int r = Rt[lane * RS + g];
        const int key = live ? r : -1 - lane;
        const unsigned peers = __match_any_sync(0xffffffffu, key);
        const int rank = __popc(peers & ((1u << lane) - 1));
        const int maxn = __reduce_max_sync(0xffffffffu, (unsigned)__popc(peers));
        const unsigned above = peers & ~((2u << lane) - 1);
        int nxt = above ? __ffs(above) - 1 : -1;
        for (int step = 1; step < maxn; step <<= 1) {
          const int src = nxt >= 0 ? nxt : lane;
          const bool take = nxt >= 0 && (rank & (2 * step - 1)) == 0;
#pragma unroll
          for (int e = 0; e <= D; ++e) {
            const float yv = __shfl_sync(0xffffffffu, x[e], src);
            if (take) x[e] += yv;
          }
          const int nn = __shfl_sync(0xffffffffu, nxt, src);
          nxt = nxt >= 0 ? nn : -1;
        }
        if (live && rank == 0) {
          float* od = a.gsum_deep + ((long long)g * B + r) * D;
          atomicAdd(reinterpret_cast<float4*>(od), make_float4(x[0], x[1], x[2], x[3]));
          atomicAdd(reinterpret_cast<float4*>(od + 4), make_float4(x[4], x[5], x[6], x[7]));
          atomicAdd(a.gsum_wide + (long long)g * B + r, x[D]);
        }
      }
      // ---------------- B2: parameter gradients, accumulated over the CTA's tiles ----------------
      {
        // second column: 256 + t % 64, hidden units 4*(t/64) .. +3 -- warp-uniform, so its dh1 quad is one of the
        // four broadcast loads above (a per-lane quad cost four shared-memory wavefronts per load)
        const int c1 = 256 + (t & 63), jsel = t >> 6;
#pragma unroll 4
        for (int s = 0; s < TS; ++s) {
          const float4* d4 = reinterpret_cast<const float4*>(Mst + s * STATE);
          const float4 q0 = d4[0], q1 = d4[1], q2 = d4[2], q3 = d4[3];
          const float dh[H1] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
          const float x0 = X[s * XS + t], x1 = X[s * XS + c1];
          const float4 dq = jsel == 0 ? q0 : (jsel == 1 ? q1 : (jsel == 2 ? q2 : q3));
          const float2 xx0 = make_float2(x0, x0), xx1 = make_float2(x1, x1);
#pragma unroll
          for (int j = 0; j < H1 / 2; ++j) acc0[j] = ffma2(make_float2(dh[2 * j], dh[2 * j + 1]), xx0, acc0[j]);
          acc1[0] = ffma2(make_float2(dq.x, dq.y), xx1, acc1[0]);
          acc1[1] = ffma2(make_float2(dq.z, dq.w), xx1, acc1[1]);
        }
        if (t < SPART * NSMALL) {  // output t % NSMALL over a third of the samples
          const int o = t % NSMALL, s0 = (t / NSMALL) * SPLEN, s1 = min(TS, s0 + SPLEN);
          for (int s = s0; s < s1; ++s) {
            const float* m = Mst + s * STATE;
            sacc += small_grad(o, m, X + s * XS + MAXG * D);
          }
        }
      }
    }
    __syncthreads();  // X / R / P are rewritten by the next tile's gather
  }
  if (BACKWARD) {
#pragma unroll
    for (int j = 0; j < H1; ++j) {
      const int dst = w1x_src(l, G, t, j);
      if (dst >= 0) atomicAdd(a.grads + dst, (j & 1) ? acc0[j >> 1].y : acc0[j >> 1].x);
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int dst = w1x_src(l, G, 256 + (t & 63), (t >> 6) * 4 + j);
      if (dst >= 0) atomicAdd(a.grads + dst, (j & 1) ? acc1[j >> 1].y : acc1[j >> 1].x);
    }
    if (t < SPART * NSMALL) P[t] = sacc;  // P is free: every thread has left the tile loop
    __syncthreads();
    if (t < NSMALL) atomicAdd(a.grads + small_grad_offset(l, t), P[t] + P[NSMALL + t] + P[2 * NSMALL + t]);
    if (warp == 0) add_warp_loss(loss_acc, a.loss, B, lane == 0);
  }
}

// The step's loss to the host without a copy-engine operation: one thread stores the value into a ring in
// MAPPED pinned host memory (a 4-byte write over PCIe) and bumps the ring cursor.  A cudaMemcpyAsync of the
// scalar between two graph launches costs a copy-engine round trip on the critical path of every step.
__global__ void k_publish_loss(const float* __restrict__ loss, float* ring, int ring_len, unsigned* cursor) {
  const unsigned at = *cursor;
  *reinterpret_cast<volatile float*>(ring + (at % (unsigned)ring_len)) = *loss;
  *cursor = at + 1;
}

void prep(dim3 grid, cudaStream_t st, const b200_deepfm_args_t& a, float* w1x, int main_grid) {
  k_tile_prep<<<grid, 256, 0, st>>>(a, layout(a.G).total, w1x, main_grid);
}

// what: 1 = prologue only (k_tile_prep), 2 = tile kernel only, 3 = both.  FM: DeepFM, else Wide & Deep.
template <bool BACKWARD, bool FM = true>
int launch(const b200_deepfm_args_t* args, void* stream, int what = 3) {
  if (check_tile_args(args, BACKWARD, FM ? "tile tower" : "Wide & Deep tile tower")) return -1;
  return launch_tile_tower<BACKWARD, k_tower_tile<BACKWARD, false, FM>, k_tower_tile<true, true, FM>>(
      args, stream, what, SMEM_BYTES, prep, g_launches);
}

}  // namespace

namespace deepfm {

template <bool BACKWARD>
int launch_xdeepfm_tile(const b200_deepfm_args_t* args, void* stream, int what, long long& launches) {
  return launch_tile_tower<BACKWARD, k_tower_tile<BACKWARD, false, false, true>, k_tower_tile<true, true, false, true>>(
      args, stream, what, SMEM_BYTES, prep, launches);
}
template int launch_xdeepfm_tile<true>(const b200_deepfm_args_t*, void*, int, long long&);
template int launch_xdeepfm_tile<false>(const b200_deepfm_args_t*, void*, int, long long&);

}  // namespace deepfm

extern "C" {

int64_t b200_deepfm_tile_launch_count(void) { return g_launches; }

int b200_deepfm_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream);
}

int b200_deepfm_tile_prologue(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 1);
}

int b200_deepfm_tile_main(const b200_deepfm_args_t* args, void* stream) {
  return launch<true>(args, stream, 2);
}

int b200_deepfm_publish_loss(const float* loss_dev, float* ring_host_mapped, int ring_len, unsigned* cursor_dev, void* stream) {
  if (!loss_dev || !ring_host_mapped || ring_len < 1 || !cursor_dev) return fail(-1, "bad publish_loss arguments");
  k_publish_loss<<<1, 1, 0, (cudaStream_t)stream>>>(loss_dev, ring_host_mapped, ring_len, cursor_dev);
  g_launches += 1;
  return launch_status();
}

int b200_deepfm_forward_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<false>(args, stream);
}

int b200_deepfm_wide_deep_fwd_bwd_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<true, false>(args, stream);
}

int b200_deepfm_wide_deep_tile_prologue(const b200_deepfm_args_t* args, void* stream) {
  return launch<true, false>(args, stream, 1);
}

int b200_deepfm_wide_deep_tile_main(const b200_deepfm_args_t* args, void* stream) {
  return launch<true, false>(args, stream, 2);
}

int b200_deepfm_wide_deep_forward_tile(const b200_deepfm_args_t* args, void* stream) {
  return launch<false, false>(args, stream);
}

}  // extern "C"
