// Tensor-core variant of the fused DeepFM tower (include/b200_deepfm.h: b200_deepfm_fwd_bwd_mma).
//
// The SIMT tower (deepfm_tower.cu) gathers every embedding row three times (forward, backward to
// the rows, parameter gradients) and is bound by those latency chains at low occupancy.  Here a
// CTA gathers the rows of MT samples ONCE, asynchronously (cp.async), into a shared-memory tile
//     X [MT][ deep 8G | dense 13 | 1.0 | 0-pad ]          (row stride = 4 mod 32 floats)
// and the three contractions of the first layer share it, as m16n8k8 TF32 `mma.sync`:
//     H   = X  . W1s^T      [MT x 16]     (W1s[j] = [W1 deep cols | W1 dense cols | b1[j] | 0])
//     dXg = dH1 . W1s[:, g]  [MT x 8]      one n-tile per id group = one embedding row
//     dW1 += dH1^T . X       [16 x KP]     K = samples; accumulated in registers over the CTA's
//                                          chunks, one atomicAdd per output at the end
// Operands are split hi + lo (3xTF32: lo*hi + hi*lo + hi*hi) so the products carry fp32-grade
// accuracy -- the parity tests compare against fp32.  The per-sample middle (ReLU, 16->4->1, FM,
// BCE, backward to dH1) runs one thread per sample between the GEMMs.  Embedding-row gradients
// leave the accumulator fragments through a warp-level id dedup (equal rows of a half-tile combine
// up a tree threaded through the __match_any_sync mask) and vector atomics.
#include "deepfm_common.cuh"
#include "mma_tf32.cuh"

namespace {

using namespace deepfm;

constexpr int MT = 32;                 // samples per chunk: two m16 tiles
constexpr int THREADS = 128;           // 4 warps
constexpr int MAX_NT_W = 12;           // dW1 n-tiles per warp (KP/8 <= 48 -> G <= 46)
constexpr int IPT = 12;                // groups gathered per thread per chunk (4 warps x 12 >= 46)
constexpr int HS = 17, DHS = 20, SS = 12, SMS = 8;  // strides of the small per-sample buffers

struct Tile {
  int ndeep, cb, kp, xs;  // deep columns, bias column, padded K, row stride
};
__host__ __device__ inline Tile tile_of(int G) {
  Tile t;
  t.ndeep = G * D;
  t.cb = t.ndeep + ND;
  t.kp = (t.cb + 1 + 7) / 8 * 8;
  t.xs = t.kp + 4;
  return t;
}
__host__ inline size_t mma_smem_bytes(int G) {
  const Tile t = tile_of(G);
  size_t f = (size_t)MT * t.xs + (size_t)H1 * t.xs + MT * HS + MT * DHS + MT * SS + MT * SMS + MT + 96;
  return f * sizeof(float) + (size_t)G * MT * sizeof(int);
}

entry::LaunchCount g_launches_mma{0};

// Fragment coordinates: mma_tf32.cuh
template <bool BACKWARD>  // 2 resident CTAs per SM: up to 255 registers (3 would cap them at 168)
__global__ void __launch_bounds__(THREADS, 2) k_tower_mma(b200_deepfm_args_t a) {
  extern __shared__ __align__(16) float smem[];
  const int G = a.G, B = a.B;
  const Layout l = layout(G);
  const Tile tl = tile_of(G);
  const int XS = tl.xs, KP = tl.kp, NDEEP = tl.ndeep, CB = tl.cb;
  float* Xs = smem;                      // [MT][XS]
  float* W1s = Xs + MT * XS;             // [H1][XS]
  float* Hs = W1s + H1 * XS;             // [MT][HS]   pre-activations of layer 1 (bias included)
  float* dHs = Hs + MT * HS;             // [MT][DHS]  d loss / d pre-activation of layer 1
  float* Ss = dHs + MT * DHS;            // [MT][SS]   FM sums s[0..7], dz at [8]
  float* Sm = Ss + MT * SS;              // [MT][SMS]  dh2[0..3], h2[0..3]
  float* lin = Sm + MT * SMS;            // [MT]       wide (dim-1) rows summed over the groups
  float* sp = lin + MT;                  // w2 64 | b2 4 | w3 4 | wd 13
  int* sinv = reinterpret_cast<int*>(sp + 96);  // [G][MT]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, gid = lane >> 2, tig = lane & 3;

  // ---- once per CTA: first-layer weights in tile column order, small parameters, constant columns
  for (int i = tid; i < H1 * XS; i += THREADS) {
    const int j = i / XS, c = i - j * XS;
    float v = 0.f;
    if (c < NDEEP) v = a.params[l.o_w1 + j * l.in + ND + c];
    else if (c < CB) v = a.params[l.o_w1 + j * l.in + (c - NDEEP)];
    else if (c == CB) v = a.params[l.o_b1 + j];
    W1s[i] = v;
  }
  for (int i = tid; i < H2 * H1; i += THREADS) sp[i] = a.params[l.o_w2 + i];
  if (tid < H2) {
    sp[64 + tid] = a.params[l.o_b2 + tid];
    sp[68 + tid] = a.params[l.o_w3 + tid];
  }
  if (tid < ND) sp[72 + tid] = a.params[l.o_wd + tid];
  for (int i = tid; i < MT * (XS - CB); i += THREADS) {
    const int s = i / (XS - CB), c = CB + i % (XS - CB);
    Xs[s * XS + c] = c == CB ? 1.0f : 0.f;  // bias column, zero padding
  }
  if (tid < MT) lin[tid] = 0.f;

  float acc[MAX_NT_W][4];  // dW1 tiles nt = warp + 4 q: rows j = gid / gid + 8, cols 8 nt + 2 tig (+1)
#pragma unroll
  for (int q = 0; q < MAX_NT_W; ++q)
#pragma unroll
    for (int e = 0; e < 4; ++e) acc[q][e] = 0.f;
  float sacc = 0.f;      // small gradient owned by thread tid < NSMALL
  float loss_acc = 0.f;  // threads < MT
  const int ntiles = KP / 8;
  const long long nchunk = ((long long)B + MT - 1) / MT;

  for (long long ch = blockIdx.x; ch < nchunk; ch += gridDim.x) {
    const long long b0 = ch * MT;
    const int n = (int)min((long long)MT, B - b0);
    __syncthreads();  // the previous chunk is fully consumed (and the one-time setup is visible)
    // ---- A: gather the rows of this chunk, once.  Item i = tid + k * THREADS is (group i / 32,
    // sample lane): all ranks are loaded first, then all row copies are issued (asynchronous), then the
    // dim-1 rows -- three batches of independent loads instead of a dependent chain per item
    {
      int rk[IPT];
#pragma unroll
      for (int k = 0; k < IPT; ++k) {
        const int g = warp + 4 * k;
        rk[k] = (g < G && lane < n) ? a.inv[(long long)g * B + b0 + lane] : -1;
      }
#pragma unroll
      for (int k = 0; k < IPT; ++k) {
        const int g = warp + 4 * k;
        if (g < G) {
          float* dst = Xs + lane * XS + g * D;
          sinv[g * MT + lane] = rk[k];
          if (rk[k] >= 0) {
            const float* row = a.bet_deep + ((long long)g * B + rk[k]) * D;
            cp_async16(dst, row);
            cp_async16(dst + 4, row + 4);
          } else {
            *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
            *reinterpret_cast<float4*>(dst + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
          }
        }
      }
      float wv[IPT];
#pragma unroll
      for (int k = 0; k < IPT; ++k) wv[k] = rk[k] >= 0 ? a.bet_wide[(long long)(warp + 4 * k) * B + rk[k]] : 0.f;
      float wsum = 0.f;
#pragma unroll
      for (int k = 0; k < IPT; ++k) wsum += wv[k];
      atomicAdd(&lin[lane], wsum);  // four warps share a sample
    }
    for (int i = tid; i < MT * ND; i += THREADS) {
      const int s = i / ND, e = i - s * ND;
      Xs[s * XS + NDEEP + e] = s < n ? a.dense[(b0 + s) * ND + e] : 0.f;
    }
    cp_async_wait_all();
    __syncthreads();
    // ---- B: H = X . W1s^T.  warp -> (m-tile = warp & 1, n-tile = warp >> 1)
    {
      const int m0 = 16 * (warp & 1), n0 = 8 * (warp >> 1);
      float d[4] = {0.f, 0.f, 0.f, 0.f};
      const float* xa = Xs + (m0 + gid) * XS + tig;
      const float* wb = W1s + (n0 + gid) * XS + tig;
      for (int k0 = 0; k0 < KP; k0 += 8) {
        uint32_t ah[4], al[4], bh[2], bl[2];
        split(xa[k0], ah[0], al[0]);
        split(xa[k0 + 8 * XS], ah[1], al[1]);
        split(xa[k0 + 4], ah[2], al[2]);
        split(xa[k0 + 8 * XS + 4], ah[3], al[3]);
        split(wb[k0], bh[0], bl[0]);
        split(wb[k0 + 4], bh[1], bl[1]);
        mma3(d, ah, al, bh, bl);
      }
      Hs[(m0 + gid) * HS + n0 + 2 * tig] = d[0];
      Hs[(m0 + gid) * HS + n0 + 2 * tig + 1] = d[1];
      Hs[(m0 + gid + 8) * HS + n0 + 2 * tig] = d[2];
      Hs[(m0 + gid + 8) * HS + n0 + 2 * tig + 1] = d[3];
    }
    __syncthreads();
    // ---- C: one thread per sample: FM, layers 2 and 3, loss, backward to dH1
    if (tid < MT) {
      const int s = tid;
      float dh1[H1];
#pragma unroll
      for (int j = 0; j < H1; ++j) dh1[j] = 0.f;
      float dz = 0.f, fs[D], dh2[H2], h2[H2];
#pragma unroll
      for (int d_ = 0; d_ < D; ++d_) fs[d_] = 0.f;
#pragma unroll
      for (int k = 0; k < H2; ++k) dh2[k] = h2[k] = 0.f;
      if (s < n) {
        float q = 0.f;
        const float4* xr = reinterpret_cast<const float4*>(Xs + s * XS);
        for (int g = 0; g < G; ++g) {
          const float4 u = xr[2 * g], v = xr[2 * g + 1];
          fs[0] += u.x; fs[1] += u.y; fs[2] += u.z; fs[3] += u.w;
          fs[4] += v.x; fs[5] += v.y; fs[6] += v.z; fs[7] += v.w;
          q = fmaf(u.x, u.x, q); q = fmaf(u.y, u.y, q); q = fmaf(u.z, u.z, q); q = fmaf(u.w, u.w, q);
          q = fmaf(v.x, v.x, q); q = fmaf(v.y, v.y, q); q = fmaf(v.z, v.z, q); q = fmaf(v.w, v.w, q);
        }
        float lt = lin[s];
#pragma unroll
        for (int e = 0; e < ND; ++e) lt = fmaf(sp[72 + e], Xs[s * XS + NDEEP + e], lt);
        float h[H1], a1[H1];
#pragma unroll
        for (int j = 0; j < H1; ++j) h[j] = Hs[s * HS + j];
        const float z = forward_tail(h, fs, q, lt, sp, sp + 64, sp + 68, a1, h2);
        if (a.logits != nullptr) a.logits[b0 + s] = z;
        if (BACKWARD) loss_acc += backward_tail(z, a.labels[b0 + s], true, B, h, h2, sp, sp + 68, dz, dh2, dh1);
      }
      lin[s] = 0.f;  // ready for the next chunk's atomics
#pragma unroll
      for (int j = 0; j < H1; ++j) dHs[s * DHS + j] = dh1[j];
#pragma unroll
      for (int d_ = 0; d_ < D; ++d_) Ss[s * SS + d_] = fs[d_];
      Ss[s * SS + 8] = dz;
#pragma unroll
      for (int k = 0; k < H2; ++k) {
        Sm[s * SMS + k] = dh2[k];
        Sm[s * SMS + 4 + k] = h2[k];
      }
    }
    if (!BACKWARD) continue;
    __syncthreads();
    // ---- D: d loss / d embedding rows, per group: dXg = dH1 . W1s[:, 8g .. 8g+8) + dz (s - e)
    {
      const int m0 = 16 * (warp & 1);
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int ks = 0; ks < 2; ++ks) {
        const float* da = dHs + (m0 + gid) * DHS + 8 * ks + tig;
        split(da[0], ah[ks][0], al[ks][0]);
        split(da[8 * DHS], ah[ks][1], al[ks][1]);
        split(da[4], ah[ks][2], al[ks][2]);
        split(da[8 * DHS + 4], ah[ks][3], al[ks][3]);
      }
      const unsigned dim_mask = 0x11111111u << tig;  // lanes that hold the same two dims
      for (int g = warp >> 1; g < G; g += 2) {
        float d[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) {
          uint32_t bh[2], bl[2];
          split(W1s[(8 * ks + tig) * XS + g * D + gid], bh[0], bl[0]);
          split(W1s[(8 * ks + tig + 4) * XS + g * D + gid], bh[1], bl[1]);
          mma3(d, ah[ks], al[ks], bh, bl);
        }
#pragma unroll
        for (int half = 0; half < 2; ++half) {
          const int s = m0 + gid + 8 * half;
          const float dz = Ss[s * SS + 8];
          float x0 = d[2 * half] + dz * (Ss[s * SS + 2 * tig] - Xs[s * XS + g * D + 2 * tig]);
          float x1 = d[2 * half + 1] + dz * (Ss[s * SS + 2 * tig + 1] - Xs[s * XS + g * D + 2 * tig + 1]);
          float xw = dz;
          const int r = sinv[g * MT + s];
          // equal rows of this half-tile combine up a tree threaded through the peer mask
          const int key = r >= 0 ? r : -1 - lane;
          const unsigned peers = __match_any_sync(0xffffffffu, key) & dim_mask;
          const int rank = __popc(peers & ((1u << lane) - 1));
          const int maxn = __reduce_max_sync(0xffffffffu, (unsigned)__popc(peers));
          const unsigned above = peers & ~((2u << lane) - 1);
          int nxt = above ? __ffs(above) - 1 : -1;
          for (int step = 1; step < maxn; step <<= 1) {
            const int src = nxt >= 0 ? nxt : lane;
            const bool take = nxt >= 0 && (rank & (2 * step - 1)) == 0;
            const float y0 = __shfl_sync(0xffffffffu, x0, src);
            const float y1 = __shfl_sync(0xffffffffu, x1, src);
            const float yw = __shfl_sync(0xffffffffu, xw, src);
            const int nn = __shfl_sync(0xffffffffu, nxt, src);
            if (take) { x0 += y0; x1 += y1; xw += yw; }
            nxt = nxt >= 0 ? nn : -1;
          }
          if (r >= 0 && rank == 0) {
            atomicAdd(reinterpret_cast<float2*>(a.gsum_deep + ((long long)g * B + r) * D + 2 * tig), make_float2(x0, x1));
            if (tig == 0) atomicAdd(a.gsum_wide + (long long)g * B + r, xw);
          }
        }
      }
    }
    // ---- E: dW1 += dH1^T . X  (K = the MT samples); warp owns n-tiles warp, warp + 4, ...
#pragma unroll
    for (int ks = 0; ks < MT / 8; ++ks) {
      uint32_t ah[4], al[4];
      const float* da = dHs + (8 * ks + tig) * DHS + gid;
      split(da[0], ah[0], al[0]);
      split(da[8], ah[1], al[1]);
      split(da[4 * DHS], ah[2], al[2]);
      split(da[4 * DHS + 8], ah[3], al[3]);
      const float* xb = Xs + (8 * ks + tig) * XS + gid;
#pragma unroll
      for (int q = 0; q < MAX_NT_W; ++q) {
        const int nt = warp + 4 * q;
        if (nt < ntiles) {
          uint32_t bh[2], bl[2];
          split(xb[8 * nt], bh[0], bl[0]);
          split(xb[8 * nt + 4 * XS], bh[1], bl[1]);
          mma3(acc[q], ah, al, bh, bl);
        }
      }
    }
    // small gradients: dW2 64 | db2 4 | dw3 4 | dw_dense 13, thread per output
    if (tid < NSMALL) {  // the small_grad of deepfm_common.cuh, read from this kernel's per-sample buffers
      for (int s = 0; s < n; ++s) {
        float v;
        if (tid < H2 * H1) v = Sm[s * SMS + tid / H1] * fmaxf(Hs[s * HS + tid % H1], 0.f);   // dh2[k] * a1[j]
        else if (tid < H2 * H1 + H2) v = Sm[s * SMS + tid - H2 * H1];                        // dh2[k]
        else if (tid < H2 * H1 + 2 * H2) v = Ss[s * SS + 8] * Sm[s * SMS + 4 + tid - H2 * H1 - H2];  // dz * h2[k]
        else v = Ss[s * SS + 8] * Xs[s * XS + NDEEP + tid - H2 * H1 - 2 * H2];              // dz * dense[e]
        sacc += v;
      }
    }
  }
  if (!BACKWARD) return;
  // ---- flush the CTA's parameter gradients
#pragma unroll
  for (int q = 0; q < MAX_NT_W; ++q) {
    const int nt = warp + 4 * q;
    if (nt >= ntiles) continue;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = gid + 8 * (e >> 1), c = 8 * nt + 2 * tig + (e & 1);
      int off = -1;
      if (c < NDEEP) off = l.o_w1 + j * l.in + ND + c;
      else if (c < CB) off = l.o_w1 + j * l.in + (c - NDEEP);
      else if (c == CB) off = l.o_b1 + j;
      if (off >= 0) atomicAdd(a.grads + off, acc[q][e]);
    }
  }
  if (tid < NSMALL) atomicAdd(a.grads + small_grad_offset(l, tid), sacc);
  if (warp == 0) add_warp_loss(loss_acc, a.loss, B, lane == 0);  // MT == 32: the per-sample threads are warp 0
}

// zero loss / grads / the live rows of the per-unique-id gradient buffers
__global__ void __launch_bounds__(256) k_mma_prep(b200_deepfm_args_t a, int n_params) { zero_step_outputs(a, n_params); }

static_assert(MT == 32, "the per-sample phase and the loss reduction assume one warp of samples");

}  // namespace

extern "C" {

int64_t b200_deepfm_mma_launch_count(void) { return g_launches_mma.load(); }

int b200_deepfm_fwd_bwd_mma(const b200_deepfm_args_t* a, void* stream) {
  if (check_common(a, true)) return -1;
  if (tile_of(a->G).kp / 8 > 4 * MAX_NT_W) return E::fail(-1, "too many id groups for the mma tower (max 46)");
  if (a->rows) return E::fail(-1, "the mma tower reads pulled rows only");
  const size_t smem = mma_smem_bytes(a->G);
  if (smem > 100 * 1024) return E::fail(-1, "the mma tower's tile does not fit in shared memory");
  cudaStream_t st = (cudaStream_t)stream;
  entry::Device d;
  int per_sm = 0;  // resident CTAs per SM
  if (int rc = E::device(&d)) return rc;
  if (int rc = E::raise_smem_limit(k_tower_mma<true>, 100 * 1024)) return rc;
  if (int rc = E::blocks_per_sm(k_tower_mma<true>, THREADS, smem, &per_sm)) return rc;
  const Layout l = layout(a->G);
  k_mma_prep<<<dim3(8, a->G), 256, 0, st>>>(*a, l.total);
  if (int rc = E::launched("k_mma_prep", g_launches_mma)) return rc;
  const long long nchunk = ((long long)a->B + MT - 1) / MT;
  const long long cap = (long long)d.sms * per_sm;
  const unsigned grid = (unsigned)(nchunk < cap ? nchunk : cap);
  k_tower_mma<true><<<grid, THREADS, smem, st>>>(*a);
  return E::launched("k_tower_mma", g_launches_mma);
}

}  // extern "C"
