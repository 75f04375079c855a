// Fused DeepFM tower for the dac_ctr workload (include/b200_deepfm.h).
//
//   k_tower_prep : zero loss / grads / the live rows of the per-unique-id gradient buffers
//   k_tower_a    : lane = sample.  gather rows through inv, FM + DNN forward, loss, backward
//                  to the activations; embedding gradients are reduced per unique id on the
//                  fly (warp-level id dedup + one vector red per distinct row per warp)
//   k_tower_b    : thread = input column.  parameter gradients (dW1 is a [16 x B] x [B x IN]
//                  contraction over the batch: each thread owns one column and 16 accumulators,
//                  per-sample backward state staged through shared memory)
//
// fp32 throughout; no tensor cores (0.3 GFLOP per batch -- the kernel is bound by the
// gather/scatter of embedding rows, not by math).
#include "deepfm_common.cuh"

namespace {

using namespace deepfm;

long long g_launches = 0;

__global__ void __launch_bounds__(256) k_tower_prep(b200_deepfm_args_t a, int n_params) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {
    // W1 transposed to [IN][16] once per step (behind the per-sample scratch): every k_tower_a block
    // then fills its shared memory with straight 16-byte copies instead of 5072 scattered stores
    const Layout l = layout(a.G);
    float* w1t = a.scratch + (long long)a.B * STATE;
    for (long long i = tid; i < (long long)H1 * l.in; i += stride) {
      const int j = (int)(i / l.in), e = (int)(i - (long long)j * l.in);
      w1t[e * H1 + j] = a.params[l.o_w1 + i];
    }
  }
  zero_step_outputs(a, n_params);
}

// shared-memory copy of the parameters: W1 transposed to [IN][16] so that the 16 outputs of
// one input are four broadcast LDS.128.
struct SmemParams {
  float* w1t;  // [IN][H1]
  float* b1;   // [H1]
  float* w2;   // [H2][H1]
  float* b2;   // [H2]
  float* w3;   // [H2]
  float* wd;   // [ND]
};
__device__ inline SmemParams carve(float* smem, int in) {
  SmemParams s;
  s.w1t = smem;
  s.b1 = s.w1t + in * H1;
  s.w2 = s.b1 + H1;
  s.b2 = s.w2 + H2 * H1;
  s.w3 = s.b2 + H2;
  s.wd = s.w3 + H2;
  return s;
}
__host__ __device__ inline size_t smem_floats(int in) { return (size_t)in * H1 + H1 + H2 * H1 + H2 + H2 + WD_PAD; }

// w1t_global: W1 already transposed by k_tower_prep (training), or nullptr (forward only)
__device__ inline void load_params(const float* __restrict__ p, const float* __restrict__ w1t_global, const Layout& l,
                                   SmemParams s) {
  if (w1t_global != nullptr) {
    const float4* src = reinterpret_cast<const float4*>(w1t_global);
    float4* dst = reinterpret_cast<float4*>(s.w1t);
    for (int i = threadIdx.x; i < H1 * l.in / 4; i += blockDim.x) dst[i] = src[i];
  } else {
    for (int i = threadIdx.x; i < H1 * l.in; i += blockDim.x) {
      int j = i / l.in, e = i - j * l.in;  // coalesced read of w1[j][e]
      s.w1t[e * H1 + j] = p[l.o_w1 + i];
    }
  }
  for (int i = threadIdx.x; i < H1; i += blockDim.x) s.b1[i] = p[l.o_b1 + i];
  for (int i = threadIdx.x; i < H2 * H1; i += blockDim.x) s.w2[i] = p[l.o_w2 + i];
  for (int i = threadIdx.x; i < H2; i += blockDim.x) { s.b2[i] = p[l.o_b2 + i]; s.w3[i] = p[l.o_w3 + i]; }
  for (int i = threadIdx.x; i < ND; i += blockDim.x) s.wd[i] = p[l.o_wd + i];
  __syncthreads();
}

__device__ __forceinline__ float dot16(const float (&h)[H1], const float* __restrict__ w) {
  const float4* w4 = reinterpret_cast<const float4*>(w);
  float acc = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    float4 v = w4[q];
    acc = fmaf(v.x, h[4 * q + 0], acc);
    acc = fmaf(v.y, h[4 * q + 1], acc);
    acc = fmaf(v.z, h[4 * q + 2], acc);
    acc = fmaf(v.w, h[4 * q + 3], acc);
  }
  return acc;
}

// k_tower_a work split: a block = SPB samples x NPART group-parts.  Warp w handles NS samples per
// lane (register blocking: every shared-memory weight read feeds NS samples -- the kernel is bound
// by shared-memory bandwidth for the broadcast weight reads, then by gather latency) and the id
// groups g = w % NPART, + NPART, ...  (lane = sample keeps every weight read a broadcast;
// splitting the 38 groups over 4 warps quadruples the independent gather chains in flight).
constexpr int NPART = 4;
constexpr int NS = 2;                          // samples per lane
constexpr int SLAB = 32 * NS;                  // samples per warp
constexpr int SPB = 2 * SLAB;                  // samples per block (2 slabs x NPART warps = 8 warps)
constexpr int TA_THREADS = (SPB / SLAB) * NPART * 32;  // 256
constexpr int RW = H1 + D + 2;                 // partial-sum record: h[16] | s[8] | q | lin

__device__ __forceinline__ void axpy16x(float (&h)[NS][H1], const float* __restrict__ w, const float (&x)[NS]) {
  const float4* w4 = reinterpret_cast<const float4*>(w);
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = w4[q];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      h[n][4 * q + 0] = fmaf(v.x, x[n], h[n][4 * q + 0]);
      h[n][4 * q + 1] = fmaf(v.y, x[n], h[n][4 * q + 1]);
      h[n][4 * q + 2] = fmaf(v.z, x[n], h[n][4 * q + 2]);
      h[n][4 * q + 3] = fmaf(v.w, x[n], h[n][4 * q + 3]);
    }
  }
}
__device__ __forceinline__ void dot16x(float (&out)[NS], const float (&h)[NS][H1], const float* __restrict__ w) {
  const float4* w4 = reinterpret_cast<const float4*>(w);
#pragma unroll
  for (int n = 0; n < NS; ++n) out[n] = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 v = w4[q];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      out[n] = fmaf(v.x, h[n][4 * q + 0], out[n]);
      out[n] = fmaf(v.y, h[n][4 * q + 1], out[n]);
      out[n] = fmaf(v.z, h[n][4 * q + 2], out[n]);
      out[n] = fmaf(v.w, h[n][4 * q + 3], out[n]);
    }
  }
}

template <bool BACKWARD>
__global__ void __launch_bounds__(TA_THREADS, 2) k_tower_a(b200_deepfm_args_t a) {
  extern __shared__ __align__(16) float smem[];
  const Layout l = layout(a.G);
  SmemParams sp = carve(smem, l.in);
  float* red = smem + smem_floats(l.in);                       // [NPART][RW][SPB]
  int* sinv = reinterpret_cast<int*>(red + NPART * RW * SPB);  // [G][SPB]
  load_params(a.params, BACKWARD ? a.scratch + (long long)a.B * STATE : nullptr, l, sp);
  const int B = a.B, G = a.G;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int part = warp % NPART;
  const int sl0 = (warp / NPART) * SLAB + lane;  // sample slots of this lane: sl0 + 32*n
  float loss_acc = 0.f;
  const long long nblk = ((long long)B + SPB - 1) / SPB;
  for (long long blk = blockIdx.x; blk < nblk; blk += gridDim.x) {
    long long bb[NS];
    bool live[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      const long long b = blk * SPB + sl0 + 32 * n;
      live[n] = b < B;
      bb[n] = live[n] ? b : B - 1;  // dead lanes replay the last sample, results discarded
    }
    float h[NS][H1];
    float lin[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      lin[n] = 0.f;
#pragma unroll
      for (int j = 0; j < H1; ++j) h[n][j] = part == 0 ? sp.b1[j] : 0.f;
    }
    if (part == 0) {
#pragma unroll
      for (int e = 0; e < ND; ++e) {
        float x[NS];
#pragma unroll
        for (int n = 0; n < NS; ++n) {
          x[n] = a.dense[bb[n] * ND + e];
          lin[n] = fmaf(sp.wd[e], x[n], lin[n]);
        }
        axpy16x(h, sp.w1t + e * H1, x);
      }
    }
    float s[NS][D], q[NS];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      q[n] = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) s[n][d] = 0.f;
    }
    // pass 1 over this warp's groups: NS rank loads, then 3*NS independent row loads in flight
    for (int g = part; g < G; g += NPART) {
      int r[NS];
#pragma unroll
      for (int n = 0; n < NS; ++n) r[n] = a.inv[(long long)g * B + bb[n]];
      float4 e0[NS], e1[NS];
      float wv[NS];
#pragma unroll
      for (int n = 0; n < NS; ++n) {
        const float4* row = reinterpret_cast<const float4*>(a.bet_deep + ((long long)g * B + r[n]) * D);
        e0[n] = row[0];
        e1[n] = row[1];
        wv[n] = a.bet_wide[(long long)g * B + r[n]];
      }
      const float* w = sp.w1t + (ND + g * D) * H1;
      float ev[D][NS];
#pragma unroll
      for (int n = 0; n < NS; ++n) {
        sinv[g * SPB + sl0 + 32 * n] = r[n];
        lin[n] += wv[n];
        ev[0][n] = e0[n].x; ev[1][n] = e0[n].y; ev[2][n] = e0[n].z; ev[3][n] = e0[n].w;
        ev[4][n] = e1[n].x; ev[5][n] = e1[n].y; ev[6][n] = e1[n].z; ev[7][n] = e1[n].w;
      }
#pragma unroll
      for (int d = 0; d < D; ++d) {
#pragma unroll
        for (int n = 0; n < NS; ++n) {
          s[n][d] += ev[d][n];
          q[n] = fmaf(ev[d][n], ev[d][n], q[n]);
        }
        axpy16x(h, w + d * H1, ev[d]);
      }
    }
    // combine the NPART partial sums of each sample through shared memory
#pragma unroll
    for (int n = 0; n < NS; ++n) {
      float* mine = red + (part * RW) * SPB + sl0 + 32 * n;
#pragma unroll
      for (int j = 0; j < H1; ++j) mine[j * SPB] = h[n][j];
#pragma unroll
      for (int d = 0; d < D; ++d) mine[(H1 + d) * SPB] = s[n][d];
      mine[(H1 + D) * SPB] = q[n];
      mine[(H1 + D + 1) * SPB] = lin[n];
    }
    __syncthreads();
    float dz[NS], dh1[NS][H1];
#pragma unroll
    for (int n = 0; n < NS; ++n) {
#pragma unroll
      for (int j = 0; j < H1; ++j) h[n][j] = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) s[n][d] = 0.f;
      q[n] = 0.f;
      lin[n] = 0.f;
#pragma unroll
      for (int pt = 0; pt < NPART; ++pt) {
        const float* src = red + (pt * RW) * SPB + sl0 + 32 * n;
#pragma unroll
        for (int j = 0; j < H1; ++j) h[n][j] += src[j * SPB];
#pragma unroll
        for (int d = 0; d < D; ++d) s[n][d] += src[(H1 + d) * SPB];
        q[n] += src[(H1 + D) * SPB];
        lin[n] += src[(H1 + D + 1) * SPB];
      }
      float a1[H1];
#pragma unroll
      for (int j = 0; j < H1; ++j) a1[j] = fmaxf(h[n][j], 0.f);
      float h2[H2], dnn = 0.f;
#pragma unroll
      for (int k = 0; k < H2; ++k) {
        h2[k] = fmaxf(sp.b2[k] + dot16(a1, sp.w2 + k * H1), 0.f);
        dnn = fmaf(sp.w3[k], h2[k], dnn);
      }
      float ss = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) ss = fmaf(s[n][d], s[n][d], ss);
      const float z = lin[n] + dnn + 0.5f * (ss - q[n]);
      const long long b = blk * SPB + sl0 + 32 * n;
      if (part == 0 && live[n] && a.logits != nullptr) a.logits[b] = z;
      dz[n] = 0.f;
      if (BACKWARD) {
        float dh2[H2];
        const float lb = backward_tail(z, a.labels[bb[n]], live[n], B, h[n], h2, sp.w2, sp.w3, dz[n], dh2, dh1[n]);
        if (part == 0 && live[n]) {
          loss_acc += lb;
          store_state(a.scratch + b * STATE, dh1[n], a1, dh2, h2, dz[n]);  // backward state for k_tower_b
        }
      }
    }
    if (BACKWARD) {
      // pass 2: d loss / d embedding rows of this warp's groups, reduced per unique id
      // (deduplicate_indexed_slices' sum)
      for (int g = part; g < G; g += NPART) {
        int r[NS];
        float4 e0[NS], e1[NS];
#pragma unroll
        for (int n = 0; n < NS; ++n) {
          r[n] = sinv[g * SPB + sl0 + 32 * n];
          const float4* row = reinterpret_cast<const float4*>(a.bet_deep + ((long long)g * B + r[n]) * D);
          e0[n] = row[0];
          e1[n] = row[1];
        }
        const float* w = sp.w1t + (ND + g * D) * H1;
        float x[NS][D + 1];
        float ev[D][NS];
#pragma unroll
        for (int n = 0; n < NS; ++n) {
          ev[0][n] = e0[n].x; ev[1][n] = e0[n].y; ev[2][n] = e0[n].z; ev[3][n] = e0[n].w;
          ev[4][n] = e1[n].x; ev[5][n] = e1[n].y; ev[6][n] = e1[n].z; ev[7][n] = e1[n].w;
        }
#pragma unroll
        for (int d = 0; d < D; ++d) {
          float dt[NS];
          dot16x(dt, dh1, w + d * H1);
#pragma unroll
          for (int n = 0; n < NS; ++n) x[n][d] = fmaf(dz[n], s[n][d] - ev[d][n], dt[n]);
        }
#pragma unroll
        for (int n = 0; n < NS; ++n) {
          x[n][D] = dz[n];  // wide row gradient
          // the small tables of this model put ~10 equal ids in every warp
          dedup_red(x[n], r[n], live[n], lane, a, g);
        }
      }
    }
    __syncthreads();  // red / sinv are reused by the next block of samples
  }
  if (BACKWARD) add_warp_loss(loss_acc, a.loss, B, lane == 0 && part == 0);
}

__host__ inline size_t tower_a_smem(int G) {
  return (smem_floats(ND + G * D) + (size_t)NPART * RW * SPB) * sizeof(float) + (size_t)G * SPB * sizeof(int);
}

// parameter gradients.  dW1 = dH1^T [16 x B] . X [B x IN] is a contraction over the batch: a block
// stages a chunk of S samples in shared memory -- the per-sample backward state written by
// k_tower_a and the gathered input rows X (cooperative, fully independent 32 B row gathers) --
// then thread e owns input column e with 16 accumulators; the remaining threads own db1 and
// the small gradients (dW2, db2, dw3, dw_dense).  One atomicAdd per output per block.
constexpr int S_CHUNK = 32;  // 52 KB of shared memory per block -> 4 blocks (16 warps) per SM
constexpr int TB_COLW = 96;                    // threads owning dW1/db1 columns (3 warps)
constexpr int TB_CPT = 4;                      // columns per thread: each staged dh1 row feeds 64 FMAs
constexpr int TB_THREADS = TB_COLW + 32;       // + one warp for the small gradients

// tile row: [deep G*8 | dense 13 | 1.0 (bias column) | pad]
__host__ __device__ inline int tb_xpad(int G) { return (G * D + ND + 1 + 3) / 4 * 4; }
__host__ inline size_t tower_b_smem(int G) {
  return ((size_t)S_CHUNK * STATE + (size_t)S_CHUNK * tb_xpad(G)) * sizeof(float) + (size_t)G * S_CHUNK * sizeof(int);
}

__global__ void __launch_bounds__(TB_THREADS, 4) k_tower_b(b200_deepfm_args_t a) {
  extern __shared__ __align__(16) float smem_b[];
  const Layout l = layout(a.G);
  const int B = a.B, G = a.G, t = threadIdx.x;
  const int IN = l.in, XP = tb_xpad(G), NDEEP = G * D, NCOL = IN + 1;
  float* sc = smem_b;                                     // [S][STATE]
  float* xt = sc + S_CHUNK * STATE;                         // [S][XP]
  int* sinv = reinterpret_cast<int*>(xt + S_CHUNK * XP);  // [G][S]
  const bool is_col = t < TB_COLW;
  float acc[TB_CPT][H1];
#pragma unroll
  for (int i = 0; i < TB_CPT; ++i)
#pragma unroll
    for (int j = 0; j < H1; ++j) acc[i][j] = 0.f;
  float sacc[3] = {0.f, 0.f, 0.f};  // small outputs o = (t - TB_COLW) + 32*i
  const long long nchunk = ((long long)B + S_CHUNK - 1) / S_CHUNK;
  for (long long c = blockIdx.x; c < nchunk; c += gridDim.x) {
    const long long b0 = c * S_CHUNK;
    const int n = (int)min((long long)S_CHUNK, B - b0);
    __syncthreads();
    {
      const float4* src = reinterpret_cast<const float4*>(a.scratch + b0 * STATE);
      float4* dst = reinterpret_cast<float4*>(sc);
      for (int i = t; i < n * (STATE / 4); i += TB_THREADS) dst[i] = src[i];
      for (int i = t; i < n * (ND + 1); i += TB_THREADS) {
        const int s_ = i / (ND + 1), e = i - s_ * (ND + 1);
        xt[s_ * XP + NDEEP + e] = e < ND ? a.dense[(b0 + s_) * ND + e] : 1.0f;
      }
      for (int i = t; i < G * n; i += TB_THREADS) {  // coalesced rank loads
        const int g = i / n, s_ = i - g * n;
        sinv[g * S_CHUNK + s_] = a.inv[(long long)g * B + b0 + s_];
      }
    }
    __syncthreads();
#pragma unroll 4
    for (int i = t; i < n * G; i += TB_THREADS) {  // independent 32 B row gathers, group fastest
      const int s_ = i / G, g = i - s_ * G;
      const float4* row = reinterpret_cast<const float4*>(a.bet_deep + ((long long)g * B + sinv[g * S_CHUNK + s_]) * D);
      const float4 e0 = row[0], e1 = row[1];
      float4* dst = reinterpret_cast<float4*>(xt + s_ * XP + g * D);
      dst[0] = e0;
      dst[1] = e1;
    }
    __syncthreads();
    if (is_col) {
#pragma unroll 2
      for (int s_ = 0; s_ < n; ++s_) {
        const float4* d4 = reinterpret_cast<const float4*>(sc + s_ * STATE);
        const float4 q0 = d4[0], q1 = d4[1], q2 = d4[2], q3 = d4[3];
        const float dh[H1] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w, q2.x, q2.y, q2.z, q2.w, q3.x, q3.y, q3.z, q3.w};
#pragma unroll
        for (int i = 0; i < TB_CPT; ++i) {
          const int col = t + TB_COLW * i;
          const float x = col < NCOL ? xt[s_ * XP + col] : 0.f;
#pragma unroll
          for (int j = 0; j < H1; ++j) acc[i][j] = fmaf(dh[j], x, acc[i][j]);
        }
      }
    } else {
      for (int s_ = 0; s_ < n; ++s_) {
        const float* r = sc + s_ * STATE;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
          const int small = (t - TB_COLW) + 32 * i;
          if (small < NSMALL) sacc[i] += small_grad(small, r, xt + s_ * XP + NDEEP);
        }
      }
    }
  }
  if (is_col) {
#pragma unroll
    for (int i = 0; i < TB_CPT; ++i) {
      const int col = t + TB_COLW * i;
      if (col < NDEEP + ND) {
        const int e = col < NDEEP ? ND + col : col - NDEEP;  // tile column -> W1 input index (dense first)
#pragma unroll
        for (int j = 0; j < H1; ++j) atomicAdd(a.grads + l.o_w1 + j * IN + e, acc[i][j]);
      } else if (col == NDEEP + ND) {
#pragma unroll
        for (int j = 0; j < H1; ++j) atomicAdd(a.grads + l.o_b1 + j, acc[i][j]);
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 3; ++i) {
      const int small = (t - TB_COLW) + 32 * i;
      if (small < NSMALL) atomicAdd(a.grads + small_grad_offset(l, small), sacc[i]);
    }
  }
}

int check_args(const b200_deepfm_args_t* a, bool backward) {
  if (check_common(a, backward)) return -1;
  if (ND + a->G * D + 1 > TB_COLW * TB_CPT) return fail(-1, "too many id groups for the fused tower (max 46)");
  if (a->rows) return fail(-1, "the fused tower reads pulled rows only");
  if (backward && !a->scratch) return fail(-1, "null output");
  return 0;
}

unsigned tower_a_grid(int B, int n_sm) {
  const long long blocks = ((long long)B + SPB - 1) / SPB, cap = (long long)n_sm * 8;
  return (unsigned)(blocks < cap ? blocks : cap);
}

}  // namespace

extern "C" {

size_t b200_deepfm_param_count(int G) { return (size_t)layout(G).total; }
int64_t b200_deepfm_launch_count(void) { return g_launches; }
const char* b200_deepfm_last_error(void) { return last_error().c_str(); }

int b200_deepfm_fwd_bwd(const b200_deepfm_args_t* args, void* stream) {
  if (check_args(args, true)) return -1;
  cudaStream_t st = (cudaStream_t)stream;
  const Layout l = layout(args->G);
  int n_sm;
  const int dev = current_device(&n_sm);
  max_dynamic_smem_once<k_tower_a<true>>(dev, 110 * 1024);
  max_dynamic_smem_once<k_tower_b>(dev, 110 * 1024);
  k_tower_prep<<<dim3(8, args->G), 256, 0, st>>>(*args, l.total);
  k_tower_a<true><<<tower_a_grid(args->B, n_sm), TA_THREADS, tower_a_smem(args->G), st>>>(*args);
  const long long chunks = ((long long)args->B + S_CHUNK - 1) / S_CHUNK;
  const long long cap = (long long)n_sm * 4;  // 4 blocks per SM by shared memory / registers
  k_tower_b<<<(unsigned)(chunks < cap ? chunks : cap), TB_THREADS, tower_b_smem(args->G), st>>>(*args);
  g_launches += 3;
  return launch_status();
}

int b200_deepfm_forward(const b200_deepfm_args_t* args, void* stream) {
  if (check_args(args, false)) return -1;
  int n_sm;
  const int dev = current_device(&n_sm);
  max_dynamic_smem_once<k_tower_a<false>>(dev, 110 * 1024);
  k_tower_a<false><<<tower_a_grid(args->B, n_sm), TA_THREADS, tower_a_smem(args->G), (cudaStream_t)stream>>>(*args);
  g_launches += 1;
  return launch_status();
}

}  // extern "C"
