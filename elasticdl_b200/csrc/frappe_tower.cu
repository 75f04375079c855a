// Frappe DeepFM tower (include/b200_frappe.h): masked dim-64 / dim-1 rows of 10 fields, FM, the linear
// Dense(64) -> Dense(1) stack, loss, backward and the two per-unique-row gradient segments.
//
// The Dense stack has no activation, so with v = K w2 [640] and c = b . w2 + b2 the deep term of sample b is
// x_b . v + c and no per-sample hidden layer is formed.  Per occurrence (b, f) the deep row's gradient is
// m_bf g_b (S_b - e_bf + v_f) and the wide row's is m_bf g_b; the dense gradients are dK = s w2^T, db = G w2,
// dw2 = K^T s + G b and db2 = G with s = sum_b g_b x_b and G = sum_b g_b.
//
// Two launches per call:
//   k_frappe_prologue: v, c into the workspace; zeroes the n_unique rows of gsum (read on the device).
//   k_frappe_main: a persistent grid over tiles of 64 samples, 10 warps per CTA.
//     phase 0  the tile's masked inverse ids and wide rows into shared memory;
//     phase 1  warp f matches the tile's occurrences of field f (__match_any_sync over 32 samples): which
//              occurrences share a row;
//     phase 2  a warp per sample (lanes = dims 2l, 2l+1): the forward, the loss, g_b; an occurrence whose row no
//              other of its 32 samples has is pushed from registers (one vector red);
//     phase 3  warp f adds up each shared row of field f over its samples (the hot rows of the small fields)
//              and issues one vector red per row and 32 samples.
//   s, G and the loss are summed per CTA in shared memory, then added to the workspace; the last CTA to arrive
//   writes the dense gradients and the loss and zeroes the accumulators and its counter.
#include <cuda_runtime.h>

#include <atomic>
#include <cstdint>
#include <string>

#include "../../include/b200_frappe.h"

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};
int fail(int code, const std::string& m) {
  g_err = m;
  return code;
}

constexpr int F = B200_FRAPPE_FIELDS;
constexpr int D = B200_FRAPPE_DIM;
constexpr int X = F * D;  // 640: the Dense(64) input
constexpr int TILE = B200_FRAPPE_TILE;
constexpr int WARPS = F;  // phase 1 / 3: one warp per field
constexpr int THREADS = 32 * WARPS;
constexpr int OB = X * D, OW2 = OB + D, OB2 = OW2 + D, NPARAM = B200_FRAPPE_PARAMS;
static_assert(OB2 + 1 == NPARAM, "flat layout");
// workspace (floats): arrival counter @0 | s [640] @16 | G @656 | loss sum @657 | v [640] @672 | c @1312
constexpr int WS_S = 16, WS_G = WS_S + X, WS_L = WS_G + 1, WS_V = 672, WS_C = WS_V + X;
constexpr size_t WS_BYTES = (WS_C + 16) * sizeof(float);

struct Smem {
  float v[X];
  float S[TILE][D];           // S_b of the tile's samples
  int inv[TILE * F];          // the dedup's inverse id of (r, f), -1 where masked or past the batch
  float wide[TILE * F];       // m_bf W[id_bf]
  unsigned peers[TILE / 32][F][32];  // __match_any_sync of field f's inverse ids over the 32 samples of a half
  float g[TILE];
  float red[X];               // the CTA's s; in the last CTA the total s
  float misc[4];              // G, loss sum, c
  float part[5][D];           // the last CTA's K^T s partials
  unsigned last;
};

__device__ __forceinline__ float warp_sum(float x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

__global__ void __launch_bounds__(256) k_frappe_prologue(b200_frappe_args_t a, int zero) {
  float* ws = reinterpret_cast<float*>(a.workspace);
  const int lane = threadIdx.x & 31;
  const int gw = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  const float2 w2 = __ldg(reinterpret_cast<const float2*>(a.params + OW2) + lane);
  for (int i = gw; i <= X; i += nw) {  // v[i] = K[i, :] . w2 (warp i < 640); c = b . w2 + b2 (warp 640)
    const float2 k = __ldg(reinterpret_cast<const float2*>(a.params + (i < X ? i * D : OB)) + lane);
    const float t = warp_sum(k.x * w2.x + k.y * w2.y);
    if (lane == 0) ws[i < X ? WS_V + i : WS_C] = i < X ? t : t + __ldg(a.params + OB2);
  }
  if (!zero) return;
  const long long n = *a.n_unique;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = (long long)gridDim.x * blockDim.x;
  float4* gd = reinterpret_cast<float4*>(a.gsum_deep);
  for (long long i = tid; i < n * (D / 4); i += stride) gd[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long i = tid; i < n; i += stride) a.gsum_wide[i] = 0.f;
}

__global__ void __launch_bounds__(THREADS, 2) k_frappe_main(b200_frappe_args_t a, int ntiles, int train) {
  __shared__ Smem s;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int64_t B = a.B;
  const float* ws_in = reinterpret_cast<const float*>(a.workspace);
  for (int i = t; i < X; i += THREADS) {
    s.v[i] = __ldcg(ws_in + WS_V + i);
    s.red[i] = 0.f;
  }
  if (t == 0) {
    s.misc[0] = 0.f;
    s.misc[1] = 0.f;
    s.misc[2] = __ldcg(ws_in + WS_C);
  }
  const float2* bet2 = reinterpret_cast<const float2*>(a.bet_deep);
  float2* gsum2 = reinterpret_cast<float2*>(a.gsum_deep);
  float2 acc[F];  // this lane's dims of s for the samples this warp owns
#pragma unroll
  for (int f = 0; f < F; ++f) acc[f] = make_float2(0.f, 0.f);
  float accG = 0.f, accL = 0.f;
  __syncthreads();
  const float c = s.misc[2];

  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t base = (int64_t)tile * TILE;
    const int n = B - base < TILE ? (int)(B - base) : TILE;
    // phase 0
    for (int i = t; i < TILE * F; i += THREADS) {
      int u = -1;
      float w = 0.f;
      if (i < n * F) {
        const int64_t j = base * F + i;
        if (__ldg(a.ids + j) != 0) {
          u = __ldg(a.inv + j);
          w = __ldg(a.bet_wide + u);
        }
      }
      s.inv[i] = u;
      s.wide[i] = w;
    }
    __syncthreads();
    // phase 1
    if (train) {
#pragma unroll
      for (int h = 0; h < TILE / 32; ++h) s.peers[h][warp][lane] = __match_any_sync(0xffffffffu, s.inv[(32 * h + lane) * F + warp]);
      __syncthreads();
    }
    // phase 2
    for (int r = warp; r < n; r += WARPS) {
      const int64_t b = base + r;
      float2 e[F];
#pragma unroll
      for (int f = 0; f < F; ++f) {
        const int u = s.inv[r * F + f];
        e[f] = u >= 0 ? __ldg(bet2 + (size_t)u * (D / 2) + lane) : make_float2(0.f, 0.f);
      }
      float2 S = make_float2(0.f, 0.f);
      float sq = 0.f, dot = 0.f, first = 0.f;
#pragma unroll
      for (int f = 0; f < F; ++f) {
        S.x += e[f].x;
        S.y += e[f].y;
        sq = fmaf(e[f].x, e[f].x, fmaf(e[f].y, e[f].y, sq));
        const float2 vf = *reinterpret_cast<const float2*>(s.v + f * D + 2 * lane);
        dot = fmaf(e[f].x, vf.x, fmaf(e[f].y, vf.y, dot));
        first += s.wide[r * F + f];
      }
      const float part = 0.5f * (fmaf(S.x, S.x, S.y * S.y) - sq) + dot;
      const float z = first + warp_sum(part) + c;
      if (lane == 0) a.logits[b] = z;
      if (!train) continue;
      const float y = __ldg(a.labels + b);
      const float p = 1.f / (1.f + expf(-z));
      const float g = (p - y) / (float)B;
      if (lane == 0) {
        accL += fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));  // sigmoid cross-entropy with logits
        accG += g;
        s.g[r] = g;
      }
      *reinterpret_cast<float2*>(&s.S[r][2 * lane]) = S;
#pragma unroll
      for (int f = 0; f < F; ++f) {
        acc[f].x = fmaf(g, e[f].x, acc[f].x);
        acc[f].y = fmaf(g, e[f].y, acc[f].y);
        const int u = s.inv[r * F + f];
        if (u >= 0 && __popc(s.peers[r >> 5][f][r & 31]) == 1) {  // no other sample of its half has this row
          const float2 vf = *reinterpret_cast<const float2*>(s.v + f * D + 2 * lane);
          atomicAdd(gsum2 + (size_t)u * (D / 2) + lane,
                    make_float2(g * ((S.x - e[f].x) + vf.x), g * ((S.y - e[f].y) + vf.y)));
          if (lane == 0) atomicAdd(a.gsum_wide + u, g);
        }
      }
    }
    if (train) {
      __syncthreads();
      // phase 3: warp = field; rows that several samples of a half share
      const int f = warp;
      const float2 vf = *reinterpret_cast<const float2*>(s.v + f * D + 2 * lane);
#pragma unroll 1
      for (int h = 0; h < TILE / 32 && 32 * h < n; ++h) {
        const unsigned pr = s.peers[h][f][lane];
        const int u = s.inv[(32 * h + lane) * F + f];
        unsigned lead = __ballot_sync(0xffffffffu, u >= 0 && __popc(pr) > 1 && lane == __ffs(pr) - 1);
        while (lead) {  // four rows at a time: their loads are in flight together
          int L[4];
          float2 er[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            L[k] = lead ? __ffs(lead) - 1 : -1;
            if (lead) lead &= lead - 1;
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const int uk = __shfl_sync(0xffffffffu, u, L[k] < 0 ? 0 : L[k]);
            er[k] = L[k] >= 0 ? __ldg(bet2 + (size_t)uk * (D / 2) + lane) : make_float2(0.f, 0.f);
          }
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            if (L[k] < 0) break;
            const int uk = __shfl_sync(0xffffffffu, u, L[k]);
            unsigned m = __shfl_sync(0xffffffffu, pr, L[k]);
            float2 sum = make_float2(0.f, 0.f);
            float C = 0.f;
            while (m) {
              const int r = 32 * h + __ffs(m) - 1;
              m &= m - 1;
              const float g = s.g[r];
              const float2 S = *reinterpret_cast<const float2*>(&s.S[r][2 * lane]);
              sum.x = fmaf(g, S.x, sum.x);
              sum.y = fmaf(g, S.y, sum.y);
              C += g;
            }
            atomicAdd(gsum2 + (size_t)uk * (D / 2) + lane,
                      make_float2(fmaf(C, vf.x - er[k].x, sum.x), fmaf(C, vf.y - er[k].y, sum.y)));
            if (lane == 0) atomicAdd(a.gsum_wide + uk, C);
          }
        }
      }
    }
    __syncthreads();
  }
  if (!train) return;

  // the CTA's s, G and loss sum -> the workspace; the last CTA finishes
  float* ws = reinterpret_cast<float*>(a.workspace);
#pragma unroll
  for (int f = 0; f < F; ++f) {
    atomicAdd(&s.red[f * D + 2 * lane], acc[f].x);
    atomicAdd(&s.red[f * D + 2 * lane + 1], acc[f].y);
  }
  if (lane == 0) {
    atomicAdd(&s.misc[0], accG);
    atomicAdd(&s.misc[1], accL);
  }
  __syncthreads();
  for (int i = t; i < X; i += THREADS) atomicAdd(ws + WS_S + i, s.red[i]);
  if (t == 0) {
    atomicAdd(ws + WS_G, s.misc[0]);
    atomicAdd(ws + WS_L, s.misc[1]);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) s.last = atomicAdd(reinterpret_cast<unsigned*>(ws), 1u) == gridDim.x - 1;
  __syncthreads();
  if (!s.last) return;
  __threadfence();
  for (int i = t; i < X; i += THREADS) s.red[i] = __ldcg(ws + WS_S + i);
  if (t == 0) {
    s.misc[0] = __ldcg(ws + WS_G);
    s.misc[1] = __ldcg(ws + WS_L);
  }
  __syncthreads();
  for (int i = t; i < X; i += THREADS) ws[WS_S + i] = 0.f;  // ready for the next call
  if (t == 0) {
    ws[WS_G] = 0.f;
    ws[WS_L] = 0.f;
    *a.loss = s.misc[1] / (float)B;
    *reinterpret_cast<unsigned*>(ws) = 0u;
  }
  const float G = s.misc[0];
  const float* K = a.params;
  const float* w2 = a.params + OW2;
  for (int i = t; i < X * D; i += THREADS) a.grads[i] = s.red[i / D] * __ldg(w2 + (i % D));
  if (t < D) {
    a.grads[OB + t] = G * __ldg(w2 + t);
    if (t == 0) a.grads[OB2] = G;
  }
  if (t < 5 * D) {  // K^T s: column t % 64, rows [128 (t / 64), +128)
    const int j = t % D, i0 = (t / D) * (X / 5);
    float p = 0.f;
#pragma unroll 8
    for (int i = i0; i < i0 + X / 5; ++i) p = fmaf(__ldg(K + i * D + j), s.red[i], p);
    s.part[t / D][j] = p;
  }
  __syncthreads();
  if (t < D) {
    const float kts = (((s.part[0][t] + s.part[1][t]) + s.part[2][t]) + s.part[3][t]) + s.part[4][t];
    a.grads[OW2 + t] = fmaf(G, __ldg(a.params + OB + t), kts);
  }
}

constexpr int kMaxDevices = 64;
std::atomic<int> g_grid[kMaxDevices], g_sms[kMaxDevices];

// CTAs of the main pass that fit on the device at once (its persistent grid), and the SM count
int main_grid_cap(int dev, int* sms_out) {
  int n = dev < kMaxDevices ? g_grid[dev].load() : 0;
  int sms = dev < kMaxDevices ? g_sms[dev].load() : 0;
  if (n == 0 || sms == 0) {
    int per = 1;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms < 1) sms = 1;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, k_frappe_main, THREADS, 0) != cudaSuccess || per < 1)
      per = 1;
    n = sms * per;
    if (dev < kMaxDevices) {
      g_sms[dev].store(sms);
      g_grid[dev].store(n);
    }
  }
  *sms_out = sms;
  return n;
}

int launch(const b200_frappe_args_t* args, void* stream, int train) {
  if (!args) return fail(-1, "args is null");
  const b200_frappe_args_t& a = *args;
  if (a.B < 1 || (int64_t)a.B * F > INT32_MAX) return fail(-1, "batch size must be in [1, 2^31 / 10)");
  if (!a.ids || !a.inv || !a.bet_deep || !a.bet_wide || !a.params || !a.logits || !a.workspace ||
      (train && (!a.n_unique || !a.labels || !a.loss || !a.grads || !a.gsum_deep || !a.gsum_wide)))
    return fail(-1, "a buffer is null");
  if ((reinterpret_cast<uintptr_t>(a.bet_deep) & 15u) || (train && (reinterpret_cast<uintptr_t>(a.gsum_deep) & 15u)) ||
      (reinterpret_cast<uintptr_t>(a.params) & 7u))
    return fail(-1, "bet_deep and gsum_deep must be 16-byte aligned, params 8-byte aligned");
  if (a.workspace_bytes < WS_BYTES)
    return fail(-1, "workspace of " + std::to_string(a.workspace_bytes) + " bytes, needs " + std::to_string(WS_BYTES));
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(-2, "cudaGetDevice failed");
  const cudaStream_t st = (cudaStream_t)stream;
  int sms = 1;
  const int cap = main_grid_cap(dev, &sms);
  // at least one warp per entry of v and c; two CTAs per SM for the zeroing
  const int pro = 2 * sms > (X + 1 + 7) / 8 ? 2 * sms : (X + 1 + 7) / 8;
  k_frappe_prologue<<<pro, 256, 0, st>>>(a, train);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(-2, std::string("k_frappe_prologue: ") + cudaGetErrorString(e));
  const int ntiles = (int)((a.B + TILE - 1) / TILE);
  k_frappe_main<<<ntiles < cap ? ntiles : cap, THREADS, 0, st>>>(a, ntiles, train);
  e = cudaGetLastError();
  if (e != cudaSuccess) return fail(-2, std::string("k_frappe_main: ") + cudaGetErrorString(e));
  g_launches.fetch_add(1);
  return 0;
}

}  // namespace

extern "C" {

const char* b200_frappe_last_error(void) { return g_err.c_str(); }
int64_t b200_frappe_launch_count(void) { return g_launches.load(); }
size_t b200_frappe_workspace_bytes(int64_t B) { return B < 1 ? 0 : WS_BYTES; }
int b200_frappe_tower(const b200_frappe_args_t* args, void* stream) { return launch(args, stream, 1); }
int b200_frappe_forward(const b200_frappe_args_t* args, void* stream) { return launch(args, stream, 0); }

}  // extern "C"
