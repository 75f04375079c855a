// What the three DeepFM towers (deepfm_tower.cu "fused", deepfm_tower2.cu "tile", deepfm_tower_mma.cu "mma") share:
// the model and its flat parameter layout (include/b200_deepfm.h), the zeroing of the step's outputs, the
// per-sample tail, the per-sample backward state and the small gradients read from it, the warp-level id dedup
// of the row gradients, the loss reduction, cp.async, and the host side of an entry point (argument checks,
// shared-memory limit, launch errors and the one error message of b200_deepfm_last_error).
#pragma once
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_deepfm.h"

namespace deepfm {

constexpr int ND = B200_DEEPFM_NDENSE, D = B200_DEEPFM_DIM, H1 = B200_DEEPFM_H1, H2 = B200_DEEPFM_H2;
constexpr int WD_PAD = 16;                     // w_dense padded to 16 floats
constexpr int NSMALL = H2 * H1 + 2 * H2 + ND;  // small gradients: dW2 64 | db2 4 | dw3 4 | dw_dense 13
// per-sample backward state record: dh1 16 | a1 16 | dh2 4 | h2 4 | dz | pad 3
constexpr int STATE = B200_DEEPFM_SCRATCH;
constexpr int ST_A1 = H1, ST_DH2 = 2 * H1, ST_H2 = ST_DH2 + H2, ST_DZ = ST_H2 + H2;
static_assert(ST_DZ + 4 == STATE, "include/b200_deepfm.h");

// flat parameter / gradient layout: [ w_dense 13 (+3 pad) | w1 16 x in | b1 16 | w2 4 x 16 | b2 4 | w3 4 ]
struct Layout {
  int in;  // ND + G*D
  int o_wd, o_w1, o_b1, o_w2, o_b2, o_w3, total;
};
__host__ __device__ inline Layout layout(int G) {
  Layout l;
  l.in = ND + G * D;
  l.o_wd = 0;
  l.o_w1 = WD_PAD;
  l.o_b1 = l.o_w1 + H1 * l.in;
  l.o_w2 = l.o_b1 + H1;
  l.o_b2 = l.o_w2 + H2 * H1;
  l.o_w3 = l.o_b2 + H2;
  l.total = l.o_w3 + H2;
  return l;
}

// Zero what a training step accumulates into: the loss and the gradients (block row y = 0) and the live rows of
// the per-unique-id sums (block rows stride over the groups; rows >= n_unique[g] are never read by the push).
// Outputs that are null (forward only) are skipped.
__device__ __forceinline__ void zero_step_outputs(const b200_deepfm_args_t& a, int n_params) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (blockIdx.y == 0) {
    if (tid == 0 && a.loss) *a.loss = 0.f;
    if (a.grads)
      for (long long i = tid; i < n_params; i += stride) a.grads[i] = 0.f;
  }
  if (a.gsum_deep == nullptr) return;
  for (int g = blockIdx.y; g < a.G; g += gridDim.y) {
    const int u = a.n_unique[g];
    float* gw = a.gsum_wide + (long long)g * a.B;
    float4* gd = reinterpret_cast<float4*>(a.gsum_deep + (long long)g * a.B * D);
    for (long long i = tid; i < u; i += stride) gw[i] = 0.f;
    for (long long i = tid; i < 2LL * u; i += stride) gd[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

// Forward of one sample from its layer-1 pre-activations hpre (b1 included), FM sums s, FM square sum q and
// linear term lin: a1 = relu(hpre), h2 = relu(W2 a1 + b2) (the sum starts at b2), returns the logit
// z = lin + w3 . h2 + (|s|^2 - q) / 2.  w2 / b2 / w3 in the flat layout's order.
__device__ __forceinline__ float forward_tail(const float (&hpre)[H1], const float (&s)[D], float q, float lin,
                                              const float* w2, const float* b2, const float* w3, float (&a1)[H1],
                                              float (&h2)[H2]) {
#pragma unroll
  for (int j = 0; j < H1; ++j) a1[j] = fmaxf(hpre[j], 0.f);
  float dnn = 0.f;
#pragma unroll
  for (int k = 0; k < H2; ++k) {
    float acc = b2[k];
#pragma unroll
    for (int j = 0; j < H1; ++j) acc = fmaf(w2[k * H1 + j], a1[j], acc);
    h2[k] = fmaxf(acc, 0.f);
    dnn = fmaf(w3[k], h2[k], dnn);
  }
  float ss = 0.f;
#pragma unroll
  for (int d = 0; d < D; ++d) ss = fmaf(s[d], s[d], ss);
  return lin + dnn + 0.5f * (ss - q);
}

// Backward of one sample with logit z and label y: returns its binary cross entropy with logits and sets
// dz = (sigmoid(z) - y) / B (0 for a dead sample), dh2 and dh1 = d loss / d layer-1 pre-activation.
__device__ __forceinline__ float backward_tail(float z, float y, bool live, int B, const float (&hpre)[H1],
                                               const float (&h2)[H2], const float* w2, const float* w3, float& dz,
                                               float (&dh2)[H2], float (&dh1)[H1]) {
  const float lb = fmaxf(z, 0.f) - z * y + log1pf(expf(-fabsf(z)));
  const float p = 1.f / (1.f + expf(-z));
  dz = live ? (p - y) / (float)B : 0.f;
#pragma unroll
  for (int k = 0; k < H2; ++k) dh2[k] = h2[k] > 0.f ? dz * w3[k] : 0.f;
#pragma unroll
  for (int j = 0; j < H1; ++j) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < H2; ++k) acc = fmaf(w2[k * H1 + j], dh2[k], acc);
    dh1[j] = hpre[j] > 0.f ? acc : 0.f;
  }
  return lb;
}

// The backward state record of one sample (m 16-byte aligned, STATE floats).
__device__ __forceinline__ void store_state(float* m, const float (&dh1)[H1], const float (&a1)[H1],
                                            const float (&dh2)[H2], const float (&h2)[H2], float dz) {
  float4* m4 = reinterpret_cast<float4*>(m);
#pragma unroll
  for (int qd = 0; qd < 4; ++qd) m4[qd] = make_float4(dh1[4 * qd], dh1[4 * qd + 1], dh1[4 * qd + 2], dh1[4 * qd + 3]);
#pragma unroll
  for (int qd = 0; qd < 4; ++qd) m4[4 + qd] = make_float4(a1[4 * qd], a1[4 * qd + 1], a1[4 * qd + 2], a1[4 * qd + 3]);
  m4[8] = make_float4(dh2[0], dh2[1], dh2[2], dh2[3]);
  m4[9] = make_float4(h2[0], h2[1], h2[2], h2[3]);
  m4[10] = make_float4(dz, 0.f, 0.f, 0.f);
}

// One sample's share of small gradient o (0 <= o < NSMALL) from its backward state record m and its dense
// features: dW2 = dh2 a1^T | db2 = dh2 | dw3 = dz h2 | dw_dense = dz dense.
__device__ __forceinline__ float small_grad(int o, const float* m, const float* dense) {
  if (o < H2 * H1) return m[ST_DH2 + o / H1] * m[ST_A1 + o % H1];
  if (o < H2 * H1 + H2) return m[ST_DH2 + o - H2 * H1];
  if (o < H2 * H1 + 2 * H2) return m[ST_DZ] * m[ST_H2 + o - H2 * H1 - H2];
  return m[ST_DZ] * dense[o - H2 * H1 - 2 * H2];
}
// small gradient o -> offset in the flat gradient layout
__host__ __device__ inline int small_grad_offset(const Layout& l, int o) {
  if (o < H2 * H1) return l.o_w2 + o;
  if (o < H2 * H1 + H2) return l.o_b2 + o - H2 * H1;
  if (o < H2 * H1 + 2 * H2) return l.o_w3 + o - H2 * H1 - H2;
  return l.o_wd + o - H2 * H1 - 2 * H2;
}

// Warp-level id dedup of one row gradient per lane, x = [deep 8 | wide 1] of row r of group g: lanes hitting the
// same row combine pairwise up a tree threaded through the __match_any_sync peer mask (pointer doubling,
// ceil(log2(max multiplicity)) rounds for the whole warp), then the lowest lane of each row adds the sum into
// gsum_deep / gsum_wide with one vector red.  A dead lane keeps a key of its own and writes nothing.  All 32
// lanes call it.
__device__ __forceinline__ void dedup_red(float (&x)[D + 1], int r, bool live, int lane, const b200_deepfm_args_t& a,
                                          int g) {
  const int key = live ? r : -1 - lane;
  const unsigned peers = __match_any_sync(0xffffffffu, key);
  const int rank = __popc(peers & ((1u << lane) - 1));
  const int maxn = __reduce_max_sync(0xffffffffu, (unsigned)__popc(peers));
  const unsigned above = peers & ~((2u << lane) - 1);
  int nxt = above ? __ffs(above) - 1 : -1;  // the peer `step` ranks above this lane
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
    float* od = a.gsum_deep + ((long long)g * a.B + r) * D;
    atomicAdd(reinterpret_cast<float4*>(od), make_float4(x[0], x[1], x[2], x[3]));
    atomicAdd(reinterpret_cast<float4*>(od + 4), make_float4(x[4], x[5], x[6], x[7]));
    atomicAdd(a.gsum_wide + (long long)g * a.B + r, x[D]);
  }
}

// Sum of the warp's loss terms; `add` (lane 0 of one warp per sample) adds sum / B into *loss.  All 32 lanes call it.
__device__ __forceinline__ void add_warp_loss(float v, float* loss, int B, bool add) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  if (add) atomicAdd(loss, v / (float)B);
}

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// ---- host side of the entry points

// The message of the last refusal or launch error of any tower entry point (b200_deepfm_last_error).
inline std::string& last_error() {
  static thread_local std::string msg;
  return msg;
}
inline int fail(int rc, const char* msg) {
  last_error() = msg;
  return rc;
}

// The checks every tower makes (-1 and the message, or 0).  A tower adds its group limit, what it needs of
// `scratch` and whether it takes a row source.  Training needs every output but `logits`, forward-only `logits`.
inline int check_common(const b200_deepfm_args_t* a, bool backward) {
  if (!a || a->G < 1 || a->B < 1) return fail(-1, "bad shape");
  if (!a->inv || !a->dense || !a->params || (!a->rows && (!a->bet_wide || !a->bet_deep))) return fail(-1, "null input");
  if (backward ? (!a->labels || !a->grads || !a->gsum_wide || !a->gsum_deep || !a->loss || !a->n_unique) : !a->logits)
    return fail(-1, "null output");
  return 0;
}

// the current device and its SM count
inline int current_device(int* n_sm) {
  int dev = 0;
  *n_sm = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(n_sm, cudaDevAttrMultiProcessorCount, dev);
  return dev;
}

// Raise Kernel's dynamic shared memory limit to `bytes`, once per device (it is a driver call).
template <auto Kernel>
void max_dynamic_smem_once(int dev, int bytes) {
  static bool done[64] = {};
  if (dev < 64 && !done[dev]) {
    cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    done[dev] = true;
  }
}

// After an entry point's launches: 0, or -2 and the launch error's message.
inline int launch_status() {
  const cudaError_t e = cudaGetLastError();
  return e == cudaSuccess ? 0 : fail(-2, cudaGetErrorString(e));
}

}  // namespace deepfm
