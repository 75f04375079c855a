// Evaluation metric kernels (include/b200_metrics.h): the Keras AUC state update as one histogram pass.
//
// k_auc_update: a grid-stride pass over the predictions; each CTA keeps its histogram in shared memory as uint32
// counters, one copy per warp (or per group of warps when T is too large for eight copies), because predictions
// cluster and one shared histogram would serialise the warps on the hot buckets.  Inside a warp, lanes with the same
// (label, bucket) are combined with __match_any_sync before one shared atomic.  At the end the CTA sums its copies
// and issues one 64-bit atomicAdd per non-zero bucket.  A CTA's counts stay below 2^31 because n does.
//
// The bucket is a closed-form guess floor(p (T - 1)) corrected by comparisons against the exact fp32 thresholds,
// so it equals the number of thresholds t with t < p whatever the guess (for Keras' thresholds the guess is off by
// at most one).
#include <cuda_runtime.h>

#include <cstdint>
#include <string>

#include "../../include/b200_metrics.h"
#include "launch.cuh"

namespace {

using E = entry::Entry<entry::Metrics>;
entry::LaunchCount g_launches{0};

constexpr int THREADS = B200_METRICS_THREADS;
constexpr int WARPS = THREADS / 32;
constexpr int UNROLL = 4;  // loads in flight per lane before the first atomic

// dynamic shared memory: thresholds float [T] | copies x uint32 [2][T + 1] | the invalid count
size_t smem_bytes(int T, int copies) {
  return sizeof(float) * T + sizeof(unsigned) * ((size_t)copies * 2 * (T + 1) + 1);
}

__global__ void __launch_bounds__(THREADS) k_auc_update(const float* __restrict__ probs,
                                                         const float* __restrict__ labels, int64_t n,
                                                         const float* __restrict__ thresholds, int T, int copies,
                                                         unsigned long long* __restrict__ hist,
                                                         unsigned long long* __restrict__ invalid) {
  extern __shared__ float smem[];
  float* thr = smem;
  unsigned* h = reinterpret_cast<unsigned*>(smem + T);
  const int bins = 2 * (T + 1);
  unsigned* bad = h + copies * bins;
  for (int i = threadIdx.x; i < T; i += THREADS) thr[i] = __ldg(thresholds + i);
  for (int i = threadIdx.x; i < copies * bins; i += THREADS) h[i] = 0u;
  if (threadIdx.x == 0) *bad = 0u;
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned* mine = h + (warp % copies) * bins;
  const float scale = (float)(T - 1);
  const int64_t stride = (int64_t)gridDim.x * THREADS;
  unsigned nbad = 0;
  // i0 is uniform over the warp, so every lane reaches __match_any_sync
  for (int64_t i0 = (int64_t)blockIdx.x * THREADS + warp * 32; i0 < n; i0 += UNROLL * stride) {
    float p[UNROLL], y[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t i = i0 + u * stride + lane;
      p[u] = i < n ? __ldg(probs + i) : 0.f;
      y[u] = i < n ? __ldg(labels + i) : 0.f;
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const int64_t i = i0 + u * stride + lane;
      int key = -1;
      if (i < n) {
        const float v = p[u];
        if (v >= 0.f && v <= 1.f) {
          int k = (int)(v * scale);
          while (k < T && thr[k] < v) ++k;
          while (k > 0 && !(thr[k - 1] < v)) --k;
          key = (y[u] != 0.f ? T + 1 : 0) + k;
        } else {
          ++nbad;  // NaN, below 0 or above 1
        }
      }
      const unsigned peers = __match_any_sync(0xffffffffu, key);
      if (key >= 0 && lane == __ffs(peers) - 1) atomicAdd(mine + key, (unsigned)__popc(peers));
    }
  }
  nbad = __reduce_add_sync(0xffffffffu, nbad);
  if (lane == 0 && nbad) atomicAdd(bad, nbad);
  __syncthreads();

  for (int b = threadIdx.x; b < bins; b += THREADS) {
    unsigned long long s = 0;
    for (int c = 0; c < copies; ++c) s += h[c * bins + b];
    if (s) atomicAdd(hist + b, s);
  }
  if (threadIdx.x == 0 && *bad) atomicAdd(invalid, (unsigned long long)*bad);
}

}  // namespace

extern "C" {

const char* b200_metrics_last_error(void) { return E::last_error().c_str(); }
int64_t b200_metrics_launch_count(void) { return g_launches.load(); }

int b200_metrics_auc_update(const float* probs, const float* labels, int64_t n, const float* thresholds, int32_t T,
                            uint64_t* hist, uint64_t* invalid, void* stream) {
  if (T < B200_METRICS_MIN_THRESHOLDS || T > B200_METRICS_MAX_THRESHOLDS)
    return E::fail(-1, "num_thresholds must be in [" + std::to_string(B200_METRICS_MIN_THRESHOLDS) + ", " +
                           std::to_string(B200_METRICS_MAX_THRESHOLDS) + "], not " + std::to_string(T));
  if (n < 0 || n > INT32_MAX) return E::fail(-1, "n must be in [0, 2^31), not " + std::to_string(n));
  if (!thresholds || !hist || !invalid) return E::fail(-1, "a buffer is null");
  if (n == 0) return 0;
  if (!probs || !labels) return E::fail(-1, "a buffer is null");
  entry::Device d;
  if (int rc = E::device(&d)) return rc;
  const int smem_max = d.smem_optin;
  int copies = WARPS;
  while (copies > 1 && smem_bytes(T, copies) > (size_t)smem_max) --copies;
  const size_t smem = smem_bytes(T, copies);
  if (smem > (size_t)smem_max)
    return E::fail(-1, std::to_string(T) + " thresholds need " + std::to_string(smem) + " bytes of shared memory, the "
                           "device has " + std::to_string(smem_max));
  int per = 0;
  if (int rc = E::raise_smem_limit(k_auc_update, smem_max)) return rc;
  if (int rc = E::blocks_per_sm(k_auc_update, THREADS, smem, &per)) return rc;
  const int64_t want = (n + B200_METRICS_MIN_PER_CTA - 1) / B200_METRICS_MIN_PER_CTA;
  const int grid = (int)(want < (int64_t)d.sms * per ? want : (int64_t)d.sms * per);
  k_auc_update<<<grid, THREADS, smem, (cudaStream_t)stream>>>(probs, labels, n, thresholds, T, copies,
                                                              reinterpret_cast<unsigned long long*>(hist),
                                                              reinterpret_cast<unsigned long long*>(invalid));
  return E::launched("k_auc_update", g_launches);
}

}  // extern "C"
