// What every C-ABI entry point of the library shares: the host side of a launch (the thread's last error message
// per include/ header, launch counters, the current device and its limits, resident blocks per SM, a kernel's
// dynamic shared-memory limit, the check after a launch) and the device side of a deterministic last-CTA
// reduction.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <cstddef>
#include <map>
#include <mutex>
#include <string>
#include <tuple>

namespace entry {

// One tag per C-ABI header; each header has one error message per host thread (its *_last_error).
struct Ps {};        // b200ps.h
struct DeepFm {};    // b200_deepfm.h: the fused, tile, mma, DCN and xDeepFM towers
struct Features {};  // b200_features.h
struct Census {};    // b200_census.h
struct CensusSqlflow {};  // b200_census_sqlflow.h
struct Frappe {};    // b200_frappe.h
struct FcDnn {};     // b200_fc_dnn.h
struct DeepctrWdl {};  // b200_deepctr_wdl.h
struct DeepctrDeepfm {};  // b200_deepctr_deepfm.h
struct Metrics {};   // b200_metrics.h

// What an exported *_launch_count reads; entry points of several host threads add to it.
using LaunchCount = std::atomic<long long>;

struct Device {
  int id;
  int sms;         // multiprocessors
  int smem_optin;  // opt-in shared memory per block (bytes)
};

namespace detail {

constexpr int kMaxCached = 64;  // devices whose limits are cached

inline cudaError_t current_device(Device* d) {
  static std::atomic<int> sms[kMaxCached], optin[kMaxCached];
  cudaError_t e = cudaGetDevice(&d->id);
  if (e != cudaSuccess) return e;
  const bool cached = d->id < kMaxCached;
  if (cached && (d->sms = sms[d->id].load()) > 0) {
    d->smem_optin = optin[d->id].load();
    return cudaSuccess;
  }
  if ((e = cudaDeviceGetAttribute(&d->sms, cudaDevAttrMultiProcessorCount, d->id)) != cudaSuccess ||
      (e = cudaDeviceGetAttribute(&d->smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, d->id)) != cudaSuccess)
    return e;
  if (cached) {
    optin[d->id].store(d->smem_optin);  // before sms: a reader that sees sms sees optin
    sms[d->id].store(d->sms);
  }
  return cudaSuccess;
}

// The occupancy and shared-memory-limit caches: driver calls, made once per key under one lock.
inline std::mutex& cache_mutex() {
  static std::mutex mu;
  return mu;
}

inline cudaError_t blocks_per_sm(const void* kernel, int threads, size_t smem, int* out) {
  static std::map<std::tuple<const void*, int, int, size_t>, int> cache;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const auto key = std::make_tuple(kernel, dev, threads, smem);
  std::lock_guard<std::mutex> lk(cache_mutex());
  auto it = cache.find(key);
  if (it == cache.end()) {
    int n = 0;
    if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem)) != cudaSuccess) return e;
    it = cache.emplace(key, n < 1 ? 1 : n).first;
  }
  *out = it->second;
  return cudaSuccess;
}

inline cudaError_t raise_smem_limit(const void* kernel, size_t bytes) {
  static std::map<std::pair<const void*, int>, size_t> set;  // the limit set per (kernel, device)
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lk(cache_mutex());
  size_t& cur = set[std::make_pair(kernel, dev)];
  if (cur >= bytes) return cudaSuccess;
  if ((e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)) != cudaSuccess)
    return e;
  cur = bytes;
  return cudaSuccess;
}

}  // namespace detail

// The host side of the entry points of the header tagged Abi.  Each returns 0, or an error code with the message
// in the calling thread's slot of the header: -1 for a refusal (fail), -2 for a CUDA error.
template <class Abi>
struct Entry {
  static std::string& last_error() {
    static thread_local std::string msg;
    return msg;
  }
  static int fail(int code, const std::string& msg) {
    last_error() = msg;
    return code;
  }
  static int cuda_fail(const char* what, cudaError_t e) {
    return fail(-2, std::string(what) + ": " + cudaGetErrorString(e));
  }

  // The current device and its limits (cached per device).
  static int device(Device* d) {
    const cudaError_t e = detail::current_device(d);
    return e == cudaSuccess ? 0 : cuda_fail("current device", e);
  }
  // Resident blocks per SM (at least 1) of `kernel` at `threads` and `smem` bytes of dynamic shared memory on the
  // current device (cached per kernel, device, threads and smem).
  template <class K>
  static int blocks_per_sm(K* kernel, int threads, size_t smem, int* out) {
    const cudaError_t e = detail::blocks_per_sm((const void*)kernel, threads, smem, out);
    return e == cudaSuccess ? 0 : cuda_fail("cudaOccupancyMaxActiveBlocksPerMultiprocessor", e);
  }
  // Raise the dynamic shared-memory limit of `kernel` on the current device to at least `bytes` (a driver call
  // the first time a kernel and device need more).
  template <class K>
  static int raise_smem_limit(K* kernel, size_t bytes) {
    const cudaError_t e = detail::raise_smem_limit((const void*)kernel, bytes);
    return e == cudaSuccess ? 0 : cuda_fail("cudaFuncSetAttribute", e);
  }
  // After launching `kernel`: 0 with `n` added to `launches`, or -2 and "<kernel>: <error>".
  static int launched(const char* kernel, LaunchCount& launches, long long n = 1) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return cuda_fail(kernel, e);
    launches.fetch_add(n);
    return 0;
  }
};

// ---- the last-CTA reduction of a deterministic kernel
// Its workspace is an arrival counter, zero between launches, in a 64-byte header, then one partial of Q floats
// per CTA.  Every CTA writes its partial; the last to arrive adds the partials in CTA order, so the sums do not
// depend on which CTA finishes when, and zeroes the counter.

constexpr size_t kPartialsHeader = 64;

inline size_t partials_bytes(int grid, int Q) { return kPartialsHeader + (size_t)grid * Q * sizeof(float); }

__device__ __forceinline__ unsigned* arrival_counter(void* workspace) { return reinterpret_cast<unsigned*>(workspace); }
__device__ __forceinline__ float* partials(void* workspace) {
  return reinterpret_cast<float*>(reinterpret_cast<char*>(workspace) + kPartialsHeader);
}

// Every thread of every CTA calls it after its writes of the CTA's result.  True in every thread of the last CTA
// to arrive, whose loads through L2 (__ldcg) then see every CTA's result.  `last` is a shared int of the caller's.
__device__ __forceinline__ bool last_to_arrive(unsigned* counter, int& last) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return false;
  __threadfence();
  return true;
}

// In the last CTA (THREADS threads): entry i of the total is the sum of entry i of the Q-float partials in CTA
// order; store(i, total) for each i.
template <int THREADS, class Store>
__device__ __forceinline__ void sum_partials(const float* parts, int Q, Store store) {
  for (int i = threadIdx.x; i < Q; i += THREADS) {
    float s = 0.f;
    for (unsigned c = 0; c < gridDim.x; ++c) s += __ldcg(parts + (size_t)c * Q + i);
    store(i, s);
  }
}

}  // namespace entry
