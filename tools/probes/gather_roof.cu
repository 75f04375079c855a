// Bare random-row gather / read-modify-write probes: what the HBM system of this GPU sustains for the ACCESS
// PATTERN of the PS row kernels (one random 32..256 B record per id out of a table far larger than L2), with
// none of the PS logic around it.  The roof the row kernels of csrc/ps_flat.cuh can be held against.
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o tools/probes/gather_roof tools/probes/gather_roof.cu
// Prints one JSON line per variant: algorithmic bytes use SURVEY 8d's formulas (id + row read + row write).
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <numeric>
#include <random>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e)); exit(1); } } while (0)

__device__ __forceinline__ float4 ldg4(const float* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void stg4(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w));
}

// LPR lanes per row, each lane moves one 16 B chunk; U rows in flight per lane group; stride in floats.
template <int LPR, int U, bool WRITE_OUT>
__global__ void __launch_bounds__(256) k_gather(const int64_t* __restrict__ ids, long long n, const float* __restrict__ table,
                                                long long stride, float* __restrict__ out, float* sink) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long item0 = (t / 32) * (32LL * U) + (t & 31);  // warp handles 32*U consecutive items
  float4 x[U];
  long long it[U];
#pragma unroll
  for (int k = 0; k < U; ++k) {
    it[k] = item0 + 32LL * k;
    const long long row = it[k] / LPR;
    x[k] = make_float4(0, 0, 0, 0);
    if (row < n) {
      const long long id = ids[row];
      x[k] = ldg4(table + id * stride + 4 * (it[k] % LPR));
    }
  }
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < U; ++k) {
    if (it[k] / LPR < n) {
      if (WRITE_OUT) stg4(out + it[k] * 4, x[k]);
      else acc += x[k].x + x[k].y + x[k].z + x[k].w;
    }
  }
  if (!WRITE_OUT && acc == 123.456f) *sink = acc;
}

// read-modify-write of a whole record of REC 16 B chunks per id (the push pattern: param + slots), one lane
// per chunk, plus a gradient read of GR chunks per row.
template <int REC, int U>
__global__ void __launch_bounds__(256) k_rmw(const int64_t* __restrict__ ids, long long n, float* __restrict__ table,
                                             long long stride, const float* __restrict__ grad, int gchunks) {
  const long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long item0 = (t / 32) * (32LL * U) + (t & 31);
  float4 x[U], g[U];
  float* p[U];
#pragma unroll
  for (int k = 0; k < U; ++k) {
    const long long it = item0 + 32LL * k, row = it / REC;
    p[k] = nullptr;
    if (row < n) {
      const int c = (int)(it % REC);
      const long long id = ids[row];
      p[k] = table + id * stride + 4 * c;
      x[k] = ldg4(p[k]);
      g[k] = ldg4(grad + (row * gchunks + c % gchunks) * 4);
    }
  }
#pragma unroll
  for (int k = 0; k < U; ++k)
    if (p[k]) {
      x[k].x = x[k].x * 0.999f + g[k].x; x[k].y = x[k].y * 0.999f + g[k].y;
      x[k].z = x[k].z * 0.999f + g[k].z; x[k].w = x[k].w * 0.999f + g[k].w;
      stg4(p[k], x[k]);
    }
}

__global__ void k_copy(const float4* __restrict__ a, float4* __restrict__ b, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) b[i] = a[i];
}

template <typename F>
static float time_us(F launch, int reps = 20) {
  cudaEvent_t a, b;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
  for (int i = 0; i < 3; ++i) launch();
  CK(cudaDeviceSynchronize());
  CK(cudaEventRecord(a));
  for (int i = 0; i < reps; ++i) launch();
  CK(cudaEventRecord(b));
  CK(cudaEventSynchronize(b));
  float ms; CK(cudaEventElapsedTime(&ms, a, b));
  return ms * 1e3f / reps;
}

int main(int argc, char** argv) {
  const long long n = argc > 1 ? atoll(argv[1]) : 4000000;       // ids per launch
  const long long rows = argc > 2 ? atoll(argv[2]) : 16000000;   // table rows (ids are a random subset)
  double peak = argc > 3 ? atof(argv[3]) : 0.0;  // GB/s; default: the stream copy measured below
  std::vector<int64_t> h(rows);
  std::iota(h.begin(), h.end(), 0);
  std::mt19937_64 rng(7);
  std::shuffle(h.begin(), h.end(), rng);
  int64_t* ids; CK(cudaMalloc(&ids, n * 8));
  CK(cudaMemcpy(ids, h.data(), n * 8, cudaMemcpyHostToDevice));
  float *out, *grad, *sink;
  CK(cudaMalloc(&out, n * 256)); CK(cudaMalloc(&grad, n * 256)); CK(cudaMalloc(&sink, 4));
  CK(cudaMemset(grad, 0, n * 256));
  // streaming copy roof of this GPU
  {
    const long long m = 1LL << 26;  // 1 GiB each way
    int dev = 0, n_sm = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&n_sm, cudaDevAttrMultiProcessorCount, dev));
    float4 *a, *b; CK(cudaMalloc(&a, m * 16)); CK(cudaMalloc(&b, m * 16)); CK(cudaMemset(a, 0, m * 16));
    const float us = time_us([&] { k_copy<<<n_sm * 16, 256>>>(a, b, m); }, 5);
    printf("{\"probe\": \"stream_copy\", \"bytes\": %lld, \"us\": %.1f, \"gbs\": %.0f}\n", 2 * m * 16, us, 2.0 * m * 16 / us / 1e3);
    if (peak <= 0.0) peak = 2.0 * m * 16 / us / 1e3;
    CK(cudaFree(a)); CK(cudaFree(b));
  }
  struct Cfg { const char* name; int dim; int slots; };
  auto report = [&](const char* name, int dim, long long stride_f, const char* what, double alg_bytes, float us) {
    printf("{\"probe\": \"%s\", \"dim\": %d, \"record_bytes\": %lld, \"ids\": %lld, \"table_mb\": %.0f, \"what\": \"%s\", \"us\": %.1f, "
           "\"alg_gbs\": %.0f, \"frac_of_copy_peak\": %.3f, \"rows_per_us\": %.0f}\n",
           name, dim, stride_f * 4, n, rows * stride_f * 4 / 1e6, what, us, alg_bytes / us / 1e3, alg_bytes / us / 1e3 / peak, n / us);
    fflush(stdout);
  };
#define GATHER(LPR, U, W, name, dim, stride_f)                                                              \
  {                                                                                                          \
    const long long items = n * LPR, threads = (items + U - 1) / U;                                          \
    const unsigned blocks = (unsigned)((threads + 255) / 256);                                               \
    const float us = time_us([&] { k_gather<LPR, U, W><<<blocks, 256>>>(ids, n, table, stride_f, out, sink); }); \
    report(name, dim, stride_f, W ? "id + row read + row write" : "id + row read (no store)",               \
           (double)n * (8 + 4.0 * dim * (W ? 2 : 1)), us);                                                   \
  }
  {  // dim 8, Adam record 96 B (param at the front): the pull of the benchmark's deep tables
    const long long stride_f = 24;
    float* table; CK(cudaMalloc(&table, rows * stride_f * 4)); CK(cudaMemset(table, 0, rows * stride_f * 4));
    GATHER(2, 1, true, "gather_u1", 8, stride_f)
    GATHER(2, 2, true, "gather_u2", 8, stride_f)
    GATHER(2, 4, true, "gather_u4", 8, stride_f)
    GATHER(2, 8, true, "gather_u8", 8, stride_f)
    GATHER(2, 4, false, "gather_u4_readonly", 8, stride_f)
    GATHER(2, 8, false, "gather_u8_readonly", 8, stride_f)
    // push pattern: RMW of the 96 B record (6 chunks) + 32 B gradient
    for (int u = 1; u <= 4; u *= 2) {
      const long long items = n * 6, threads = (items + u - 1) / u;
      const unsigned blocks = (unsigned)((threads + 255) / 256);
      float us;
      if (u == 1) us = time_us([&] { k_rmw<6, 1><<<blocks, 256>>>(ids, n, table, stride_f, grad, 2); });
      else if (u == 2) us = time_us([&] { k_rmw<6, 2><<<blocks, 256>>>(ids, n, table, stride_f, grad, 2); });
      else us = time_us([&] { k_rmw<6, 4><<<blocks, 256>>>(ids, n, table, stride_f, grad, 2); });
      char nm[32]; snprintf(nm, sizeof nm, "rmw_u%d", u);
      report(nm, 8, stride_f, "id + grad + record read + record write (Adam push pattern)", (double)n * (8 + 32 + 192), us);
    }
    CK(cudaFree(table));
  }
  {  // dim 8 packed rows (32 B stride): the same gather without the slot bytes between rows
    const long long stride_f = 8;
    float* table; CK(cudaMalloc(&table, rows * stride_f * 4)); CK(cudaMemset(table, 0, rows * stride_f * 4));
    GATHER(2, 4, true, "gather_u4_packed32", 8, stride_f)
    CK(cudaFree(table));
  }
  {  // dim 1, 16 B record
    const long long stride_f = 4;
    float* table; CK(cudaMalloc(&table, rows * stride_f * 4)); CK(cudaMemset(table, 0, rows * stride_f * 4));
    {
      const long long threads = (n + 3) / 4;
      const unsigned blocks = (unsigned)((threads + 255) / 256);
      const float us = time_us([&] { k_gather<1, 4, true><<<blocks, 256>>>(ids, n, table, stride_f, out, sink); });
      report("gather16_u4", 1, stride_f, "id + 16 B record read + 16 B write (dim-1 record [p,m,v,-])", (double)n * (8 + 4 + 4), us);
    }
    CK(cudaFree(table));
  }
  {  // dim 64, Adam record 768 B: 16 lanes per row
    const long long stride_f = 192, r64 = rows / 4;
    std::vector<int64_t> h2(r64);
    std::iota(h2.begin(), h2.end(), 0);
    std::shuffle(h2.begin(), h2.end(), rng);
    const long long n64 = std::min(n, r64);
    CK(cudaMemcpy(ids, h2.data(), n64 * 8, cudaMemcpyHostToDevice));
    float* table; CK(cudaMalloc(&table, r64 * stride_f * 4)); CK(cudaMemset(table, 0, r64 * stride_f * 4));
    const long long nsave = n;
    {
      const long long n = std::min(nsave, (long long)1000000);
      auto rep64 = [&](const char* name, float us, bool w) {
        printf("{\"probe\": \"%s\", \"dim\": 64, \"record_bytes\": 768, \"ids\": %lld, \"table_mb\": %.0f, \"us\": %.1f, \"alg_gbs\": %.0f, "
               "\"frac_of_copy_peak\": %.3f}\n", name, n, r64 * stride_f * 4 / 1e6, us, n * (8 + 256.0 * (w ? 2 : 1)) / us / 1e3,
               n * (8 + 256.0 * (w ? 2 : 1)) / us / 1e3 / peak);
      };
      {
        const long long threads = n * 16;
        const unsigned blocks = (unsigned)((threads + 255) / 256);
        rep64("gather256_u1", time_us([&] { k_gather<16, 1, true><<<blocks, 256>>>(ids, n, table, stride_f, out, sink); }), true);
      }
      {
        const long long threads = n * 16 / 4;
        const unsigned blocks = (unsigned)((threads + 255) / 256);
        rep64("gather256_u4", time_us([&] { k_gather<16, 4, true><<<blocks, 256>>>(ids, n, table, stride_f, out, sink); }), true);
        rep64("gather256_u4_readonly", time_us([&] { k_gather<16, 4, false><<<blocks, 256>>>(ids, n, table, stride_f, out, sink); }), false);
      }
    }
    CK(cudaFree(table));
  }
  return 0;
}
