// Owner-computes exchange for rank-per-GPU groups: the all-to-all-v the reference performs with 2*M
// RPCs per step (python/worker/ps_client.py:105-130 pull, :243-277 push), as NVLink traffic that is
// contiguous in both directions and needs NO memory fences between GPUs.
//
// Scattered 32 B accesses to a peer GPU -- reads AND writes -- run at a small fraction of the link
// rate, bound by sectors per second whatever the request size (tools/mgpu_probe.py measures it);
// coalesced peer traffic runs at the link rate.  So nothing scattered crosses NVLink:
//   pull  k_x_post      requester buckets its unique ids BY OWNER (id % N) into its exchange buffer as
//                       {id, slot} words: block-level histogram in shared memory, one cursor
//                       reservation per (block, owner), the per-owner counts travel with the flag
//         k_x_serve     every OWNER streams ITS bucket of every requester's list over NVLink (coalesced
//                       reads of exactly the ids it owns: an all-to-all-v -- round 1 had every owner read
//                       every whole list, N x the bytes), gathers those rows from its own HBM and writes
//                       {row, slot} to the same index of the requester's response region; it
//                       remembers (id, group) of what it served, in order
//         k_x_unscatter requester copies the rows of each owner's region to bet[slot]
//   push  k_x_send_upd  requester walks each owner's response region again (its order == the owner's
//                       serve order) and writes the matching gradient rows CONTIGUOUSLY into the
//                       owner's inbox: no bucketing, no atomics
//         k_x_apply     the owner applies the fused optimizer to its own shard: entry i of source s
//                       updates the row it served as entry i (with the source's lr / Adam alpha); one
//                       launch per source in rank order, so a row several ranks pushed gets every update
// A push therefore rides on the routing of the pull that precedes it (the training step's order).
// An id outside the owner's table is served as a zero row and flagged in the response header word; the
// REQUESTER's k_x_unscatter raises the range error, as the direct pull reports it to its caller.
//
// Cross-GPU synchronisation is flag-in-data (the idea of NCCL's LL protocol): everything a peer
// reads is made of naturally aligned 16-byte (or 8-byte) words whose last lane is the epoch TAG,
// written with one volatile vector store and polled with one volatile vector load, so a word is
// either the stale epoch's or complete -- no ordering between different words is ever needed.
// The first versions used st.release.sys / __threadfence_system(); a MEMBAR.SYS also waits on
// the PCIe side, and with the next batch's H2D copy in flight the step time nearly doubled
// (tools/xchg_dma_probe.py).  All ranks launch the same kernels in the same order (bulk-synchronous
// step); polls time out after ~2 s and raise instead of hanging the GPU.
#pragma once
#include "ps_kernels.cuh"

namespace b200ps_impl {

constexpr int kXIdEntry = 16;  // bytes: {int64 id; int32 slot; int32 tag}
constexpr int kXResp = 64;     // bytes: {d0 d1 d2 tag}{d3 d4 d5 tag}{d6 d7 wide tag}{slot 0 0 tag}
constexpr int kXUpd = 48;      // bytes: {g0 g1 g2 tag}{g3 g4 g5 tag}{g6 g7 gwide tag}
constexpr int kXServed = 16;   // bytes: {int64 id; int32 grp; int32 pad}   (owner-local)

struct XHeader {  // first page of every rank's exchange buffer
  // written by source ranks into the OWNER's header (self-validating words)
  int2 req[kMaxShards];   // [src] {ids published, tag}
  int4 updh[kMaxShards];  // [src] {lr, alpha, l2adj (float bits), tag}
  // written by owner ranks into the REQUESTER's header
  int4 resp[kMaxShards];    // [owner] {rows returned, 1 if an id was outside the table, 0, tag}
  int applied[kMaxShards];  // [owner] tag: that owner has applied my updates
  // local
  int epoch;
  int post_cursor[kMaxShards]; // requester: ids bucketed so far for each owner (this epoch)
  int served_cnt[kMaxShards];  // owner: rows served to each source by the last pull
  unsigned done_blocks;
  unsigned done_src[kMaxShards];
  unsigned range_src[kMaxShards];  // owner: an id of that source's bucket was outside the table (this pull)
};

struct XView {
  char* buf[kMaxShards];  // every rank's exchange buffer (peer-mapped); buf[me] is local
  long long off_ids, off_resp, off_upd, off_served;  // byte offsets of the regions
  long long cap;                                     // entries per (owner, source) lane = G * B
  int n, me, G, B;
};

__device__ __forceinline__ XHeader* xhdr(const XView& x, int r) { return reinterpret_cast<XHeader*>(x.buf[r]); }
// bucket of the ids requester r wants from owner o (cap entries each)
__device__ __forceinline__ char* xids(const XView& x, int r, int o) {
  return x.buf[r] + x.off_ids + ((long long)o * x.cap) * kXIdEntry;
}
__device__ __forceinline__ char* xresp(const XView& x, int requester, int owner) {
  return x.buf[requester] + x.off_resp + ((long long)owner * x.cap) * kXResp;
}
__device__ __forceinline__ char* xupd(const XView& x, int owner, int src) {
  return x.buf[owner] + x.off_upd + ((long long)src * x.cap) * kXUpd;
}
__device__ __forceinline__ char* xserved(const XView& x, int owner, int src) {
  return x.buf[owner] + x.off_served + ((long long)src * x.cap) * kXServed;
}

constexpr unsigned kErrTimeout = 8u;
constexpr long long kXSpins = 1LL << 24;  // ~2 s with the sleep below

// ---- self-validating words: one volatile vector access each (relaxed, system scope) ----
__device__ __forceinline__ void st_word16(void* p, int a, int b, int c, int tag) {
  asm volatile("st.volatile.global.v4.s32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(tag) : "memory");
}
__device__ __forceinline__ int4 ld_word16(const void* p) {
  int4 v;
  asm volatile("ld.volatile.global.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_word8(void* p, int a, int tag) {
  asm volatile("st.volatile.global.v2.s32 [%0], {%1,%2};" ::"l"(p), "r"(a), "r"(tag) : "memory");
}
__device__ __forceinline__ int2 ld_word8(const void* p) {
  int2 v;
  asm volatile("ld.volatile.global.v2.s32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ int ld_word4(const int* p) {
  int v;
  asm volatile("ld.volatile.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

// Poll a 16-byte word until its tag is `tag` (normally the first load succeeds: the writer ran
// a whole kernel earlier).  On timeout the error bit is raised and the stale word returned.
__device__ __forceinline__ int4 poll16(const void* p, int tag, unsigned* err) {
  int4 v = ld_word16(p);
  if (v.w == tag) return v;
  for (long long spins = 0; spins < kXSpins; ++spins) {
    __nanosleep(64);
    v = ld_word16(p);
    if (v.w == tag) return v;
  }
  atomicOr(err, kErrTimeout);
  return v;
}
__device__ __forceinline__ int2 poll8(const void* p, int tag, unsigned* err) {
  int2 v = ld_word8(p);
  if (v.y == tag) return v;
  for (long long spins = 0; spins < kXSpins; ++spins) {
    __nanosleep(64);
    v = ld_word8(p);
    if (v.y == tag) return v;
  }
  atomicOr(err, kErrTimeout);
  return v;
}

// Largest g with prefix[g] <= w (prefix[0] == 0, prefix[G] == total > w).
__device__ __forceinline__ int group_of(const int* prefix, int G, int w) {
  int lo = 0, hi = G;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (prefix[mid] <= w) lo = mid; else hi = mid;
  }
  return lo;
}

// Requester: open a new epoch and publish this step's unique ids, bucketed by owner, as tagged {id, slot}
// words in its own exchange buffer; every owner is told how many of them are its own.
constexpr int kXPostPer = 4;  // ids per thread per block iteration
__global__ void __launch_bounds__(256) k_x_post(XView x, const int64_t* __restrict__ uniq, const int* __restrict__ n_unique) {
  XHeader* h = xhdr(x, x.me);
  __shared__ int s_prefix[kMaxSegs + 1];
  __shared__ int s_u[kMaxSegs];
  __shared__ int s_hist[kMaxShards];           // ids of this chunk per owner
  __shared__ int s_wbase[8][kMaxShards];       // per warp: its offset inside the block's range of that owner
  __shared__ int s_base[kMaxShards];           // the block's reservation in each owner's bucket
  const int epoch = *(volatile int*)&h->epoch + 1;  // every block reads it before the last one bumps it
  if (threadIdx.x < x.G) {
    const int u = n_unique[threadIdx.x];
    s_u[threadIdx.x] = u < x.B ? u : x.B;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < x.G; ++g) {
      s_prefix[g] = acc;
      acc += s_u[g];
    }
    s_prefix[x.G] = acc;
  }
  __syncthreads();
  const int total = s_prefix[x.G];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const bool pow2 = (x.n & (x.n - 1)) == 0;
  constexpr int kChunk = 256 * kXPostPer;
  for (int chunk = blockIdx.x * kChunk; chunk < total; chunk += gridDim.x * kChunk) {
    long long id[kXPostPer];
    int slot[kXPostPer], own[kXPostPer], rk[kXPostPer];
    if (threadIdx.x < x.n) s_hist[threadIdx.x] = 0;
#pragma unroll
    for (int j = 0; j < kXPostPer; ++j) {
      const int w = chunk + j * 256 + threadIdx.x;
      own[j] = -1;
      slot[j] = 0;
      id[j] = 0;
      if (w < total) {
        const int g = group_of(s_prefix, x.G, w);
        slot[j] = g * x.B + (w - s_prefix[g]);
        id[j] = uniq[slot[j]];
        own[j] = pow2 ? (int)(id[j] & (x.n - 1)) : (int)(((id[j] % x.n) + x.n) % x.n);
      }
    }
    __syncthreads();
    // per warp and owner: how many ids, and each lane's rank among them (ballots, no atomics).
    // lane o (< n) keeps the warp's running count of owner o over the rounds.
    int cnt_prev = 0;
#pragma unroll
    for (int j = 0; j < kXPostPer; ++j) {
      rk[j] = 0;
      int addv = 0;
      for (int o = 0; o < x.n; ++o) {
        const unsigned m = __ballot_sync(0xffffffffu, own[j] == o);
        const int before = __shfl_sync(0xffffffffu, cnt_prev, o);
        if (own[j] == o) rk[j] = before + __popc(m & ((1u << lane) - 1));
        if (lane == o) addv = __popc(m);
      }
      cnt_prev += addv;
    }
    if (lane < x.n) s_wbase[wid][lane] = atomicAdd(&s_hist[lane], cnt_prev);  // warp's offset inside the block's range
    __syncthreads();
    if (threadIdx.x < x.n) s_base[threadIdx.x] = s_hist[threadIdx.x] ? atomicAdd(&h->post_cursor[threadIdx.x], s_hist[threadIdx.x]) : 0;
    __syncthreads();
#pragma unroll
    for (int j = 0; j < kXPostPer; ++j) {
      if (own[j] < 0) continue;
      const int at = s_base[own[j]] + s_wbase[wid][own[j]] + rk[j];
      st_word16(xids(x, x.me, own[j]) + (long long)at * kXIdEntry, (int)(id[j] & 0xffffffffLL), (int)(id[j] >> 32), slot[j], epoch);
    }
    __syncthreads();  // s_hist / s_wbase / s_base are rewritten by the next chunk
  }
  __shared__ bool last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&h->done_blocks, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (threadIdx.x < x.n) {  // tell every owner how many of my ids are its own
    const int cnt = *(volatile int*)&h->post_cursor[threadIdx.x];
    st_word8(&xhdr(x, threadIdx.x)->req[x.me], cnt, epoch);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    h->epoch = epoch;
    h->done_blocks = 0;
  }
  if (threadIdx.x < kMaxShards) {
    h->post_cursor[threadIdx.x] = 0;
    h->done_src[threadIdx.x] = 0;
  }
}

__device__ __forceinline__ long long id_of(int lo, int hi) {
  return (long long)(((unsigned long long)(unsigned)hi << 32) | (unsigned)lo);
}

// The owner's table constants, resolved once on the host by b200ps_xchg_create and passed as a
// __grid_constant__: base pointer, created-row bitmap, stride and row count of each of the G (deep, wide)
// pairs on MY shard, so no table directory is read between an id and its record.  Every pass of a data
// kernel is a chain of two to four dependent round trips (NVLink word -> HBM record -> NVLink store), so
// each 4-lane group keeps XU entries in flight: all words of an iteration are loaded before the first
// one is used, then all records, then the stores.
constexpr int kXMaxG = kMaxSegs / 2;
struct XTabs {
  float* deep[kXMaxG];
  float* wide[kXMaxG];
  uint32_t* deep_pres[kXMaxG];
  uint32_t* wide_pres[kXMaxG];
  long long deep_rows[kXMaxG], wide_rows[kXMaxG];  // rows on my shard
  int deep_stride[kXMaxG], wide_stride[kXMaxG];    // floats
  int deep_soff[kMaxSlots + 1], wide_soff[kMaxSlots + 1];
  int shard_shift;  // log2(n) or -1
};

__device__ __forceinline__ long long xslot_of(const XView& x, const XTabs& t, long long id) {
  return t.shard_shift >= 0 ? id >> t.shard_shift : id / x.n;
}

// Owner: stream MY bucket of source blockIdx.y's id list, gather the rows, return them at the same index.
template <int XU>
__global__ void __launch_bounds__(256) k_x_serve(const __grid_constant__ XView x, const __grid_constant__ XTabs t, unsigned* err) {
  const int src = blockIdx.y;
  XHeader* h = xhdr(x, x.me);
  __shared__ int s_epoch, s_total;
  if (threadIdx.x == 0) {
    s_epoch = h->epoch;
    s_total = poll8(&h->req[src], s_epoch, err).x;
  }
  __syncthreads();
  const int epoch = s_epoch, total = s_total;
  const char* ids = xids(x, src, x.me);
  char* resp = xresp(x, src, x.me);
  char* served = xserved(x, x.me, src);
  const int lane = threadIdx.x & 31, lane4 = threadIdx.x & 3;
  const unsigned gm = 0xfu << (lane & 28);
  const long long stride = (long long)gridDim.x * blockDim.x / 4;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 4; i0 < total; i0 += stride * XU) {
    int4 e[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {  // all remote id words of this iteration
      const long long i = i0 + k * stride;
      e[k] = make_int4(0, 0, 0, epoch);
      if (lane4 == 0 && i < total) e[k] = ld_word16(ids + i * kXIdEntry);
    }
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      if (lane4 == 0 && i < total && e[k].w != epoch) e[k] = poll16(ids + i * kXIdEntry, epoch, err);
      e[k].x = __shfl_sync(gm, e[k].x, 0, 4);
      e[k].y = __shfl_sync(gm, e[k].y, 0, 4);
      e[k].z = __shfl_sync(gm, e[k].z, 0, 4);
    }
    float4 v[XU];
    uint32_t* pres[XU];
    uint32_t word[XU], bit[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {  // all records (and their created-row bitmap words)
      const long long i = i0 + k * stride;
      v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      pres[k] = nullptr;
      word[k] = 0xffffffffu;
      bit[k] = 0;
      if (i >= total) continue;
      const long long id = id_of(e[k].x, e[k].y);
      const int g = e[k].z / x.B;
      const long long sl = xslot_of(x, t, id);
      if (lane4 < 2) {
        const bool ok = id >= 0 && sl < t.deep_rows[g];
        if (ok) {
          v[k] = ld_f4(t.deep[g] + sl * t.deep_stride[g] + 4 * lane4);
          if (lane4 == 0 && t.deep_pres[g]) { pres[k] = t.deep_pres[g] + (sl >> 5); bit[k] = 1u << (sl & 31); }
        } else if (lane4 == 0) {
          atomicOr(&h->range_src[src], 1u);  // the requester reports it (k_x_unscatter), not this shard
        }
      } else if (lane4 == 2) {
        if (id >= 0 && sl < t.wide_rows[g]) {
          v[k].x = *(t.wide[g] + sl * t.wide_stride[g]);
          if (t.wide_pres[g]) { pres[k] = t.wide_pres[g] + (sl >> 5); bit[k] = 1u << (sl & 31); }
        }
      }
      if (pres[k]) word[k] = *(volatile uint32_t*)pres[k];
    }
#pragma unroll
    for (int k = 0; k < XU; ++k) {  // responses: entry i answers id i
      const long long i = i0 + k * stride;
      if (i >= total) continue;
      const float d3 = __shfl_sync(gm, v[k].w, 0, 4), d6 = __shfl_sync(gm, v[k].z, 1, 4), d7 = __shfl_sync(gm, v[k].w, 1, 4);
      char* out = resp + i * kXResp + 16 * lane4;
      if (lane4 == 0) st_word16(out, __float_as_int(v[k].x), __float_as_int(v[k].y), __float_as_int(v[k].z), epoch);
      else if (lane4 == 1) st_word16(out, __float_as_int(d3), __float_as_int(v[k].x), __float_as_int(v[k].y), epoch);
      else if (lane4 == 2) st_word16(out, __float_as_int(d6), __float_as_int(d7), __float_as_int(v[k].x), epoch);
      else {
        st_word16(out, e[k].z, 0, 0, epoch);
        *reinterpret_cast<int4*>(served + i * kXServed) = make_int4(e[k].x, e[k].y, e[k].z / x.B, 0);
      }
    }
#pragma unroll
    for (int k = 0; k < XU; ++k)
      if (pres[k] && !(word[k] & bit[k])) atomicOr(pres[k], bit[k]);
  }
  __shared__ bool last;
  __threadfence();  // served records: local, read by this GPU's later kernels
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&h->done_src[src], 1u) == gridDim.x - 1;
  __syncthreads();
  if (last && threadIdx.x == 0) {
    h->served_cnt[src] = total;
    const unsigned bad = atomicExch(&h->range_src[src], 0u);  // every block's flag: they fenced before done_src
    st_word16(&xhdr(x, src)->resp[x.me], total, (int)bad, 0, epoch);
    h->done_src[src] = 0;
  }
}

// Requester: rows of owner blockIdx.y land in my response region -> bet_d / bet_w.
template <int XU>
__global__ void __launch_bounds__(256) k_x_unscatter(const __grid_constant__ XView x, unsigned* err, float* bet_d, float* bet_w) {
  const int owner = blockIdx.y;
  XHeader* h = xhdr(x, x.me);
  __shared__ int s_cnt, s_epoch;
  if (threadIdx.x == 0) {
    s_epoch = h->epoch;
    const int4 r = poll16(&h->resp[owner], s_epoch, err);
    s_cnt = r.x;
    if (r.y && blockIdx.x == 0) atomicOr(err, kErrRange);  // an id I asked that owner for is outside the table
  }
  __syncthreads();
  const int cnt = s_cnt, epoch = s_epoch;
  const char* resp = xresp(x, x.me, owner);
  const int lane = threadIdx.x & 31, lane4 = threadIdx.x & 3;
  const unsigned gm = 0xfu << (lane & 28);
  const long long stride = (long long)gridDim.x * blockDim.x / 4;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 4; i0 < cnt; i0 += stride * XU) {
    int4 p[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      p[k] = make_int4(0, 0, 0, epoch);
      if (i < cnt) p[k] = ld_word16(resp + i * kXResp + 16 * lane4);
    }
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      if (i < cnt && p[k].w != epoch) p[k] = poll16(resp + i * kXResp + 16 * lane4, epoch, err);
      const int slot = __shfl_sync(gm, p[k].x, 3, 4);
      if (i >= cnt) continue;
      float* row = bet_d + (long long)slot * 8;
      if (lane4 == 0) {
        row[0] = __int_as_float(p[k].x); row[1] = __int_as_float(p[k].y); row[2] = __int_as_float(p[k].z);
      } else if (lane4 == 1) {
        row[3] = __int_as_float(p[k].x); row[4] = __int_as_float(p[k].y); row[5] = __int_as_float(p[k].z);
      } else if (lane4 == 2) {
        row[6] = __int_as_float(p[k].x); row[7] = __int_as_float(p[k].y);
        bet_w[slot] = __int_as_float(p[k].z);
      }
    }
  }
}

// Requester: gradient rows to owner blockIdx.y, in the order that owner served my rows.
template <int XU>
__global__ void __launch_bounds__(256) k_x_send_upd(const __grid_constant__ XView x, const PushRt* rt, const float* __restrict__ gsum_d,
                                                    const float* __restrict__ gsum_w) {
  const int owner = blockIdx.y;
  XHeader* h = xhdr(x, x.me);
  const int epoch = h->epoch;
  const int cnt = ld_word16(&h->resp[owner]).x;  // validated by this step's unscatter
  const char* resp = xresp(x, x.me, owner);
  char* upd = xupd(x, owner, x.me);  // remote, contiguous
  const int lane = threadIdx.x & 31, lane4 = threadIdx.x & 3;
  const unsigned gm = 0xfu << (lane & 28);
  if (blockIdx.x == 0 && threadIdx.x == 0)  // this push's lr / Adam alpha / l2 for that shard (k_push_begin; Nadam: nadam_coefs)
    st_word16(&xhdr(x, owner)->updh[x.me], __float_as_int(rt->lr[owner]), __float_as_int(rt->alpha[owner]),
              __float_as_int(rt->l2adj[owner]), epoch);
  const long long stride = (long long)gridDim.x * blockDim.x / 4;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 4; i0 < cnt; i0 += stride * XU) {
    int slot[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      slot[k] = 0;
      if (i < cnt) slot[k] = ld_word16(resp + i * kXResp + 48).x;
    }
    float4 v[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (i >= cnt) continue;
      if (lane4 < 2) v[k] = *reinterpret_cast<const float4*>(gsum_d + (long long)slot[k] * 8 + 4 * lane4);
      else if (lane4 == 2) v[k].x = gsum_w[slot[k]];
    }
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      if (i >= cnt) continue;
      const float g3 = __shfl_sync(gm, v[k].w, 0, 4), g6 = __shfl_sync(gm, v[k].z, 1, 4), g7 = __shfl_sync(gm, v[k].w, 1, 4);
      char* out = upd + i * kXUpd + 16 * lane4;
      if (lane4 == 0) st_word16(out, __float_as_int(v[k].x), __float_as_int(v[k].y), __float_as_int(v[k].z), epoch);
      else if (lane4 == 1) st_word16(out, __float_as_int(g3), __float_as_int(v[k].x), __float_as_int(v[k].y), epoch);
      else if (lane4 == 2) st_word16(out, __float_as_int(g6), __float_as_int(g7), __float_as_int(v[k].x), epoch);
    }
  }
}

// Owner: apply the updates of source `src` to the rows served to it (its own ApplyGradients:
// lr / Adam alpha were fixed by the source's push_begin on this shard).  One launch per source, in rank
// order: two sources may update the same row in one step, and each launch reads what the one before it wrote,
// so every source's update lands, as if the ranks had pushed one after the other.
template <int OPT, int XU>
__global__ void __launch_bounds__(256) k_x_apply(const __grid_constant__ XView x, const __grid_constant__ XTabs t, unsigned* err,
                                                 const OptParams o, const int src) {
  constexpr int S = opt_slots(OPT);
  XHeader* h = xhdr(x, x.me);
  __shared__ int s_epoch, s_cnt;
  __shared__ float s_lr, s_alpha, s_l2;
  if (threadIdx.x == 0) {
    s_epoch = h->epoch;
    const int4 hd = poll16(&h->updh[src], s_epoch, err);
    s_cnt = h->served_cnt[src];
    s_lr = __int_as_float(hd.x);
    s_alpha = __int_as_float(hd.y);
    s_l2 = __int_as_float(hd.z);
  }
  __syncthreads();
  const int cnt = s_cnt, epoch = s_epoch;
  const float lr = s_lr, alpha = s_alpha, l2adj = s_l2;
  const char* upd = xupd(x, x.me, src);
  const char* served = xserved(x, x.me, src);
  const int lane = threadIdx.x & 31, lane4 = threadIdx.x & 3;  // deep lo, deep hi, wide, idle
  const unsigned gm = 0xfu << (lane & 28);
  const long long stride = (long long)gridDim.x * blockDim.x / 4;
  for (long long i0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 4; i0 < cnt; i0 += stride * XU) {
    int4 e[XU], p[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {  // what I served as entry i (local) and its update words (inbox, written by the peer)
      const long long i = i0 + k * stride;
      e[k] = make_int4(0, 0, 0, 0);
      p[k] = make_int4(0, 0, 0, epoch);
      if (i >= cnt) continue;
      e[k] = *reinterpret_cast<const int4*>(served + i * kXServed);
      if (lane4 < 3) p[k] = ld_word16(upd + i * kXUpd + 16 * lane4);
    }
    float* rec[XU];
    float4 pr[XU], s0[XU], s1[XU], s2[XU], g[XU];
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      const long long i = i0 + k * stride;
      rec[k] = nullptr;
      if (i < cnt && lane4 < 3 && p[k].w != epoch) p[k] = poll16(upd + i * kXUpd + 16 * lane4, epoch, err);
      // words {g0 g1 g2}{g3 g4 g5}{g6 g7 gw} -> lane 0: g0..g3, lane 1: g4..g7, lane 2: gw
      const int q1x = __shfl_sync(gm, p[k].x, 1, 4), q2x = __shfl_sync(gm, p[k].x, 2, 4), q2y = __shfl_sync(gm, p[k].y, 2, 4);
      if (i >= cnt) continue;
      const long long id = id_of(e[k].x, e[k].y);
      const int gi = e[k].z;
      const long long sl = xslot_of(x, t, id);
      if (lane4 < 2) {
        if (!(id >= 0 && sl < t.deep_rows[gi])) continue;  // already reported by the serving pass
        g[k] = lane4 == 0 ? make_float4(__int_as_float(p[k].x), __int_as_float(p[k].y), __int_as_float(p[k].z), __int_as_float(q1x))
                          : make_float4(__int_as_float(p[k].y), __int_as_float(p[k].z), __int_as_float(q2x), __int_as_float(q2y));
        rec[k] = t.deep[gi] + sl * t.deep_stride[gi] + 4 * lane4;
        pr[k] = ld_f4(rec[k]);
        if (S > 0) s0[k] = ld_f4(rec[k] + t.deep_soff[1]);
        if (S > 1) s1[k] = ld_f4(rec[k] + t.deep_soff[2]);
        if (S > 2) s2[k] = ld_f4(rec[k] + t.deep_soff[3]);
      } else if (lane4 == 2) {
        if (!(id >= 0 && sl < t.wide_rows[gi])) continue;
        g[k].x = __int_as_float(p[k].z);
        rec[k] = t.wide[gi] + sl * t.wide_stride[gi];
        pr[k].x = *rec[k];
        if (S > 0) s0[k].x = rec[k][t.wide_soff[1]];
        if (S > 1) s1[k].x = rec[k][t.wide_soff[2]];
        if (S > 2) s2[k].x = rec[k][t.wide_soff[3]];
      }
    }
#pragma unroll
    for (int k = 0; k < XU; ++k) {
      if (rec[k] == nullptr) continue;
      if (lane4 < 2) {
        float* gf = reinterpret_cast<float*>(&g[k]);
        float* pf = reinterpret_cast<float*>(&pr[k]);
        float* af = reinterpret_cast<float*>(&s0[k]);
        float* bf = reinterpret_cast<float*>(&s1[k]);
        float* cf = reinterpret_cast<float*>(&s2[k]);
#pragma unroll
        for (int c = 0; c < 4; ++c) opt_update<OPT>(gf[c], pf[c], af[c], bf[c], cf[c], lr, alpha, l2adj, o);
        st_f4(rec[k], pr[k]);
        if (S > 0) st_f4(rec[k] + t.deep_soff[1], s0[k]);
        if (S > 1) st_f4(rec[k] + t.deep_soff[2], s1[k]);
        if (S > 2) st_f4(rec[k] + t.deep_soff[3], s2[k]);
      } else {
        opt_update<OPT>(g[k].x, pr[k].x, s0[k].x, s1[k].x, s2[k].x, lr, alpha, l2adj, o);
        *rec[k] = pr[k].x;
        if (S > 0) rec[k][t.wide_soff[1]] = s0[k].x;
        if (S > 1) rec[k][t.wide_soff[2]] = s1[k].x;
        if (S > 2) rec[k][t.wide_soff[3]] = s2[k].x;
      }
    }
  }
  __shared__ bool last;
  __threadfence();  // rows are local: this GPU's later kernels (its next serve) read them in stream order
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(&h->done_src[src], 1u) == gridDim.x - 1;
  __syncthreads();
  if (last && threadIdx.x == 0) {
    asm volatile("st.volatile.global.s32 [%0], %1;" ::"l"(&xhdr(x, src)->applied[x.me]), "r"(epoch) : "memory");
    h->done_src[src] = 0;
  }
}

// Requester: all owners have applied my updates (push_end bumps the versions after this).
__global__ void k_x_wait_applied(XView x, unsigned* err) {
  XHeader* h = xhdr(x, x.me);
  if (threadIdx.x >= x.n) return;
  const int epoch = h->epoch;
  for (long long spins = 0; spins < kXSpins; ++spins) {
    if (ld_word4(&h->applied[threadIdx.x]) >= epoch) return;
    __nanosleep(64);
  }
  atomicOr(err, kErrTimeout);
}

}  // namespace b200ps_impl
