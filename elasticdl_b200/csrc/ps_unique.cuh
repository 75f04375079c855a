// unique (tf.unique, first-occurrence order + inverse index) over T equal-length id segments as ONE
// persistent kernel (round 1: seven launches).
//
//   phase 0  (only when something must be cleared) hash keys / position arrays
//   phase A  insert: position array entry of every id <- min(position); all id loads, then all probes,
//            then the atomics; lanes of a warp that would write the same entry elect one writer
//   ---- grid barrier ----
//   phase B  per tile (256 x PPT positions, coalesced): first-occurrence flags, ballot ranks, decoupled look-back over
//            the tile aggregates of the segment (single pass: no scan kernel), global ranks,
//            unique ids written in rank order, n_unique by the last tile of each segment
//   ---- grid barrier ----
//   phase C  inverse index: inv[i] = rank of the first occurrence of ids[i]
//
// The grid is sized to be co-resident (occupancy x #SM, capped) so the hand-rolled barrier cannot
// deadlock: blocks only ever wait for blocks of this same launch, all of which are (or will become)
// resident because nothing resident waits on anything outside the launch.  Every spin has a bound
// and raises the error word instead of hanging the GPU.  ids may be int64 or int32 (narrow id
// transport: the widening happens at the first read); outputs are the same either way.
// Replaces tf.unique at python/elasticdl/embedding_delegate.py:85 and the key pass of
// deduplicate_indexed_slices (python/common/tensor_utils.py:53-58).
#pragma once
#include "ps_kernels.cuh"

namespace b200ps_impl {

constexpr long long kEmptyKey = (long long)0x8000000000000000ULL;
constexpr int kUThreads = 256;
constexpr long long kUSpins = 1LL << 22;
constexpr unsigned kErrUnique = 16u;

struct UniqueBounds {      // per segment: ids are known to be < bound (0 = unknown): the segment dedups
  int bound[kMaxSegs];     // through a direct-address position array dpos[off .. off+bound) instead of
  long long off[kMaxSegs]; // the hash table: no keys, no CAS, no probing
  int* dpos;
};

// Direct-address segments are not cleared between calls: positions are stored under an epoch prefix
// that DEcreases from call to call, so atomicMin prefers this call's entries and stale ones read as
// empty.  hdr = {magic, epoch, cleared cycle, -, barrier counter} lives in the workspace (a fresh /
// foreign workspace fails the magic test and is cleared); every kUniqEpochs calls the prefix wraps
// and the arrays are cleared for real by the first tagged call of the new cycle.
constexpr int kUniqPosBits = 20;
constexpr int kUniqEpochs = 2047;  // prefixes 0..2046 keep the value below 0x7fffffff (= empty)

struct UIdLayout {               // ids_kind == 2: every segment has its own element width and byte offset
  long long off[kMaxSegs];       // byte offset of segment t inside the ids buffer
  unsigned char width[kMaxSegs]; // 1, 2, 4 (unsigned) or 8 (int64) bytes per id
};

struct UArgs {
  const void* ids;
  long long k;
  int T, ids32;                  // ids32: 0 = int64 [T][k], 1 = int32 [T][k], 2 = per-segment layout (UIdLayout)
  long long* keys;              // [T][cap]   (hashed segments)
  int* minpos;                  // [T][cap]
  int* fp;                      // [T][k]  slot / id, then first position of the id at i
  int* rank_at;                 // [T][k]
  unsigned long long* status;   // [T][ntiles] look-back descriptors {tag:30 | flag:2 | value:32}
  unsigned long long* hdr;
  unsigned long long magic;
  int cap, ntiles, tagged, use_bounds, n_direct, n_hashed;
  UniqueBounds ub;
  int64_t* uniq;
  int* inv;
  int* n_unique;
  unsigned* err;
  long long* dbg;               // optional [blocks][8] globaltimer stamps per phase (profiling aid)
};

__device__ __forceinline__ long long u_id(const UArgs& a, const UIdLayout& L, int t, long long i) {
  if (a.ids32 == 0) return reinterpret_cast<const long long*>(a.ids)[(long long)t * a.k + i];
  if (a.ids32 == 1) return (long long)reinterpret_cast<const int*>(a.ids)[(long long)t * a.k + i];
  const unsigned char* base = reinterpret_cast<const unsigned char*>(a.ids) + L.off[t];
  const int w = L.width[t];
  if (w == 1) return (long long)base[i];
  if (w == 2) return (long long)reinterpret_cast<const unsigned short*>(base)[i];
  if (w == 4) return (long long)reinterpret_cast<const unsigned int*>(base)[i];
  return reinterpret_cast<const long long*>(base)[i];
}
// Branch-free id loads for unrolled loops: the element width is a property of the SEGMENT, so it is dispatched
// once around the loop (U_KIND_SWITCH) and every load inside is one plain instruction.  With u_id() in the loop
// each load sat behind its own width branch and the loads of a thread ran one after the other (32 sequential
// round trips in k_unique_small).
template <int W, bool SGN>
__device__ __forceinline__ long long u_ld(const unsigned char* b, long long i) {
  if (W == 1) return (long long)b[i];
  if (W == 2) return (long long)reinterpret_cast<const unsigned short*>(b)[i];
  if (W == 4) return SGN ? (long long)reinterpret_cast<const int*>(b)[i] : (long long)reinterpret_cast<const unsigned int*>(b)[i];
  return reinterpret_cast<const long long*>(b)[i];
}
// kind: 0 = 1 byte, 1 = 2 bytes, 2 = 4 bytes unsigned, 3 = int32, 4 = int64
__device__ __forceinline__ int u_seg_kind(const UArgs& a, const UIdLayout& L, int t, const unsigned char** base) {
  const unsigned char* ids = reinterpret_cast<const unsigned char*>(a.ids);
  if (a.ids32 == 0) { *base = ids + (long long)t * a.k * 8; return 4; }
  if (a.ids32 == 1) { *base = ids + (long long)t * a.k * 4; return 3; }
  *base = ids + L.off[t];
  const int w = L.width[t];
  return w == 1 ? 0 : (w == 2 ? 1 : (w == 4 ? 2 : 4));
}
#define U_KIND_SWITCH(KIND, ...)                                              \
  switch (KIND) {                                                             \
    case 0: { constexpr int W = 1; constexpr bool SG = false; __VA_ARGS__; } break; \
    case 1: { constexpr int W = 2; constexpr bool SG = false; __VA_ARGS__; } break; \
    case 2: { constexpr int W = 4; constexpr bool SG = false; __VA_ARGS__; } break; \
    case 3: { constexpr int W = 4; constexpr bool SG = true; __VA_ARGS__; } break;  \
    default: { constexpr int W = 8; constexpr bool SG = true; __VA_ARGS__; } break; \
  }

__device__ __forceinline__ unsigned long long u_ldv(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.volatile.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void u_stv(unsigned long long* p, unsigned long long v) {
  asm volatile("st.volatile.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

__device__ __forceinline__ long long u_now() {
  long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
#define U_STAMP(slot) do { if (a.dbg && threadIdx.x == 0) a.dbg[(long long)blockIdx.x * 8 + (slot)] = u_now(); } while (0)

__device__ __forceinline__ void u_grid_barrier(unsigned* bar, unsigned target, unsigned* err) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(bar, 1u);
    long long spins = 0;
    while (*(volatile unsigned*)bar < target) {
      __nanosleep(40);
      if (++spins > kUSpins) {
        if (err) atomicOr(err, kErrUnique);
        break;
      }
    }
    __threadfence();
  }
  __syncthreads();
}

constexpr unsigned kUFlagA = 1u, kUFlagP = 2u;
__device__ __forceinline__ unsigned long long u_word(unsigned tag, unsigned flag, unsigned value) {
  return ((unsigned long long)((tag << 2) | flag) << 32) | value;
}

// Work unit = 1024 consecutive positions of one segment (256 threads x 4; thread tid owns positions
// q*256 + tid, so every global access of a warp is coalesced).  A block takes a RUN of consecutive units of
// one segment (host-built map): segments whose ids are mostly distinct -- large tables: every position
// costs an atomic and two uncached 32 B sector reads -- get one unit per block, segments with tiny id
// ranges -- cache-resident position arrays, almost every position a duplicate -- several, so that all
// blocks of a phase finish together (with equal tiles the large-table blocks took much longer than the
// median and every other block waited at the grid barrier; tools/unique_timeline.py shows it).
constexpr int kUPPT = 4;
constexpr int kUUnit = kUThreads * kUPPT;  // 1024

struct URuns {                     // run slot -> (segment, first unit, units); a block takes slots b, b + grid, ...
  int blk_prefix[kMaxSegs + 1];    // per-segment map (T <= kMaxSegs): first slot of segment t
  int run[kMaxSegs];               // units per slot of segment t
  int per_seg;                     // 1: the map above; 0: `bps` slots of `uniform_run` units per segment
  int uniform_run, bps;
  int nslots;
};

__global__ void __launch_bounds__(kUThreads, 4) k_unique(const __grid_constant__ UArgs a, const __grid_constant__ URuns ur,
                                                         const __grid_constant__ UIdLayout idl) {
  constexpr int NW = kUThreads / 32;
  constexpr int PPT = kUPPT;
  __shared__ int s_cnt[PPT * NW];  // first-occurrence counts per (q, warp), then their exclusive prefix
  __shared__ int s_excl;
  // header snapshot: stable until block 0 rewrites it after the last barrier
  const bool fresh = a.hdr[0] != a.magic;
  const unsigned long long epoch64 = fresh ? 0ULL : a.hdr[1];
  const bool stale_cycle = fresh || a.hdr[2] != epoch64 / kUniqEpochs;
  const int epoch = (int)(epoch64 % kUniqEpochs);
  const int prefix = a.tagged ? (kUniqEpochs - 1 - epoch) << kUniqPosBits : 0;
  const int pos_mask = a.tagged ? (1 << kUniqPosBits) - 1 : 0x7fffffff;
  const unsigned tag = (unsigned)((epoch64 + 1ULL) % 0x3ffffffeULL) + 1u;
  unsigned* bar = reinterpret_cast<unsigned*>(a.hdr + 4);  // zeroed by the host before every launch
  unsigned target = 0;
  const long long gsz = (long long)gridDim.x * kUThreads;
  const long long gtid = (long long)blockIdx.x * kUThreads + threadIdx.x;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  const long long k = a.k;
  const int T = a.T;
  const int ups = a.ntiles;  // units per segment
  const long long units = (long long)T * ups;  // descriptors are sized for one per unit (>= run slots)

  // run slot -> segment t, first unit j0 (inside the segment), number of units
  auto slot_of = [&](const int slot, int& t, long long& j0, int& cnt) {
    int r, u0;
    if (ur.per_seg) {
      int lo = 0, hi = T;
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (ur.blk_prefix[mid] <= slot) lo = mid; else hi = mid;
      }
      t = lo;
      r = ur.run[lo];
      u0 = (slot - ur.blk_prefix[lo]) * r;
    } else {
      t = slot / ur.bps;
      r = ur.uniform_run;
      u0 = (slot - t * ur.bps) * r;
    }
    j0 = u0;
    cnt = u0 < ups ? (ups - u0 < r ? ups - u0 : r) : 0;
  };
  const int nslots = ur.nslots;

  // ---- phase 0: clear what this call cannot read as empty ----
  const bool clear_direct = a.n_direct > 0 && (!a.tagged || stale_cycle);
  if (a.n_hashed > 0 || clear_direct || fresh) {
    if (fresh) {  // descriptors of a foreign layout could carry this call's tag
      for (long long i = gtid; i < units; i += gsz) a.status[i] = 0ULL;
    }
    if (a.n_hashed > 0 || clear_direct) {
      if (!a.use_bounds) {
        const long long n = (long long)T * a.cap;
        for (long long i = gtid; i < n; i += gsz) {
          a.keys[i] = kEmptyKey;
          a.minpos[i] = 0x7fffffff;
        }
      } else {
        for (int t = 0; t < T; ++t) {
          if (a.ub.bound[t] > 0) {
            if (!clear_direct) continue;
            int* dp = a.ub.dpos + a.ub.off[t];
            for (long long i = gtid; i < a.ub.bound[t]; i += gsz) dp[i] = 0x7fffffff;
          } else {
            long long* keys = a.keys + (long long)t * a.cap;
            int* mp = a.minpos + (long long)t * a.cap;
            for (long long i = gtid; i < a.cap; i += gsz) {
              keys[i] = kEmptyKey;
              mp[i] = 0x7fffffff;
            }
          }
        }
      }
    }
    target += gridDim.x;
    u_grid_barrier(bar, target, a.err);
  }
  U_STAMP(0);

  // ---- phase A: insert.  position array entry of every id <- min(position) ----
  for (int slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
   int t, gcnt;
   long long j0;
   slot_of(slot, t, j0, gcnt);
   for (int gi = 0; gi < gcnt; ++gi) {
    const long long base = (j0 + gi) * kUUnit;
    const bool direct = a.use_bounds && a.ub.bound[t] > 0;
    int* fp = a.fp + (long long)t * k;
    if (direct) {
      int* dp = a.ub.dpos + a.ub.off[t];
      const int bound = a.ub.bound[t];
      // probing first only pays when most positions are duplicates (small id range); for sparse segments
      // the probe is one more uncached sector read per position and almost never saves the atomic
      const bool probe = (long long)bound * 2 < k;
      int id[PPT], cur[PPT];  // bounded ids fit 32 bits
      bool any_bad = false;    // reported once per unit, after the loads and probes are in flight (a memory
                               // operation between them would serialise the loads behind it)
      {
        const unsigned char* sbase;
        const int kind = u_seg_kind(a, idl, t, &sbase);
        long long raw[PPT];
        U_KIND_SWITCH(kind, {
          _Pragma("unroll")
          for (int q = 0; q < PPT; ++q) {  // all id loads first, one instruction each
            const long long i = base + q * kUThreads + threadIdx.x;
            raw[q] = i < k ? u_ld<W, SG>(sbase, i) : 0;
          }
        });
#pragma unroll
        for (int q = 0; q < PPT; ++q) {
          const long long i = base + q * kUThreads + threadIdx.x;
          const bool bad = raw[q] < 0 || raw[q] >= bound;  // counted as id 0 and reported (kErrRange -> b200ps_check)
          id[q] = bad ? 0 : (int)raw[q];
          if (i < k) fp[i] = id[q];
          any_bad |= bad && i < k;
        }
      }
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        cur[q] = (probe && i < k) ? *(volatile int*)(dp + id[q]) : 0x7fffffff;
      }
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        const int v = prefix | (int)i;
        // warp-level id dedup among the lanes that would write: equal ids elect their lowest lane
        // (= smallest position); later units of this block see what the earlier ones recorded
        const bool want = i < k && cur[q] > v;
        const unsigned wm = __ballot_sync(0xffffffffu, want);
        if (wm) {
          const unsigned peers = __match_any_sync(0xffffffffu, want ? id[q] : -1 - lane) & wm;
          if (want && (__ffs(peers) - 1) == lane) atomicMin(dp + id[q], v);
        }
      }
      if (any_bad && a.err) atomicOr(a.err, kErrRange);
    } else {
      unsigned long long* keys = reinterpret_cast<unsigned long long*>(a.keys + (long long)t * a.cap);
      int* mp = a.minpos + (long long)t * a.cap;
      const unsigned mask = a.cap - 1;
      long long id[PPT];
      {
        const unsigned char* sbase;
        const int kind = u_seg_kind(a, idl, t, &sbase);
        U_KIND_SWITCH(kind, {
          _Pragma("unroll")
          for (int q = 0; q < PPT; ++q) {
            const long long i = base + q * kUThreads + threadIdx.x;
            id[q] = i < k ? u_ld<W, SG>(sbase, i) : 0;
          }
        });
      }
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        const bool live = i < k;
        const unsigned livem = __ballot_sync(0xffffffffu, live);  // dead lanes (ragged tail) never match
        const unsigned peers = __match_any_sync(0xffffffffu, id[q]) & livem;
        const int leader = live ? __ffs(peers) - 1 : lane;
        unsigned sl = 0;
        if (live && lane == leader) {
          sl = (unsigned)mix64((uint64_t)id[q]) & mask;
          while (true) {
            unsigned long long prev = keys[sl];
            if (prev == (unsigned long long)kEmptyKey)
              prev = atomicCAS(&keys[sl], (unsigned long long)kEmptyKey, (unsigned long long)id[q]);
            if (prev == (unsigned long long)kEmptyKey || prev == (unsigned long long)id[q]) break;
            sl = (sl + 1) & mask;
          }
          if (*(volatile int*)&mp[sl] > (int)i) atomicMin(&mp[sl], (int)i);
        }
        sl = __shfl_sync(0xffffffffu, sl, leader);
        if (live) fp[i] = (int)sl;
      }
    }
   }
  }
  U_STAMP(1);
  target += gridDim.x;
  u_grid_barrier(bar, target, a.err);
  U_STAMP(2);

  // ---- phase B: flags, single-pass scan over the RUNS of each segment, ranks, unique ids ----
  // The look-back works on whole runs: pass 1 counts the first occurrences of all the block's units and
  // publishes ONE aggregate, then looks back over the predecessor runs of the segment; pass 2 assigns the
  // ranks.  (Per-unit descriptors made a block's first unit wait for the previous block's LAST unit, which
  // itself sat behind that block's earlier look-backs: the segment was processed serially, as
  // tools/unique_timeline.py showed.)
  for (int slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
    int t, gcnt;
    long long j0;  // first unit of the run inside its segment
    slot_of(slot, t, j0, gcnt);
    if (gcnt == 0) continue;  // block-uniform
    __syncthreads();          // s_cnt / s_excl of the previous slot have been consumed
    const bool direct = a.use_bounds && a.ub.bound[t] > 0;
    const int* mp = direct ? a.ub.dpos + a.ub.off[t] : a.minpos + (long long)t * a.cap;
    const int pm = direct ? pos_mask : 0x7fffffff;
    int* fp = a.fp + (long long)t * k;
    // pass 1: first position of every id, per-thread count of first occurrences over the run
    int mine = 0;
    for (int gi = 0; gi < gcnt; ++gi) {
      const long long base = (j0 + gi) * kUUnit;
      int v[PPT];
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        v[q] = i < k ? fp[i] : 0;
      }
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        v[q] = i < k ? (mp[v[q]] & pm) : -1;
      }
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        if (i < k) {
          fp[i] = v[q];  // pass 2 and phase C read the first position from here (coalesced)
          mine += v[q] == (int)i;
        }
      }
    }
    // run total -> descriptor of this block's run; look back over the predecessor runs of the segment
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if (lane == 0) s_cnt[wid] = mine;
    __syncthreads();
    if (wid == 0) {
      int tot = lane < NW ? s_cnt[lane] : 0;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      // the runs of one segment are consecutive slots: first_slot .. slot - 1 precede this one
      const int first_slot = ur.per_seg ? ur.blk_prefix[t] : t * ur.bps;
      const long long jr = (long long)slot - first_slot;  // index of this run inside its segment
      if (lane == 0) u_stv(&a.status[slot], u_word(tag, jr == 0 ? kUFlagP : kUFlagA, (unsigned)tot));
      int excl = 0;
      long long look = jr - 1;
      long long spins = 0;
      while (look >= 0) {
        const long long idx = look - lane;
        bool valid = true;  // lanes before the segment start count as an exclusive prefix of 0
        unsigned flag = kUFlagP, val = 0;
        if (idx >= 0) {
          const unsigned long long wv = u_ldv(&a.status[first_slot + idx]);
          const unsigned hi = (unsigned)(wv >> 32);
          valid = (hi >> 2) == tag && (hi & 3u) != 0;
          flag = hi & 3u;
          val = (unsigned)wv;
        }
        if (!__all_sync(0xffffffffu, valid)) {
          if (++spins > kUSpins) {
            if (lane == 0 && a.err) atomicOr(a.err, kErrUnique);
            break;
          }
          __nanosleep(20);
          continue;
        }
        const unsigned pmask = __ballot_sync(0xffffffffu, flag == kUFlagP);
        const int stop = pmask ? __ffs(pmask) - 1 : 31;  // nearest run that already knows its inclusive prefix
        int contrib = lane <= stop ? (int)val : 0;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(0xffffffffu, contrib, o);
        excl += contrib;
        if (pmask) break;
        look -= 32;
      }
      if (lane == 0) {
        s_excl = excl;
        if (jr > 0) u_stv(&a.status[slot], u_word(tag, kUFlagP, (unsigned)(excl + tot)));
        if (j0 + gcnt == ups) a.n_unique[t] = excl + tot;  // the run that ends the segment
      }
    }
    __syncthreads();
    // pass 2: ranks in position order (unit by unit, q major, warp minor), unique ids, inverse of the firsts
    int run_base = s_excl;
    int* rank_at = a.rank_at + (long long)t * k;
    int* inv = a.inv + (long long)t * k;
    for (int gi = 0; gi < gcnt; ++gi) {
      const long long base = (j0 + gi) * kUUnit;
      int v[PPT];
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        v[q] = i < k ? fp[i] : -1;
      }
      __syncthreads();  // s_cnt of the previous unit (or of the run total) has been consumed
      unsigned fmask = 0;
      int wrank[PPT];
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const long long i = base + q * kUThreads + threadIdx.x;
        const bool f = i < k && v[q] == (int)i;
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        wrank[q] = __popc(bal & lt_mask);
        if (f) fmask |= 1u << q;
        if (lane == 0) s_cnt[q * NW + wid] = __popc(bal);
      }
      __syncthreads();
      if (wid == 0) {  // exclusive scan of the PPT*NW = 32 counts
        const int c = s_cnt[lane];
        int incl = c;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += y;
        }
        s_cnt[lane] = incl - c;
        if (lane == 31) s_excl = incl;  // this unit's total (the run's exclusive prefix was copied to run_base)
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        if (fmask >> q & 1u) {
          const long long i = base + q * kUThreads + threadIdx.x;
          const int r = run_base + s_cnt[q * NW + wid] + wrank[q];
          rank_at[i] = r;
          inv[i] = r;
          fp[i] = -1;  // done: phase C skips it
          a.uniq[(long long)t * k + r] = u_id(a, idl, t, i);
        }
      }
      run_base += s_excl;
    }
  }
  U_STAMP(3);
  target += gridDim.x;
  u_grid_barrier(bar, target, a.err);
  U_STAMP(4);

  // ---- phase C: inverse index of the duplicates = rank of their id's first occurrence ----
  for (int slot = blockIdx.x; slot < nslots; slot += gridDim.x) {
   int t, gcnt;
   long long j0;
   slot_of(slot, t, j0, gcnt);
   for (int gi = 0; gi < gcnt; ++gi) {
    const long long base = (j0 + gi) * kUUnit;
    const int* fp = a.fp + (long long)t * k;
    const int* rank_at = a.rank_at + (long long)t * k;
    int* inv = a.inv + (long long)t * k;
    int f[PPT];
#pragma unroll
    for (int q = 0; q < PPT; ++q) {
      const long long i = base + q * kUThreads + threadIdx.x;
      f[q] = i < k ? fp[i] : -1;
    }
#pragma unroll
    for (int q = 0; q < PPT; ++q) {
      const long long i = base + q * kUThreads + threadIdx.x;
      if (f[q] >= 0) inv[i] = rank_at[f[q]];
    }
   }
  }
  U_STAMP(5);
  if (blockIdx.x == 0 && threadIdx.x == 0) {  // every block took its header snapshot before barrier 1
    if (a.tagged) a.hdr[2] = epoch64 / kUniqEpochs;  // the position arrays are valid for this cycle
    else if (fresh) a.hdr[2] = ~0ULL;
    a.hdr[1] = epoch64 + 1ULL;
    a.hdr[0] = a.magic;
  }
}

// =============================================================================
// Segments with a SMALL id range (bound <= kUSmallMax): the whole segment is deduplicated by ONE block of 1024
// threads whose position array lives in shared memory -- shared-memory atomics instead of L2 atomics, an
// in-block scan instead of the decoupled look-back, no grid barrier, nothing read from the workspace.
// 30 of the 38 id groups of the DeepFM batch qualify (<= 16384 rows); they are 79 % of its ids, and phase A
// of the grid-wide kernel above is bound by the rate of L2 atomics on scattered addresses.  Same results:
// first-occurrence order, inverse index, n_unique; out-of-range ids count as id 0 and set kErrRange in the group's error word (b200ps_check raises).
// Taken when k <= 32768 (the ids of a segment then fit the registers of one block, see below).
//   A  pos[id] <- min(position)                (shared-memory atomicMin, checked first)
//   B  chunks of 4096 positions in order: first-occurrence flags -> ballot ranks -> block scan -> uniq[rank] = id,
//      pos[id] <- -(rank + 1)
//   C  inv[i] = -pos[id_i] - 1
// =============================================================================
constexpr int kUSmallMax = 16384;
constexpr int kUSThreads = 1024;
struct USmall {
  int seg[kMaxSegs];
  int n;
};

// IPT = ids per thread (k <= IPT * 1024): every id is loaded ONCE, with all of a thread's loads in flight together,
// and stays in a register through the three passes (a one-block-per-SM kernel has nothing else to hide a load
// behind: re-reading the ids per pass made it slower).  Thread tid owns positions j * 1024 + tid.
template <int IPT>
__global__ void __launch_bounds__(kUSThreads, 1) k_unique_small(const __grid_constant__ UArgs a, const __grid_constant__ UIdLayout idl,
                                                                const __grid_constant__ USmall us) {
  extern __shared__ int s_pos[];  // [bound]
  constexpr int NW = kUSThreads / 32, PPT = 4;
  static_assert(IPT % PPT == 0, "chunks of PPT positions per thread");
  __shared__ int s_cnt[PPT * NW];
  __shared__ int s_tot;
  const int t = us.seg[blockIdx.x];
  const int bound = a.ub.bound[t];
  const long long k = a.k;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned lt_mask = (1u << lane) - 1u;
  // two ids per register (bound <= 16384 < 0xffff = "no position"): 32 ids in 16 registers
  unsigned pk[IPT / 2];
  bool any_bad = false;
  {
    const unsigned char* sbase;
    const int kind = u_seg_kind(a, idl, t, &sbase);
    U_KIND_SWITCH(kind, {
      _Pragma("unroll")
      for (int j = 0; j < IPT; ++j) {
        const long long i = (long long)j * kUSThreads + tid;
        long long v = i < k ? u_ld<W, SG>(sbase, i) : 0xffff;
        const bool bad = i < k && (v < 0 || v >= bound);  // counted as id 0 and reported (kErrRange -> b200ps_check)
        if (bad) v = 0;
        any_bad |= bad;  // reported once, after the loads (a memory operation in this loop would serialise them)
        if (j & 1) pk[j >> 1] |= (unsigned)v << 16;
        else pk[j >> 1] = (unsigned)v;
      }
    });
  }
#define US_ID(j) ((int)((pk[(j) >> 1] >> (16 * ((j) & 1))) & 0xffffu))
#define US_LIVE(j) (US_ID(j) != 0xffff)
  for (int i = tid; i < bound; i += kUSThreads) s_pos[i] = 0x7fffffff;
  __syncthreads();
  if (any_bad && a.err) atomicOr(a.err, kErrRange);
  // ---- A ----
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    const int i = j * kUSThreads + tid;
    if (US_LIVE(j) && *(volatile int*)&s_pos[US_ID(j)] > i) atomicMin(&s_pos[US_ID(j)], i);
  }
  __syncthreads();
  // ---- B ----
  int run_base = 0;
  int64_t* uniq = a.uniq + (long long)t * k;
#pragma unroll
  for (int c = 0; c < IPT / PPT; ++c) {
    if ((long long)c * PPT * kUSThreads < k) {  // block-uniform
      int wrank[PPT];
      unsigned fmask = 0;
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        const int j = c * PPT + q;
        const int i = j * kUSThreads + tid;
        const bool f = US_LIVE(j) && s_pos[US_ID(j)] == i;
        const unsigned bal = __ballot_sync(0xffffffffu, f);
        wrank[q] = __popc(bal & lt_mask);
        if (f) fmask |= 1u << q;
        if (lane == 0) s_cnt[q * NW + wid] = __popc(bal);
      }
      __syncthreads();
      if (wid == 0) {  // exclusive scan of the PPT * NW = 128 counts (linear order = q major, warp minor): four per lane
        int cc[4], sum = 0;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          cc[x] = s_cnt[lane * 4 + x];
          sum += cc[x];
        }
        int incl = sum;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int y = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += y;
        }
        int run = incl - sum;
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          s_cnt[lane * 4 + x] = run;
          run += cc[x];
        }
        if (lane == 31) s_tot = incl;
      }
      __syncthreads();
#pragma unroll
      for (int q = 0; q < PPT; ++q) {
        if (fmask >> q & 1u) {
          const int j = c * PPT + q;
          const int r = run_base + s_cnt[q * NW + wid] + wrank[q];
          uniq[r] = (int64_t)US_ID(j);
          s_pos[US_ID(j)] = -(r + 1);
        }
      }
      run_base += s_tot;
      __syncthreads();  // s_cnt / s_tot are rewritten by the next chunk, which must also see the ranks in s_pos
    }
  }
  // ---- C ----
  int* inv = a.inv + (long long)t * k;
#pragma unroll
  for (int j = 0; j < IPT; ++j) {
    const long long i = (long long)j * kUSThreads + tid;
    if (US_LIVE(j)) inv[i] = -s_pos[US_ID(j)] - 1;
  }
  if (tid == 0) a.n_unique[t] = run_base;
#undef US_ID
#undef US_LIVE
}

}  // namespace b200ps_impl
