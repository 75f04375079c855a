// Flat-scheduled row kernels (round 2): pull / set / push for every direct-indexed table and
// dense-parameter row view, any dim, up to kMaxSegs (table, ids) segments in ONE launch.
//
// Why one flat launch rather than one grid row per segment (blockIdx.y = segment, as the hashed-table kernels
// k_rows_copy / k_push_rows of ps_kernels.cuh still run):
//   * a DeepFM step addresses 76 tables whose live sizes (device-side unique counts) range from 3 to
//     25 000 rows.  blockIdx.y = segment gave the big segments 3+ grid-stride passes of dependent
//     latencies while the blocks of the small ones exited at once.  Here the lane-items of all
//     segments form ONE index space (prefix over the live counts, built per block in shared memory
//     from the device-side counts) that a persistent grid walks in whole-warp runs, so every SM
//     carries the same share whatever the split;
//   * everything a row access depends on besides the id -- the table's per-shard base pointers, bitmap
//     pointers, strides, slot offsets -- is resolved on the HOST and travels in the kernel's parameter
//     block (up to 21 KB; sm_70+ takes 32 KB): the kernels read it through the constant cache with a
//     warp-uniform index and never touch the device-side table directory.  The per-row dependent
//     chain is id -> record -> store (it was count -> id -> TableView -> runtime scalars -> record ->
//     store).  [The first flat version staged the directory into shared memory per block: with 8 blocks
//     per SM x 76 segments that prologue dominated the kernel.]
//   * each thread keeps U independent rows in flight: all id loads, then all record / gradient
//     loads, then the arithmetic and the stores;
//   * the update is "lane = (row, column)": the 8 lanes of a dim-8 row read 32 contiguous bytes of
//     param, of each slot and of the gradient -- one full sector per array per row, no shuffles --
//     and every lane executes exactly one element update.
// Measured and rejected (git history, commit "flat kernels: warp-uniform segment fast path"): specialising the
// loop body for warp-iterations that lie inside one segment (segment constants loaded once, no per-item search)
// cut instructions but cost 12-16 registers and no time: these kernels are bound by memory round trips, not by
// issue slots.
// Arithmetic is opt_update<> of ps_kernels.cuh: results stay bit-identical to the oracle.
// Replaces go/pkg/kernel/kernel.go:35-199 (Sparse* / Indexed* row loops) and
// go/pkg/common/embedding_table.go:61-77 (Get / SetEmbeddingVectors).
#pragma once
#include "ps_kernels.cuh"

namespace b200ps_impl {

struct FlatSegP {          // one segment, fully resolved by the host (96 B)
  const int64_t* ids;
  const int32_t* n_dev;    // live count on the device (<= n) or nullptr
  float* rows;             // user rows [n, dim]
  long long rows_cap;      // rows per shard (striped) / total rows (dense view)
  long long soff[kMaxSlots + 1];
  int n, stride, dim, lpr; // lpr = lanes per row
  int shift, owner, vec, pad;  // shift = log2(lpr) or -1; vec: 16 B chunks (copy kernels)
};

template <int NSMAX>
struct FlatArgs {
  FlatSegP seg[kMaxSegs];
  float* base[kMaxSegs * NSMAX];        // [seg * ns + shard]
  uint32_t* present[kMaxSegs * NSMAX];  // created-row bitmaps (nullptr: untracked)
  const PushRt* rt;
  unsigned* err;
  int nseg, ns, shard_shift, slot;
};

__device__ __forceinline__ float ld_f1(const float* p) {
  float v;
  asm volatile("ld.global.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ void st_f1(float* p, float v) {
  asm volatile("st.global.L1::no_allocate.f32 [%0], %1;" ::"l"(p), "f"(v));
}

// Largest s < nseg with prefix[s] <= w (empty segments repeat their prefix and are skipped).
__device__ __forceinline__ int flat_seg_of(const long long* prefix, int nseg, long long w) {
  int lo = 0, hi = nseg;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (prefix[mid] <= w) lo = mid; else hi = mid;
  }
  return lo;
}

// Block prologue: live lane-items of every segment (device-side counts) -> exclusive prefix.
template <int NSMAX>
__device__ __forceinline__ void flat_prefix(const FlatArgs<NSMAX>& p, long long* prefix) {
  const int nseg = p.nseg;
  for (int s = threadIdx.x; s < nseg; s += blockDim.x) {
    int n = p.seg[s].n;
    const int32_t* nd = p.seg[s].n_dev;
    if (nd != nullptr) {
      const int live = *nd;
      n = live < n ? live : n;
    }
    prefix[s + 1] = (long long)n * p.seg[s].lpr;  // count for now, scanned below
  }
  __syncthreads();
  if (threadIdx.x < 32) {  // exclusive scan of <= 96 counts: three per lane
    constexpr int PER = (kMaxSegs + 31) / 32;
    const int lane = threadIdx.x;
    long long v[PER], sum = 0;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int idx = lane * PER + j;
      v[j] = idx < nseg ? prefix[idx + 1] : 0;
      sum += v[j];
    }
    long long incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += y;
    }
    long long run = incl - sum;
#pragma unroll
    for (int j = 0; j < PER; ++j) {
      const int idx = lane * PER + j;
      run += v[j];
      if (idx < nseg) prefix[idx + 1] = run;
    }
    if (lane == 0) prefix[0] = 0;
  }
  __syncthreads();
}

struct FlatLoc {
  float* rec;
  uint32_t* pres;  // bitmap word of this row (nullptr: untracked)
  uint32_t bit;
  int shard;
  bool ok;
};

template <int NSMAX>
__device__ __forceinline__ FlatLoc flat_locate(const FlatArgs<NSMAX>& p, int seg, long long id) {
  const FlatSegP& sp = p.seg[seg];
  FlatLoc r;
  const bool nonneg = id >= 0;
  const long long uid = nonneg ? id : 0;
  long long slot;
  if (NSMAX == 1) {
    r.shard = 0;
    slot = uid;
  } else if (sp.owner >= 0) {
    r.shard = sp.owner;
    slot = uid;
  } else if (p.shard_shift >= 0) {
    r.shard = (int)(uid & (long long)(p.ns - 1));
    slot = uid >> p.shard_shift;
  } else {
    slot = uid / p.ns;
    r.shard = (int)(uid - slot * p.ns);
  }
  r.ok = nonneg && slot < sp.rows_cap;
  if (!r.ok) slot = 0;
  const int at = NSMAX == 1 ? seg : seg * p.ns + r.shard;
  r.rec = p.base[at] + slot * sp.stride;
  uint32_t* bm = p.present[at];
  r.pres = bm ? bm + (slot >> 5) : nullptr;
  r.bit = 1u << (slot & 31);
  return r;
}

__device__ __forceinline__ void flat_mark_present(const FlatLoc& r) {
  if (r.pres == nullptr) return;
  if (!(*(volatile uint32_t*)r.pres & r.bit)) atomicOr_system(r.pres, r.bit);  // the shard may be a peer GPU
}
// The same in two halves: the bitmap word is LOADED together with the row's record (it arrives with it) and
// tested after the stores, so the test never adds a dependent round trip of its own.
__device__ __forceinline__ uint32_t flat_present_word(const FlatLoc& r) {
  return r.pres ? *(volatile uint32_t*)r.pres : 0xffffffffu;
}
__device__ __forceinline__ void flat_mark_present(const FlatLoc& r, uint32_t word) {
  if (!(word & r.bit)) atomicOr_system(r.pres, r.bit);
}

// item w of the flat space -> (segment, row, column); `seg` is a running hint (items of one thread ascend)
struct FlatItem {
  long long row;
  int seg, col;
  bool live;
};
template <int NSMAX>
__device__ __forceinline__ FlatItem flat_item(const FlatArgs<NSMAX>& p, const long long* prefix, long long w, long long total,
                                              int& seg) {
  FlatItem it;
  it.live = w < total;
  if (it.live)
    while (w >= prefix[seg + 1]) ++seg;
  it.seg = seg;
  const long long local = it.live ? w - prefix[seg] : 0;
  const int sh = p.seg[seg].shift, lpr = p.seg[seg].lpr;
  it.row = sh >= 0 ? local >> sh : local / lpr;
  it.col = (int)(local - it.row * lpr);
  return it;
}

// ---------------------------------------------------------------------------
// pull (WRITE = false, PullEmbeddingVectors) / set (WRITE = true, SetEmbeddingVectors / slot access):
// item = (row, 16 B chunk) when the segment is vectorisable, else (row, float).
// ---------------------------------------------------------------------------
template <bool WRITE, int U, int NSMAX>
__global__ void __launch_bounds__(256) k_copy_flat(const __grid_constant__ FlatArgs<NSMAX> p) {
  __shared__ long long prefix[kMaxSegs + 1];
  flat_prefix(p, prefix);
  const int nseg = p.nseg;
  const long long total = prefix[nseg];
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarp = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long wb = warp * (32 * U); wb < total; wb += nwarp * (32 * U)) {
    const long long w0 = wb + lane;
    int seg = flat_seg_of(prefix, nseg, w0 < total ? w0 : total - 1);
    FlatItem it[U];
    long long id[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      it[k] = flat_item(p, prefix, wb + k * 32 + lane, total, seg);
      id[k] = it[k].live ? p.seg[it[k].seg].ids[it[k].row] : 0;
    }
    FlatLoc loc[U];
    float4 x[U];
    float* dst[U];
    bool vec[U];
    uint32_t pw[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      dst[k] = nullptr;
      vec[k] = false;
      pw[k] = 0xffffffffu;
      if (!it[k].live) continue;
      const FlatSegP& sp = p.seg[it[k].seg];
      loc[k] = flat_locate(p, it[k].seg, id[k]);
      if (!loc[k].ok) {
        if (it[k].col == 0) atomicOr(p.err, kErrRange);
        continue;
      }
      vec[k] = sp.vec != 0;
      const int off = vec[k] ? 4 * it[k].col : it[k].col;
      float* rec = loc[k].rec + sp.soff[p.slot] + off;
      float* user = sp.rows + it[k].row * sp.dim + off;
      const float* src = WRITE ? user : rec;
      dst[k] = WRITE ? rec : user;
      if (vec[k]) x[k] = ld_f4(src);
      else x[k].x = ld_f1(src);
      if (it[k].col == 0) pw[k] = flat_present_word(loc[k]);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (dst[k] == nullptr) continue;
      if (vec[k]) st_f4(dst[k], x[k]);
      else st_f1(dst[k], x[k].x);
    }
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (dst[k] != nullptr) flat_mark_present(loc[k], pw[k]);
  }
}

// ---------------------------------------------------------------------------
// push: lane = (row, column).  dim-1 tables whose record is one float4 [p, s0, s1, s2] keep the
// single 16 B access.
// ---------------------------------------------------------------------------
template <int OPT, int U, int NSMAX>
__global__ void __launch_bounds__(256) k_push_flat(const __grid_constant__ FlatArgs<NSMAX> p, const OptParams o) {
  constexpr int S = opt_slots(OPT);
  __shared__ long long prefix[kMaxSegs + 1];
  __shared__ float s_lr[kMaxShards], s_alpha[kMaxShards], s_l2[kMaxShards];
  if (threadIdx.x < p.ns) {  // this push's effective lr / Adam alpha / FTRL l2 per shard (k_push_begin)
    s_lr[threadIdx.x] = p.rt->lr[threadIdx.x];
    s_alpha[threadIdx.x] = p.rt->alpha[threadIdx.x];
    s_l2[threadIdx.x] = p.rt->l2adj[threadIdx.x];
  }
  flat_prefix(p, prefix);
  const int nseg = p.nseg;
  const long long total = prefix[nseg];
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long nwarp = (long long)gridDim.x * (blockDim.x >> 5);
  for (long long wb = warp * (32 * U); wb < total; wb += nwarp * (32 * U)) {
    const long long w0 = wb + lane;
    int seg = flat_seg_of(prefix, nseg, w0 < total ? w0 : total - 1);
    FlatItem it[U];
    long long id[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      it[k] = flat_item(p, prefix, wb + k * 32 + lane, total, seg);
      id[k] = it[k].live ? p.seg[it[k].seg].ids[it[k].row] : 0;
    }
    FlatLoc loc[U];
    float g[U], pv[U], s0[U], s1[U], s2[U];
    float* rp[U];
    bool rec4[U];
    uint32_t pw[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      rp[k] = nullptr;
      rec4[k] = false;
      pw[k] = 0xffffffffu;
      s0[k] = s1[k] = s2[k] = 0.f;
      if (!it[k].live) continue;
      const FlatSegP& sp = p.seg[it[k].seg];
      loc[k] = flat_locate(p, it[k].seg, id[k]);
      if (!loc[k].ok) {
        if (it[k].col == 0) atomicOr(p.err, kErrRange);
        continue;
      }
      const int dim = sp.dim;
      g[k] = ld_f1(sp.rows + it[k].row * dim + it[k].col);
      rp[k] = loc[k].rec + it[k].col;
      rec4[k] = S > 0 && dim == 1 && sp.stride == 4 && sp.soff[1] == 1;
      if (rec4[k]) {
        const float4 r = ld_f4(rp[k]);
        pv[k] = r.x; s0[k] = r.y; s1[k] = r.z; s2[k] = r.w;
      } else {
        pv[k] = ld_f1(rp[k]);
        if (S > 0) s0[k] = ld_f1(rp[k] + sp.soff[1]);
        if (S > 1) s1[k] = ld_f1(rp[k] + sp.soff[2]);
        if (S > 2) s2[k] = ld_f1(rp[k] + sp.soff[3]);
      }
      if (it[k].col == 0) pw[k] = flat_present_word(loc[k]);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      if (rp[k] == nullptr) continue;
      const FlatSegP& sp = p.seg[it[k].seg];
      const int sh = loc[k].shard;
      opt_update<OPT>(g[k], pv[k], s0[k], s1[k], s2[k], s_lr[sh], s_alpha[sh], s_l2[sh], o);
      if (rec4[k]) {
        st_f4(rp[k], make_float4(pv[k], s0[k], s1[k], s2[k]));
      } else {
        st_f1(rp[k], pv[k]);
        if (S > 0) st_f1(rp[k] + sp.soff[1], s0[k]);
        if (S > 1) st_f1(rp[k] + sp.soff[2], s1[k]);
        if (S > 2) st_f1(rp[k] + sp.soff[3], s2[k]);
      }
    }
#pragma unroll
    for (int k = 0; k < U; ++k)
      if (rp[k] != nullptr) flat_mark_present(loc[k], pw[k]);
  }
}

}  // namespace b200ps_impl
