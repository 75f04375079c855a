// sm_90a kernels of the PS hot path.  All of them are HBM-bound integer /
// fp32 elementwise work (no dense contraction -> no tensor cores): the rules
// that matter are one 32-byte sector (two 128-bit accesses) per thread,
// enough loads in flight to cover HBM / NVLink latency, and no wasted sectors.
#pragma once
#include "ps_types.cuh"

namespace b200ps_impl {

// ---------------------------------------------------------------------------
// Optimizer arithmetic: exact operation order of go/pkg/kernel/capi/
// kernel_api.cc with round-to-nearest intrinsics so that nvcc cannot contract
// mul+add into FMA (the reference is built without FMA, elasticdl/Makefile:23-25).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ float fdiv(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float fsqrt(float a) { return __fsqrt_rn(a); }

template <int OPT>
__device__ __forceinline__ void opt_update(float g, float& p, float& s0, float& s1, float& s2,
                                           float lr, float alpha, float l2adj, const OptParams& o) {
  if (OPT == kSGD) {  // kernel_api.cc:6-14
    p = sub(p, mul(lr, g));
  } else if (OPT == kMomentum) {  // kernel_api.cc:16-38
    float v = add(mul(o.mu, s0), g);
    s0 = v;
    if (o.nesterov)
      p = sub(p, mul(lr, add(g, mul(o.mu, v))));
    else
      p = sub(p, mul(lr, v));
  } else if (OPT == kAdam || OPT == kAMSGrad) {  // kernel_api.cc:40-77
    float m = add(mul(o.beta1, s0), mul(o.c1, g));
    float v = add(mul(o.beta2, s1), mul(o.c2, mul(g, g)));
    s0 = m;
    s1 = v;
    float den = v;
    if (OPT == kAMSGrad) {
      float ms = s2 < v ? v : s2;
      s2 = ms;
      den = ms;
    }
    p = sub(p, fdiv(mul(alpha, m), add(fsqrt(den), o.epsilon)));
  } else if (OPT == kAdagrad) {  // kernel_api.cc:79-96
    float a = add(s0, mul(g, g));
    s0 = a;
    p = sub(p, fdiv(mul(lr, g), add(fsqrt(a), o.epsilon)));
  } else {  // FTRL: TF ApplyFtrl, lr_power = -0.5 (restated in DESIGN.md; parity unpinned)
    float gs = add(g, mul(mul(2.0f, o.l2s), p));
    float a_new = add(s0, mul(g, g));
    float sigma = fdiv(sub(fsqrt(a_new), fsqrt(s0)), lr);
    float lin = add(s1, sub(gs, mul(sigma, p)));
    float quad = add(fdiv(fsqrt(a_new), lr), mul(2.0f, l2adj));
    float sgn = lin > 0.0f ? 1.0f : (lin < 0.0f ? -1.0f : 0.0f);
    p = fabsf(lin) > o.l1 ? fdiv(sub(mul(sgn, o.l1), lin), quad) : 0.0f;
    s1 = lin;
    s0 = a_new;
  }
}

// ---------------------------------------------------------------------------
// Row addressing: shard = id % N, slot = id / N (hash_utils.py:22-23).
// ---------------------------------------------------------------------------
struct RowLoc {
  float* rec;
  int64_t slot;
  int shard;
  bool ok;
};

__host__ __device__ __forceinline__ uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33; return x;
}

// Hashed table (unbounded ids, the reference's map[int64]*Tensor, embedding_table.go:22-58):
// find the slot of `id` on its shard, claiming an empty slot on first touch (lazy creation on
// pull OR push, kernel_test.go:56-66).  Linear probing, system-scope CAS (the shard may be a peer).
__device__ __forceinline__ int64_t probe_slot(long long* keys, int64_t rows, int64_t id, bool* ok) {
  const uint64_t mask = (uint64_t)rows - 1;  // rows is a power of two
  uint64_t h = mix64((uint64_t)id) & mask;
  for (int64_t tries = 0; tries < rows; ++tries) {
    long long k = *(volatile long long*)(keys + h);
    if (k == kEmptySlot)
      k = (long long)atomicCAS_system((unsigned long long*)(keys + h), (unsigned long long)kEmptySlot, (unsigned long long)id);
    if (k == kEmptySlot || k == id) return (int64_t)h;
    h = (h + 1) & mask;
  }
  *ok = false;
  return 0;
}

__device__ __forceinline__ RowLoc locate(const GroupView& gv, const TableView& tv, int64_t id) {
  RowLoc r;
  int64_t slot;
  if (tv.owner >= 0) {
    r.shard = tv.owner;
    slot = id;
  } else if (gv.shard_shift >= 0) {
    r.shard = (int)(id & (int64_t)(gv.n_shards - 1));
    slot = id >> gv.shard_shift;
  } else {
    slot = id / gv.n_shards;
    r.shard = (int)(id - slot * gv.n_shards);
  }
  r.ok = (id >= 0) && (slot < tv.rows);
  if (tv.keys[r.shard] != nullptr) {  // hashed: `slot` so far is id / N, the key
    r.ok = id >= 0;
    bool found = true;
    slot = r.ok ? probe_slot(tv.keys[r.shard], tv.rows, id, &found) : 0;
    if (!found) {
      atomicOr(gv.err, kErrFull);
      r.ok = false;
    }
  }
  r.slot = slot;
  r.rec = tv.base[r.shard] + slot * tv.row_stride;
  return r;
}

// Created-row bitmap (len(EmbeddingVectors) / ToIndexedSlices).  Called AFTER the row loads
// are issued so that the (possibly remote) bitmap read overlaps them.
__device__ __forceinline__ void mark_present(const TableView& tv, const RowLoc& r) {
  uint32_t* bm = tv.present[r.shard];
  if (bm == nullptr) return;
  uint32_t* w = bm + (r.slot >> 5);
  const uint32_t bit = 1u << (r.slot & 31);
  if (!(*(volatile uint32_t*)w & bit)) atomicOr_system(w, bit);  // the shard may be a peer GPU
}

__device__ __forceinline__ int seg_count(const b200ps_seg_t& sg) {
  int n = sg.n;
  if (sg.n_dev != nullptr) {
    int live = *sg.n_dev;
    n = live < n ? live : n;
  }
  return n;
}

// 128-bit accesses that do not pollute L1 (every row is touched once per launch).
__device__ __forceinline__ float4 ld_f4(const float* p) {
  float4 v;
  asm volatile("ld.global.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(p));
  return v;
}
__device__ __forceinline__ void st_f4(float* p, float4 v) {
  asm volatile("st.global.L1::no_allocate.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y),
               "f"(v.z), "f"(v.w));
}

// ---------------------------------------------------------------------------
// pull_rows: rows_dev[i, :] = row(ids[i]).  VPT = 128-bit vectors per thread
// (2 -> one 32 B sector per thread, dim % 8 == 0; 1 -> dim % 4 == 0; 0 -> scalar).
// WRITE = false: gather (PullEmbeddingVectors); true: scatter (SetEmbeddingVectors).
// ---------------------------------------------------------------------------
template <int VPT, bool WRITE>
__global__ void __launch_bounds__(256) k_rows_copy(GroupView gv, SegBatch sb, int slot) {
  const b200ps_seg_t& sg = sb.seg[blockIdx.y];
  const TableView& tv = gv.tables[sg.table];
  const int n = seg_count(sg);
  const int dim = tv.dim;
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;  // floats per thread
  const int chunks = dim / W;
  const long long work = (long long)n * chunks;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < work; w += stride) {
    const long long row = chunks == 1 ? w : w / chunks;
    const int c = chunks == 1 ? 0 : (int)(w - row * chunks);
    const int64_t id = sg.ids_dev[row];
    RowLoc loc = locate(gv, tv, id);
    float* user = sg.rows_dev + row * dim + c * W;
    if (!loc.ok) {
      atomicOr(gv.err, kErrRange);
      continue;
    }
    float* rec = loc.rec + tv.slot_off[slot] + c * W;
    if (VPT == 0) {
      if (WRITE) { *rec = *user; if (c == 0) mark_present(tv, loc); }
      else { float x = *rec; if (c == 0) mark_present(tv, loc); *user = x; }
    } else {
      float4 x[VPT == 0 ? 1 : VPT];
#pragma unroll
      for (int v = 0; v < VPT; ++v) x[v] = ld_f4((WRITE ? user : rec) + 4 * v);
      if (c == 0) mark_present(tv, loc);
#pragma unroll
      for (int v = 0; v < VPT; ++v) st_f4((WRITE ? rec : user) + 4 * v, x[v]);
    }
  }
}

// ---------------------------------------------------------------------------
// push_rows: Sparse*/Indexed* kernels (kernel.go:35-55,69-96,119-160,172-199)
// fused with the optimizer update, one launch for many tables.  ids are unique
// within a segment (PSClient dedups before pushing, ps_client.py:255-257).
// ---------------------------------------------------------------------------
template <int OPT, int VPT>
__global__ void __launch_bounds__(256) k_push_rows(GroupView gv, SegBatch sb, OptParams o) {
  constexpr int S = opt_slots(OPT);
  const b200ps_seg_t& sg = sb.seg[blockIdx.y];
  const TableView& tv = gv.tables[sg.table];
  const int n = seg_count(sg);
  const int dim = tv.dim;
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  const int chunks = dim / W;
  const long long work = (long long)n * chunks;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const int64_t o0 = tv.slot_off[1], o1 = tv.slot_off[2], o2 = tv.slot_off[3];
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < work; w += stride) {
    const long long row = chunks == 1 ? w : w / chunks;
    const int c = chunks == 1 ? 0 : (int)(w - row * chunks);
    const int64_t id = sg.ids_dev[row];
    RowLoc loc = locate(gv, tv, id);
    if (!loc.ok) {
      atomicOr(gv.err, kErrRange);
      continue;
    }
    const float lr = gv.rt->lr[loc.shard];
    const float alpha = gv.rt->alpha[loc.shard];
    const float l2adj = gv.rt->l2adj[loc.shard];
    const float* gp = sg.rows_dev + row * dim + c * W;
    float* rec = loc.rec + c * W;
    if (VPT == 0) {
      float g = *gp, p = *rec, s0 = 0.f, s1 = 0.f, s2 = 0.f;
      if (S > 0) s0 = rec[o0];
      if (S > 1) s1 = rec[o1];
      if (S > 2) s2 = rec[o2];
      if (c == 0) mark_present(tv, loc);
      opt_update<OPT>(g, p, s0, s1, s2, lr, alpha, l2adj, o);
      *rec = p;
      if (S > 0) rec[o0] = s0;
      if (S > 1) rec[o1] = s1;
      if (S > 2) rec[o2] = s2;
    } else {
      constexpr int NV = VPT == 0 ? 1 : VPT;
      float4 g[NV], p[NV], s0[NV], s1[NV], s2[NV];
#pragma unroll
      for (int v = 0; v < VPT; ++v) {  // all loads first: VPT*(2+S) 128-bit requests in flight
        g[v] = ld_f4(gp + 4 * v);
        p[v] = ld_f4(rec + 4 * v);
        if (S > 0) s0[v] = ld_f4(rec + o0 + 4 * v);
        if (S > 1) s1[v] = ld_f4(rec + o1 + 4 * v);
        if (S > 2) s2[v] = ld_f4(rec + o2 + 4 * v);
      }
      if (c == 0) mark_present(tv, loc);
#pragma unroll
      for (int v = 0; v < VPT; ++v) {
        float* gf = reinterpret_cast<float*>(&g[v]);
        float* pf = reinterpret_cast<float*>(&p[v]);
        float* af = reinterpret_cast<float*>(&s0[v]);
        float* bf = reinterpret_cast<float*>(&s1[v]);
        float* cf = reinterpret_cast<float*>(&s2[v]);
#pragma unroll
        for (int e = 0; e < 4; ++e) opt_update<OPT>(gf[e], pf[e], af[e], bf[e], cf[e], lr, alpha, l2adj, o);
      }
#pragma unroll
      for (int v = 0; v < VPT; ++v) {
        st_f4(rec + 4 * v, p[v]);
        if (S > 0) st_f4(rec + o0 + 4 * v, s0[v]);
        if (S > 1) st_f4(rec + o1 + 4 * v, s1[v]);
        if (S > 2) st_f4(rec + o2 + 4 * v, s2[v]);
      }
    }
  }
}

// float4 shuffle within groups of `width` lanes (the paired-record kernels below)
__device__ __forceinline__ float4 shfl4(float4 v, int src, int width) {
  float4 r;
  r.x = __shfl_sync(0xffffffffu, v.x, src, width);
  r.y = __shfl_sync(0xffffffffu, v.y, src, width);
  r.z = __shfl_sync(0xffffffffu, v.z, src, width);
  r.w = __shfl_sync(0xffffffffu, v.w, src, width);
  return r;
}

// ---------------------------------------------------------------------------
// Paired tables (b200ps_table_register_pair): a dim-8 table A and a dim-1 table B that are always
// addressed with the SAME ids (DeepFM's deep and wide embeddings of one id group,
// model_zoo/dac_ctr/deepfm_model.py:42-49) share one record per id,
//   [ A.p(8) B.p(1) pad(3) | A.s0(8) B.s0(1) pad(3) | ... ]   (48 B sections),
// so one request per id serves both tables: a pull is ONE 48 B read (lanes 0-1: A, lane 2: B)
// and an update is ONE contiguous read and ONE contiguous write of 48*(1+S) B.  Remote (NVLink)
// reads are bounded by outstanding requests x latency, so halving the requests halves the time.
// Each logical table stays addressable on its own through its TableView (generic kernels).
// ---------------------------------------------------------------------------
struct PairBatch {
  b200ps_seg_t a[kMaxSegs / 2];  // table A (dim 8): ids, n_dev, rows
  float* rows_b[kMaxSegs / 2];   // table B (dim 1) rows of the same ids
  int32_t table_b[kMaxSegs / 2];
  int nseg;
};

__global__ void __launch_bounds__(256) k_pair_pull(GroupView gv, PairBatch pb) {
  const b200ps_seg_t& sg = pb.a[blockIdx.y];
  const TableView& ta = gv.tables[sg.table];
  const TableView& tb = gv.tables[pb.table_b[blockIdx.y]];
  float* rows_b = pb.rows_b[blockIdx.y];
  const int n = seg_count(sg);
  const int lane = threadIdx.x & 31, c = lane & 3;
  const long long rows_pad = ((long long)n + 7) / 8 * 8;
  const long long stride = (long long)gridDim.x * blockDim.x / 4;
  for (long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 4; row < rows_pad; row += stride) {
    const bool live = row < n;
    long long id = (live && c == 0) ? sg.ids_dev[row] : 0;
    id = __shfl_sync(0xffffffffu, id, 0, 4);
    if (!live) continue;
    RowLoc loc = locate(gv, ta, id);
    if (!loc.ok) {
      if (c == 0) atomicOr(gv.err, kErrRange);
      continue;
    }
    if (c < 3) {
      const float4 x = ld_f4(loc.rec + 4 * c);  // lanes 0,1: A row; lane 2: [B.p, pad]
      if (c == 0) mark_present(ta, loc);
      if (c == 2) {
        mark_present(tb, loc);
        rows_b[row] = x.x;
      } else {
        st_f4(sg.rows_dev + row * 8 + 4 * c, x);
      }
    }
  }
}

template <int OPT>
__global__ void __launch_bounds__(256) k_pair_push(GroupView gv, PairBatch pb, OptParams o) {
  constexpr int S = opt_slots(OPT);
  constexpr int R4 = 3 * (1 + S);                       // 16 B chunks per record
  constexpr int LPR = R4 <= 4 ? 4 : R4 <= 8 ? 8 : 16;   // lanes per record
  const b200ps_seg_t& sg = pb.a[blockIdx.y];
  const TableView& ta = gv.tables[sg.table];
  const TableView& tb = gv.tables[pb.table_b[blockIdx.y]];
  const float* grad_b = pb.rows_b[blockIdx.y];
  const int n = seg_count(sg);
  const int lane = threadIdx.x & 31, c = lane & (LPR - 1);
  constexpr int RPW = 32 / LPR;
  const long long rows_pad = ((long long)n + RPW - 1) / RPW * RPW;
  const long long stride = (long long)gridDim.x * blockDim.x / LPR;
  for (long long row = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / LPR; row < rows_pad; row += stride) {
    const bool live = row < n;
    long long id = (live && c == 0) ? sg.ids_dev[row] : 0;
    id = __shfl_sync(0xffffffffu, id, 0, LPR);
    RowLoc loc = live ? locate(gv, ta, id) : RowLoc{nullptr, 0, 0, false};
    const bool ok = live && loc.ok;
    if (live && !loc.ok && c == 0) atomicOr(gv.err, kErrRange);
    float* rec = loc.rec + 4 * c;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f), g = v;
    if (ok && c < R4) v = ld_f4(rec);
    if (ok && c < 2) g = ld_f4(sg.rows_dev + row * 8 + 4 * c);
    if (ok && c == 2) g.x = grad_b[row];
    if (ok && c == 0) mark_present(ta, loc);
    if (ok && c == 2) mark_present(tb, loc);
    // chunk q of section k lives in lane 3k + q; bring the slot chunks to lanes q = 0,1,2
    const int q = c < 3 ? c : 0;
    float4 p = v, s0 = v, s1 = v, s2 = v;
    if (S > 0) s0 = shfl4(v, q + 3, LPR);
    if (S > 1) s1 = shfl4(v, q + 6, LPR);
    if (S > 2) s2 = shfl4(v, q + 9, LPR);
    if (c < 3) {
      const float lr = gv.rt->lr[loc.shard], alpha = gv.rt->alpha[loc.shard], l2adj = gv.rt->l2adj[loc.shard];
      float* gf = reinterpret_cast<float*>(&g);
      float* pf = reinterpret_cast<float*>(&p);
      float* af = reinterpret_cast<float*>(&s0);
      float* bf = reinterpret_cast<float*>(&s1);
      float* cf = reinterpret_cast<float*>(&s2);
      const int ne = c == 2 ? 1 : 4;  // lane 2 holds the single B element, its padding stays untouched
      for (int e = 0; e < ne; ++e) opt_update<OPT>(gf[e], pf[e], af[e], bf[e], cf[e], lr, alpha, l2adj, o);
    }
    // return section k's chunks to lanes 3k + q
    const int sec = c / 3, qq = c - 3 * sec;
    float4 out = p;
    if (S > 0) { const float4 t = shfl4(s0, qq, LPR); if (sec == 1) out = t; }
    if (S > 1) { const float4 t = shfl4(s1, qq, LPR); if (sec == 2) out = t; }
    if (S > 2) { const float4 t = shfl4(s2, qq, LPR); if (sec == 3) out = t; }
    if (ok && c < R4) st_f4(rec, out);
  }
}

// ---------------------------------------------------------------------------
// Dense kernels (kernel.go:27-32,58-66,99-116,163-169): whole-tensor update,
// optionally reducing R replica gradients first (sync-SGD averaging fused with
// the update).  param/slots are contiguous arrays on the owner shard.
// ---------------------------------------------------------------------------
struct ReplicaGrads {
  const float* g[kMaxShards];
  int n;
  float scale;
  int divide;  // 1: g = sum / scale (sync-SGD average, servicer.py:207); 0: g = sum * scale (allreduce postscale)
};

template <int OPT, int VEC, bool TWICE>
__device__ __forceinline__ void dense_update_range(const GroupView& gv, const TableView& tv,
                                                   const ReplicaGrads& rg, const OptParams& o) {
  constexpr int S = opt_slots(OPT);
  const int sh = tv.owner;
  const float lr = gv.rt->lr[sh], alpha = gv.rt->alpha[sh], l2adj = gv.rt->l2adj[sh];
  const long long numel = tv.rows * tv.dim;
  float* P = tv.base[sh];
  const long long nvec = numel / VEC;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float g[VEC], p[VEC], s0[VEC], s1[VEC], s2[VEC];
    if (VEC == 4) {
      float4 acc = ld_f4(rg.g[0] + 4 * i);
      for (int r = 1; r < rg.n; ++r) {
        float4 x = ld_f4(rg.g[r] + 4 * i);
        acc.x = add(acc.x, x.x); acc.y = add(acc.y, x.y); acc.z = add(acc.z, x.z); acc.w = add(acc.w, x.w);
      }
      g[0] = acc.x; g[1] = acc.y; g[2] = acc.z; g[3] = acc.w;
      *reinterpret_cast<float4*>(p) = *reinterpret_cast<const float4*>(P + 4 * i);
      if (S > 0) *reinterpret_cast<float4*>(s0) = *reinterpret_cast<const float4*>(P + tv.slot_off[1] + 4 * i);
      if (S > 1) *reinterpret_cast<float4*>(s1) = *reinterpret_cast<const float4*>(P + tv.slot_off[2] + 4 * i);
      if (S > 2) *reinterpret_cast<float4*>(s2) = *reinterpret_cast<const float4*>(P + tv.slot_off[3] + 4 * i);
    } else {
      float acc = rg.g[0][i];
      for (int r = 1; r < rg.n; ++r) acc = add(acc, rg.g[r][i]);
      g[0] = acc;
      p[0] = P[i];
      if (S > 0) s0[0] = P[tv.slot_off[1] + i];
      if (S > 1) s1[0] = P[tv.slot_off[2] + i];
      if (S > 2) s2[0] = P[tv.slot_off[3] + i];
    }
#pragma unroll
    for (int e = 0; e < VEC; ++e) {
      if (rg.divide) g[e] = fdiv(g[e], rg.scale);
      else if (rg.scale != 1.0f) g[e] = mul(g[e], rg.scale);
      opt_update<OPT>(g[e], p[e], s0[e], s1[e], s2[e], lr, alpha, l2adj, o);
      if (TWICE) {  // quirk Q1: dense AMSGrad falls through into plain Adam (optimizer.go:186-192)
        opt_update<kAdam>(g[e], p[e], s0[e], s1[e], s2[e], lr, alpha, l2adj, o);
      }
    }
    if (VEC == 4) {
      *reinterpret_cast<float4*>(P + 4 * i) = *reinterpret_cast<float4*>(p);
      if (S > 0) *reinterpret_cast<float4*>(P + tv.slot_off[1] + 4 * i) = *reinterpret_cast<float4*>(s0);
      if (S > 1) *reinterpret_cast<float4*>(P + tv.slot_off[2] + 4 * i) = *reinterpret_cast<float4*>(s1);
      if (S > 2) *reinterpret_cast<float4*>(P + tv.slot_off[3] + 4 * i) = *reinterpret_cast<float4*>(s2);
    } else {
      P[i] = p[0];
      if (S > 0) P[tv.slot_off[1] + i] = s0[0];
      if (S > 1) P[tv.slot_off[2] + i] = s1[0];
      if (S > 2) P[tv.slot_off[3] + i] = s2[0];
    }
  }
}

// One launch for all dense gradients of a push, whatever their sizes: a segment whose element count is a
// multiple of 4 and whose gradient is 16 B aligned takes the 128-bit path (block-uniform branch).
template <int OPT, bool TWICE>
__global__ void __launch_bounds__(256) k_push_dense(GroupView gv, SegBatch sb, OptParams o) {
  const b200ps_seg_t& sg = sb.seg[blockIdx.y];
  const TableView& tv = gv.tables[sg.table];
  ReplicaGrads rg;
  rg.g[0] = sg.rows_dev;
  rg.n = 1;
  rg.scale = 1.0f;
  rg.divide = 0;
  const bool vec = ((tv.rows * tv.dim) & 3) == 0 && ((uintptr_t)sg.rows_dev & 15u) == 0;
  if (vec) dense_update_range<OPT, 4, TWICE>(gv, tv, rg, o);
  else dense_update_range<OPT, 1, TWICE>(gv, tv, rg, o);
}

template <int OPT, int VEC, bool TWICE>
__global__ void __launch_bounds__(256) k_push_dense_reduce(GroupView gv, int table, ReplicaGrads rg, OptParams o) {
  dense_update_range<OPT, VEC, TWICE>(gv, gv.tables[table], rg, o);
}

// The reference's own C ABI (go/pkg/kernel/capi/kernel_api.h:10-37) on raw device arrays:
// grad / param / slot pointers + size, in place.
template <int OPT, int VEC>
__global__ void __launch_bounds__(256) k_raw_dense(const float* __restrict__ G, float* P, float* S0, float* S1, float* S2,
                                                   long long n, float lr, float alpha, float l2adj, OptParams o) {
  constexpr int S = opt_slots(OPT);
  const long long nvec = n / VEC;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += stride) {
    float g[VEC], p[VEC], s0[VEC], s1[VEC], s2[VEC];
    if (VEC == 4) {
      *reinterpret_cast<float4*>(g) = ld_f4(G + 4 * i);
      *reinterpret_cast<float4*>(p) = *reinterpret_cast<const float4*>(P + 4 * i);
      if (S > 0) *reinterpret_cast<float4*>(s0) = *reinterpret_cast<const float4*>(S0 + 4 * i);
      if (S > 1) *reinterpret_cast<float4*>(s1) = *reinterpret_cast<const float4*>(S1 + 4 * i);
      if (S > 2) *reinterpret_cast<float4*>(s2) = *reinterpret_cast<const float4*>(S2 + 4 * i);
    } else {
      g[0] = G[i]; p[0] = P[i];
      if (S > 0) s0[0] = S0[i];
      if (S > 1) s1[0] = S1[i];
      if (S > 2) s2[0] = S2[i];
    }
#pragma unroll
    for (int e = 0; e < VEC; ++e) opt_update<OPT>(g[e], p[e], s0[e], s1[e], s2[e], lr, alpha, l2adj, o);
    if (VEC == 4) {
      *reinterpret_cast<float4*>(P + 4 * i) = *reinterpret_cast<float4*>(p);
      if (S > 0) *reinterpret_cast<float4*>(S0 + 4 * i) = *reinterpret_cast<float4*>(s0);
      if (S > 1) *reinterpret_cast<float4*>(S1 + 4 * i) = *reinterpret_cast<float4*>(s1);
      if (S > 2) *reinterpret_cast<float4*>(S2 + 4 * i) = *reinterpret_cast<float4*>(s2);
    } else {
      P[i] = p[0];
      if (S > 0) S0[i] = s0[0];
      if (S > 1) S1[i] = s1[0];
      if (S > 2) S2[i] = s2[0];
    }
  }
}

// pull_dense / set_dense: whole-parameter copy owner shard <-> caller buffer.
template <bool WRITE>
__global__ void __launch_bounds__(256) k_dense_copy(GroupView gv, SegBatch sb, int slot) {
  const b200ps_seg_t& sg = sb.seg[blockIdx.y];
  const TableView& tv = gv.tables[sg.table];
  float* P = tv.base[tv.owner] + tv.slot_off[slot];
  float* U = sg.rows_dev;
  const long long numel = tv.rows * tv.dim;
  const bool vec = (numel & 3) == 0 && ((uintptr_t)U & 15u) == 0;  // block-uniform: one launch for all sizes
  const long long stride = (long long)gridDim.x * blockDim.x;
  if (vec) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel / 4; i += stride) {
      if (WRITE) st_f4(P + 4 * i, ld_f4(U + 4 * i)); else st_f4(U + 4 * i, ld_f4(P + 4 * i));
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < numel; i += stride) {
      if (WRITE) P[i] = U[i]; else U[i] = P[i];
    }
  }
}

// ---------------------------------------------------------------------------
// Push control (server.go:176-206, optimizer.go:43-44): one thread per shard.
// ---------------------------------------------------------------------------
struct VersionsIn {
  int v[kMaxShards];
};

__global__ void k_push_begin(GroupView gv, OptParams o, float learning_rate, VersionsIn mv,
                             int staleness_modulation, int bump_only, int only_shard) {
  int s = threadIdx.x;
  if (s >= gv.n_shards) return;
  if (only_shard >= 0 && s != only_shard) return;  // an ApplyGradients that reaches one shard only
  ShardCtl* ctl = gv.ctl[s];
  long long step = (long long)atomicAdd_system((unsigned long long*)&ctl->step, 1ULL) + 1;  // optimizer.go:44
  if (bump_only) return;
  int version = *(volatile int*)&ctl->version;
  float lr = 1.0f;
  if (staleness_modulation && version > mv.v[s]) lr = fdiv(lr, (float)(version - mv.v[s]));  // server.go:179-182
  if (learning_rate > 0.0f) lr = mul(lr, learning_rate); else lr = mul(lr, o.lr);          // server.go:183-187
  PushRt* rt = gv.rt;
  rt->lr[s] = lr;
  rt->step[s] = step;
  // kernel_api.cc:67: lr *= sqrt(1 - pow(beta2, step)) / (1 - pow(beta1, step)) in double
  double corr = sqrt(1.0 - pow((double)o.beta2, (double)step)) / (1.0 - pow((double)o.beta1, (double)step));
  rt->alpha[s] = (float)((double)lr * corr);
  rt->l2adj[s] = o.beta != 0.0f ? add(o.l2, fdiv(o.beta, mul(2.0f, lr))) : o.l2;
}

__global__ void k_push_end(GroupView gv, int* versions_out, int only_shard) {
  int s = threadIdx.x;
  if (s >= gv.n_shards) return;
  if (only_shard >= 0 && s != only_shard) {
    if (versions_out) versions_out[s] = *(volatile int*)&gv.ctl[s]->version;
    return;
  }
  int v = atomicAdd_system(&gv.ctl[s]->version, 1) + 1;  // server.go:196-199
  gv.rt->version[s] = v;
  if (versions_out) versions_out[s] = v;
}

__global__ void k_snapshot(GroupView gv, long long* out) {
  int s = threadIdx.x;
  if (s >= gv.n_shards) return;
  volatile ShardCtl* c = gv.ctl[s];
  out[3 * s + 0] = c->version;
  out[3 * s + 1] = c->step;
  out[3 * s + 2] = c->initialized == 1 ? 1 : 0;
}

// Device-side barrier of a rank-per-GPU group: every rank adds 1 to the counter in EVERY shard's control
// block (system-scope atomics over NVLink) and waits until its own counter shows all N arrivals of this
// epoch.  Kernels launched before it on the stream have completed (their writes are in the owner's L2,
// where peer reads are served), kernels after it see every peer's pre-barrier writes.  Bounded spin.
__global__ void k_group_barrier(GroupView gv, int me, unsigned* err) {
  __shared__ int s_epoch;
  if (threadIdx.x == 0) s_epoch = ++gv.ctl[me]->bar_epoch;
  __syncwarp();
  __threadfence_system();
  if ((int)threadIdx.x < gv.n_shards) atomicAdd_system(&gv.ctl[threadIdx.x]->bar_count, 1);
  if (threadIdx.x == 0) {
    const int target = s_epoch * gv.n_shards;
    long long spins = 0;
    while (*(volatile int*)&gv.ctl[me]->bar_count < target) {
      __nanosleep(100);
      if (++spins > (1LL << 24)) {
        atomicOr(err, 8u /* kErrTimeout */);
        break;
      }
    }
  }
  __threadfence_system();
}

// initialized: 0 = no, 2 = a writer holds the claim, 1 = yes (server.go:209-221)
__global__ void k_try_init(ShardCtl* ctl, int* won) {
  *won = atomicCAS_system(&ctl->initialized, 0, 2) == 0 ? 1 : 0;
}
__global__ void k_finish_init(ShardCtl* ctl, int version) {
  if (version >= 1) ctl->version = version;  // model.go:84-86
  __threadfence_system();
  atomicExch_system(&ctl->initialized, 1);
}

// ---------------------------------------------------------------------------
// Table initialisation on the owning shard: param = uniform(-0.05, 0.05) from
// the counter-based generator shared with the oracle (oracle_uniform_init) or
// zeros; slots = their constant.
// ---------------------------------------------------------------------------
__host__ __device__ __forceinline__ float uniform_init(uint64_t seed, int64_t id, int64_t col) {
  uint64_t h = mix64(seed ^ mix64((uint64_t)id * 0x9E3779B97F4A7C15ULL + (uint64_t)col));
  float u = (float)(h >> 40) * (1.0f / 16777216.0f);
#ifdef __CUDA_ARCH__
  return __fadd_rn(__fmul_rn(u, 0.1f), -0.05f);  // initializer.go:116
#else
  return u * 0.1f + (-0.05f);
#endif
}

struct InitArgs {
  float* base;
  long long rows, row_stride;
  long long slot_off[kMaxSlots + 1];
  float slot_init[kMaxSlots + 1];
  int dim, n_slots, uniform, shard, n_shards, is_dense;
  unsigned long long seed;
};

__global__ void __launch_bounds__(256) k_init_rows(InitArgs a) {
  const long long per_row = (long long)a.dim * (a.n_slots + 1);
  const long long work = a.rows * per_row;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < work; w += stride) {
    long long row = w / per_row;
    int r = (int)(w - row * per_row);
    int k = r / a.dim, c = r - k * a.dim;
    float v = a.slot_init[k];
    if (k == 0 && a.uniform) {
      long long id = a.is_dense ? row : row * a.n_shards + a.shard;
      v = uniform_init(a.seed, id, c);
    }
    a.base[row * a.row_stride + a.slot_off[k] + c] = v;
  }
}

__global__ void __launch_bounds__(256) k_fill_keys(long long* keys, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) keys[i] = kEmptySlot;
}

__global__ void __launch_bounds__(256) k_key_ids(const long long* keys, long long rows, int64_t* ids, long long cap,
                                                 unsigned long long* count) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long slot = (long long)blockIdx.x * blockDim.x + threadIdx.x; slot < rows; slot += stride) {
    const long long k = keys[slot];
    if (k != kEmptySlot) {
      unsigned long long at = atomicAdd(count, 1ULL);
      if (ids != nullptr && (long long)at < cap) ids[at] = k;
    }
  }
}

// Created-row ids of one table shard (ToIndexedSlices key walk, embedding_table.go:80-88).
__global__ void __launch_bounds__(256) k_present_ids(const uint32_t* present, long long rows, int shard,
                                                     int n_shards, int64_t* ids, long long cap,
                                                     unsigned long long* count) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long slot = (long long)blockIdx.x * blockDim.x + threadIdx.x; slot < rows; slot += stride) {
    if (present[slot >> 5] >> (slot & 31) & 1u) {
      unsigned long long at = atomicAdd(count, 1ULL);
      if (ids != nullptr && (long long)at < cap) ids[at] = slot * n_shards + shard;
    }
  }
}

// ---------------------------------------------------------------------------
// segment_sum: out[t][inv[i], :] += values[t][i, :]   (deduplicate_indexed_slices'
// sum / gather backward).  Warp-level id dedup: lanes of a warp that hit the
// same output row combine through shuffles (lane order) and the lowest lane
// issues ONE vector reduction to global memory.
// ---------------------------------------------------------------------------
template <int VPT>
__global__ void __launch_bounds__(256) k_segment_sum(const float* values, const int* inv, long long k, int dim,
                                                     float* out) {
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  const int t = blockIdx.y;
  const int chunks = dim / W;
  const long long work = k * chunks;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const float* V = values + (long long)t * k * dim;
  float* O = out + (long long)t * k * dim;
  const int* I = inv + (long long)t * k;
  const long long wmax = (work + 31) / 32 * 32;  // keep warps converged for the shuffles
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < wmax; w += stride) {
    const bool live = w < work;
    const long long row = live ? (chunks == 1 ? w : w / chunks) : 0;
    const int c = live ? (int)(w - row * chunks) : 0;
    const int dst = live ? I[row] : -1;
    float x[W];
    if (live) {
      if (VPT == 0) x[0] = V[row * dim + c];
      else {
#pragma unroll
        for (int v = 0; v < VPT; ++v) *reinterpret_cast<float4*>(&x[4 * v]) = ld_f4(V + row * dim + c * W + 4 * v);
      }
    } else {
#pragma unroll
      for (int e = 0; e < W; ++e) x[e] = 0.f;
    }
    // dst * chunks + c < k * chunks <= INT32_MAX (b200ps_segment_sum refuses more): no live key wraps onto another
    const int key = live ? dst * chunks + c : -1 - (int)(threadIdx.x & 31);
    const unsigned peers = __match_any_sync(0xffffffffu, key);
    const int lane = threadIdx.x & 31;
    const bool leader = (__ffs(peers) - 1) == lane;
    unsigned rest = peers & ~(1u << lane);
    const int maxn = __reduce_max_sync(0xffffffffu, (unsigned)__popc(peers));
    for (int j = 1; j < maxn; ++j) {
      int src = rest ? __ffs(rest) - 1 : lane;
#pragma unroll
      for (int e = 0; e < W; ++e) {
        float y = __shfl_sync(0xffffffffu, x[e], src);
        if (leader && rest) x[e] = add(x[e], y);
      }
      rest &= rest - 1;
    }
    if (live && leader) {
      float* o = O + (long long)dst * dim + c * W;
      if (VPT == 0) atomicAdd(o, x[0]);
      else {
#pragma unroll
        for (int v = 0; v < VPT; ++v) atomicAdd(reinterpret_cast<float4*>(o + 4 * v), *reinterpret_cast<float4*>(&x[4 * v]));
      }
    }
  }
}

// gather_rows: out[t][i, :] = bet[t][inv[i], :]  (tf.gather(batch_embedding, idx),
// embedding_delegate.py:95)
template <int VPT>
__global__ void __launch_bounds__(256) k_gather_rows(const float* bet, const int* inv, long long k, int dim,
                                                     float* out) {
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  const int t = blockIdx.y;
  const int chunks = dim / W;
  const long long work = k * chunks;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const float* Bt = bet + (long long)t * k * dim;
  float* O = out + (long long)t * k * dim;
  const int* I = inv + (long long)t * k;
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < work; w += stride) {
    const long long row = chunks == 1 ? w : w / chunks;
    const int c = chunks == 1 ? 0 : (int)(w - row * chunks);
    const float* src = Bt + (long long)I[row] * dim + c * W;
    float* dst = O + row * dim + c * W;
    if (VPT == 0) *dst = *src;
    else {
#pragma unroll
      for (int v = 0; v < VPT; ++v) st_f4(dst + 4 * v, *reinterpret_cast<const float4*>(src + 4 * v));
    }
  }
}

__global__ void __launch_bounds__(256) k_zero(float* p, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = 0.f;
}

}  // namespace b200ps_impl
