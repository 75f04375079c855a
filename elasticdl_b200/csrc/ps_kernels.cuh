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
  static_assert(OPT >= 0 && OPT < kNumOptKinds, "opt_update: unknown optimizer kind");
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
  } else if (OPT == kRMSprop || OPT == kRMSpropMomentum || OPT == kRMSpropCentered ||
             OPT == kRMSpropCenteredMomentum) {
    // Keras RMSprop, sparse form; slots rms[, momentum][, mg].  momentum = 0: eps outside the square
    // root (Keras' python ops); momentum > 0: TF SparseApply[Centered]RMSProp, eps inside it (Q13).
    constexpr bool MOM = OPT == kRMSpropMomentum || OPT == kRMSpropCenteredMomentum;
    constexpr bool CEN = OPT == kRMSpropCentered || OPT == kRMSpropCenteredMomentum;
    float rms = add(mul(o.beta1, s0), mul(o.c1, mul(g, g)));
    s0 = rms;
    float den = rms;
    if (CEN) {
      float& mg_slot = MOM ? s2 : s1;
      float mg = add(mul(o.beta1, mg_slot), mul(o.c1, g));
      mg_slot = mg;
      den = sub(rms, mul(mg, mg));
    }
    if (MOM) {
      float mom = add(mul(o.mu, s1), fdiv(mul(lr, g), fsqrt(add(den, o.epsilon))));
      s1 = mom;
      p = sub(p, mom);
    } else {
      p = sub(p, fdiv(mul(lr, g), add(fsqrt(den), o.epsilon)));
    }
  } else if (OPT == kAdadelta) {  // TF SparseApplyAdadelta; slots accum_grad, accum_var
    float ag = add(mul(o.beta1, s0), mul(o.c1, mul(g, g)));
    s0 = ag;
    float u = mul(fdiv(fsqrt(add(s1, o.epsilon)), fsqrt(add(ag, o.epsilon))), g);
    p = sub(p, mul(lr, u));
    s1 = add(mul(o.beta1, s1), mul(o.c1, mul(u, u)));
  } else if (OPT == kAdamax) {  // Keras Adamax._resource_apply_sparse; alpha = lr/(1-b1^t)
    float m = add(mul(o.beta1, s0), mul(o.c1, g));
    float v = fmaxf(mul(o.beta2, s1), fabsf(g));
    s0 = m;
    s1 = v;
    p = sub(p, fdiv(mul(alpha, m), add(v, o.epsilon)));
  } else if (OPT == kNadam) {  // Keras Nadam with its per-push scalars folded (nadam_coefs)
    float m = add(mul(o.beta1, s0), mul(o.c1, g));
    float v = add(mul(o.beta2, s1), mul(o.c2, mul(g, g)));
    s0 = m;
    s1 = v;
    p = sub(p, fdiv(add(mul(lr, g), mul(alpha, m)), add(fsqrt(v), l2adj)));
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
  // TORCH only: the caller's copy of the parameter (read instead of the PS copy, which is written), and this
  // step's Adam coefficients from the double hyper-parameters, as torch.optim.Adam has them
  const float* param;
  float alpha, eps, c1, c2;
};

// TORCH (the dense allreduce of a torch optimizer): the parameter is read from rg.param, and Adam's alpha, eps
// and (1 - beta) come from rg.  Off, the update is kernel_api.cc's: coefficients from k_push_begin and the
// fp32 betas.
template <int OPT, int VEC, bool TWICE, bool TORCH = false>
__device__ __forceinline__ void dense_update_range(const GroupView& gv, const TableView& tv,
                                                   const ReplicaGrads& rg, const OptParams& o_in) {
  constexpr int S = opt_slots(OPT);
  const int sh = tv.owner;
  const float lr = gv.rt->lr[sh], alpha = TORCH ? rg.alpha : gv.rt->alpha[sh], l2adj = gv.rt->l2adj[sh];
  OptParams o = o_in;
  if (TORCH) {
    o.epsilon = rg.eps;
    o.c1 = rg.c1;
    o.c2 = rg.c2;
  }
  const long long numel = tv.rows * tv.dim;
  float* P = tv.base[sh];
  const float* Pin = TORCH ? rg.param : P;
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
      *reinterpret_cast<float4*>(p) = *reinterpret_cast<const float4*>(Pin + 4 * i);
      if (S > 0) *reinterpret_cast<float4*>(s0) = *reinterpret_cast<const float4*>(P + tv.slot_off[1] + 4 * i);
      if (S > 1) *reinterpret_cast<float4*>(s1) = *reinterpret_cast<const float4*>(P + tv.slot_off[2] + 4 * i);
      if (S > 2) *reinterpret_cast<float4*>(s2) = *reinterpret_cast<const float4*>(P + tv.slot_off[3] + 4 * i);
    } else {
      float acc = rg.g[0][i];
      for (int r = 1; r < rg.n; ++r) acc = add(acc, rg.g[r][i]);
      g[0] = acc;
      p[0] = Pin[i];
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

template <int OPT, int VEC, bool TWICE, bool TORCH>
__global__ void __launch_bounds__(256) k_push_dense_reduce(GroupView gv, int table, ReplicaGrads rg, OptParams o) {
  dense_update_range<OPT, VEC, TWICE, TORCH>(gv, gv.tables[table], rg, o);
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
// Keras Nadam's momentum cache u_t = beta_1 * (1 - 0.5 * 0.96^(0.004 t)), in double, rounded to float32
// (the float32 value Keras multiplies into its schedule).
__host__ __device__ __forceinline__ float nadam_u(float beta1, long long t) {
  return (float)((double)beta1 * (1.0 - 0.5 * pow(0.96, 0.004 * (double)t)));
}

// Nadam's per-push scalars at step t, folded into the three words every row kernel takes:
//   p -= lr * mbar / (sqrt(v / (1 - b2^t)) + eps),  mbar = (1 - u_t) g / (1 - S_t) + u_{t+1} m / (1 - S_{t+1})
// is, multiplied through by sqrt(1 - b2^t),
//   p -= (cg * g + cm * m) / (sqrt(v) + ce),  cg = lr (1 - u_t) sqrt(1 - b2^t) / (1 - S_t),
//                                            cm = lr u_{t+1} sqrt(1 - b2^t) / (1 - S_{t+1}),  ce = eps sqrt(1 - b2^t).
// S_{t+1} = S_t * u_{t+1} is Keras' m_schedule_next.  Each scalar is formed in double and rounded once.
// sched: S_t for t = 0..last (b200ps.cu nadam_schedule); S_t = sched[min(t, last)].
__device__ __forceinline__ void nadam_coefs(const OptParams& o, const float* sched, long long last, float lr, long long t,
                                            float* cg, float* cm, float* ce) {
  const double ut = nadam_u(o.beta1, t), ut1 = nadam_u(o.beta1, t + 1);
  const double st = sched[t < last ? t : last];
  const double st1 = sched[t + 1 < last ? t + 1 : last];
  const double sb = sqrt(1.0 - pow((double)o.beta2, (double)t));
  *cg = (float)((double)lr * (1.0 - ut) * sb / (1.0 - st));
  *cm = (float)((double)lr * ut1 * sb / (1.0 - st1));
  *ce = (float)((double)o.epsilon * sb);
}

struct VersionsIn {
  int v[kMaxShards];
};

__global__ void k_push_begin(GroupView gv, OptParams o, float learning_rate, VersionsIn mv,
                             int staleness_modulation, int bump_only, int only_shard, const float* nadam_sched,
                             long long nadam_last) {
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
  if (o.kind == kNadam) {
    nadam_coefs(o, nadam_sched, nadam_last, lr, step, &rt->lr[s], &rt->alpha[s], &rt->l2adj[s]);
    return;
  }
  if (o.kind == kAdamax) {  // Keras Adamax: lr_t = lr / (1 - beta_1^t), power in double, rounded once
    rt->alpha[s] = (float)((double)lr / (1.0 - pow((double)o.beta1, (double)step)));
  } else {
    // kernel_api.cc:67: lr *= sqrt(1 - pow(beta2, step)) / (1 - pow(beta1, step)) in double
    double corr = sqrt(1.0 - pow((double)o.beta2, (double)step)) / (1.0 - pow((double)o.beta1, (double)step));
    rt->alpha[s] = (float)((double)lr * corr);
  }
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
// The row source of a segment sum: LOAD.live(row) says whether entry `row` contributes, LOAD.load(row, c, x) reads
// its W floats of chunk c.
template <int VPT>
struct RowsLoad {  // values[row, :]
  const float* V;
  int dim;
  __device__ __forceinline__ bool live(long long) const { return true; }
  __device__ __forceinline__ void load(long long row, int c, float* x) const {
    constexpr int W = VPT == 0 ? 1 : 4 * VPT;
    if (VPT == 0) x[0] = V[row * dim + c];
    else {
#pragma unroll
      for (int v = 0; v < VPT; ++v) *reinterpret_cast<float4*>(&x[4 * v]) = ld_f4(V + row * dim + c * W + 4 * v);
    }
  }
};

template <int VPT, class LOAD>
__device__ __forceinline__ void segment_sum_loop(const LOAD& ld, const int* I, long long k, int dim, float* O) {
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  const int chunks = dim / W;
  const long long work = k * chunks;
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long wmax = (work + 31) / 32 * 32;  // keep warps converged for the shuffles
  for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < wmax; w += stride) {
    const bool in = w < work;
    const long long row = in ? (chunks == 1 ? w : w / chunks) : 0;
    const bool live = in && ld.live(row);
    const int c = live ? (int)(w - row * chunks) : 0;
    const int dst = live ? I[row] : -1;
    float x[W];
    if (live) {
      ld.load(row, c, x);
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

template <int VPT>
__global__ void __launch_bounds__(256) k_segment_sum(const float* values, const int* inv, long long k, int dim,
                                                     float* out) {
  const int t = blockIdx.y;
  const RowsLoad<VPT> ld{values + (long long)t * k * dim, dim};
  segment_sum_loop<VPT>(ld, inv + (long long)t * k, k, dim, out + (long long)t * k * dim);
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

// ---------------------------------------------------------------------------
// Pooled lookup of a sparse [B, L] input (safe_embedding_lookup_sparse without weights,
// embedding_delegate.py:108-230): prune ids < 0, give each empty row the id 0, combine per row
// (sum / mean / sqrtn), write 0 for the rows that were empty.
//
// Workspace (int32 words, offsets from SparseLayout; n = nnz, K = nnz + B filled entries):
//   bad[4]      entries whose row lies outside [0, B) (dropped)
//   cnt[B]      kept ids per row
//   off[B+1]    CSR offsets of the filled stream, off[b] = sum_{r<b} max(cnt[r], 1)
//   ebef[B]     empty rows before row b
//   poff[B+1]   piece offsets: row b is combined in np_b = ceil(max(cnt, 1) / kSpPiece) pieces
//   moff[B+1]   partial-sum slots of the rows with np_b > 1
//   arrive[B]   pieces of row b that have finished (forward of a multi-piece row)
//   prow[PB]    row of each piece
//   tkept[NT], tbase[NT], tlast[NT]   per input tile: kept entries, kept entries before it, last kept index
//   last[2]     the last filled id (int64), copied into the tail [off[B], K)
//   rowf[K]     row of each filled entry, -1 for the fill of an empty row and for the tail
//   part[MB*dim] float partial sums of multi-piece rows
// ---------------------------------------------------------------------------
constexpr int kSpPiece = 256;  // filled entries one warp sums before a row is split across warps
constexpr int kSpTile = 1024;  // input entries per block and tile of the prep's count and scatter passes
constexpr int kSpScanThreads = 1024;

enum { kSpSum = 0, kSpMean = 1, kSpSqrtn = 2 };

struct SparseLayout {
  long long B, nnz, K, PB, MB, NT;
  long long cnt, off, ebef, poff, moff, arrive, prow, tkept, tbase, tlast, last, rowf, part, words;
  __host__ __device__ static long long up4(long long x) { return (x + 3) / 4 * 4; }
  __host__ __device__ SparseLayout(long long B_, long long nnz_, int dim) : B(B_), nnz(nnz_) {
    K = nnz + B;
    PB = B + K / kSpPiece + 1;      // sum_b ceil(len_b / P) <= K / P + B
    MB = 2 * (K / kSpPiece) + 1;    // a row with np > 1 has len > P, so np < 2 len / P
    NT = (nnz + kSpTile - 1) / kSpTile;
    cnt = 4;
    off = up4(cnt + B);
    ebef = up4(off + B + 1);
    poff = up4(ebef + B);
    moff = up4(poff + B + 1);
    arrive = up4(moff + B + 1);
    prow = up4(arrive + B);
    tkept = up4(prow + PB);
    tbase = up4(tkept + NT);
    tlast = up4(tbase + NT);
    last = up4(tlast + NT);
    rowf = up4(last + 2);
    part = up4(rowf + K);
    words = up4(part + MB * (long long)dim);
  }
};

__device__ __forceinline__ int sp_pieces(int cnt) { return ((cnt > 1 ? cnt : 1) + kSpPiece - 1) / kSpPiece; }

// Pass 1: count kept ids per row (warp-aggregated atomics: a coalesced input is row-major), kept entries and the
// last kept index per tile; report rows outside [0, B).
template <typename V>
__global__ void __launch_bounds__(256) k_sparse_count(const long long* rows, const V* vals, SparseLayout L, int* ws) {
  int* cnt = ws + L.cnt;
  __shared__ int s_kept, s_last;
  const int lane = threadIdx.x & 31;
  for (long long t = blockIdx.x; t < L.NT; t += gridDim.x) {
    if (threadIdx.x == 0) { s_kept = 0; s_last = -1; }
    __syncthreads();
    int kept = 0, last = -1, bad = 0;
    for (int q = 0; q < kSpTile / 256; ++q) {
      const long long i = t * kSpTile + q * 256 + threadIdx.x;
      long long r = -1;
      bool keep = false;
      if (i < L.nnz) {
        r = rows[i];
        const bool rok = r >= 0 && r < L.B;
        bad += !rok;
        keep = rok && (long long)vals[i] >= 0;
      }
      const unsigned km = __ballot_sync(0xffffffffu, keep);
      const unsigned peers = __match_any_sync(0xffffffffu, keep ? r : -1LL) & km;
      if (keep && (__ffs(peers) - 1) == lane) atomicAdd(cnt + r, __popc(peers));
      kept += keep;
      if (keep) last = (int)i;
    }
    kept = __reduce_add_sync(0xffffffffu, kept);
    last = (int)__reduce_max_sync(0xffffffffu, (unsigned)(last + 1)) - 1;
    bad = __reduce_add_sync(0xffffffffu, bad);
    if (lane == 0) {
      atomicAdd(&s_kept, kept);
      atomicMax(&s_last, last);
      if (bad) atomicAdd(ws, bad);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      ws[L.tkept + t] = s_kept;
      ws[L.tlast + t] = s_last;
    }
    __syncthreads();
  }
}

// Block-wide exclusive scan of int4 (one value per thread, kSpScanThreads threads) and the block total.
struct SpScan {
  int4 excl, tot;
};
__device__ __forceinline__ SpScan sp_block_scan(int4 v) {
  __shared__ int4 s_w[kSpScanThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int4 x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int a = __shfl_up_sync(0xffffffffu, x.x, o), b = __shfl_up_sync(0xffffffffu, x.y, o);
    const int c = __shfl_up_sync(0xffffffffu, x.z, o), d = __shfl_up_sync(0xffffffffu, x.w, o);
    if (lane >= o) { x.x += a; x.y += b; x.z += c; x.w += d; }
  }
  if (lane == 31) s_w[warp] = x;
  __syncthreads();
  if (warp == 0) {
    int4 y = lane < kSpScanThreads / 32 ? s_w[lane] : make_int4(0, 0, 0, 0);
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a = __shfl_up_sync(0xffffffffu, y.x, o), b = __shfl_up_sync(0xffffffffu, y.y, o);
      const int c = __shfl_up_sync(0xffffffffu, y.z, o), d = __shfl_up_sync(0xffffffffu, y.w, o);
      if (lane >= o) { y.x += a; y.y += b; y.z += c; y.w += d; }
    }
    if (lane < kSpScanThreads / 32) s_w[lane] = y;  // inclusive warp totals
  }
  __syncthreads();
  const int4 wb = warp ? s_w[warp - 1] : make_int4(0, 0, 0, 0);
  const int4 tot = s_w[kSpScanThreads / 32 - 1];
  __syncthreads();
  return SpScan{make_int4(wb.x + x.x - v.x, wb.y + x.y - v.y, wb.z + x.z - v.z, wb.w + x.w - v.w), tot};
}

// Pass 2 (one block): the per-row offsets (off, ebef, poff, moff), the arrival counters, the tiles' kept bases and
// the last filled id.  Each thread scans a contiguous run of rows.
template <typename V>
__global__ void __launch_bounds__(kSpScanThreads) k_sparse_scan(const V* vals, SparseLayout L, int* ws) {
  const int* cnt = ws + L.cnt;
  const long long per = (L.B + kSpScanThreads - 1) / kSpScanThreads;
  const long long b0 = threadIdx.x * per, b1 = b0 + per < L.B ? b0 + per : L.B;
  int4 s = make_int4(0, 0, 0, 0);  // filled length, empty rows, pieces, multi-piece slots
  for (long long b = b0; b < b1; ++b) {
    const int c = cnt[b], np = sp_pieces(c);
    s.x += c > 1 ? c : 1; s.y += c == 0; s.z += np; s.w += np > 1 ? np : 0;
  }
  const SpScan sc = sp_block_scan(s);
  int4 e = sc.excl;
  const int4 tot = sc.tot;
  for (long long b = b0; b < b1; ++b) {
    const int c = cnt[b], np = sp_pieces(c);
    ws[L.off + b] = e.x; ws[L.ebef + b] = e.y; ws[L.poff + b] = e.z; ws[L.moff + b] = e.w;
    ws[L.arrive + b] = 0;
    e.x += c > 1 ? c : 1; e.y += c == 0; e.z += np; e.w += np > 1 ? np : 0;
  }
  if (threadIdx.x == 0) {
    ws[L.off + L.B] = tot.x; ws[L.poff + L.B] = tot.z; ws[L.moff + L.B] = tot.w;
  }
  // tiles: exclusive scan of the kept counts; the last kept index overall
  int base = 0, last = -1;
  for (long long t0 = 0; t0 < L.NT; t0 += kSpScanThreads) {
    const long long t = t0 + threadIdx.x;
    const int k = t < L.NT ? ws[L.tkept + t] : 0;
    if (t < L.NT && ws[L.tlast + t] > last) last = ws[L.tlast + t];
    const SpScan sc = sp_block_scan(make_int4(k, 0, 0, 0));
    if (t < L.NT) ws[L.tbase + t] = base + sc.excl.x;
    base += sc.tot.x;
  }
  last = (int)__reduce_max_sync(0xffffffffu, (unsigned)(last + 1)) - 1;
  __shared__ int s_last;
  if (threadIdx.x == 0) s_last = -1;
  __syncthreads();
  if ((threadIdx.x & 31) == 0) atomicMax(&s_last, last);
  __syncthreads();
  if (threadIdx.x == 0) {
    // the last filled entry is row B-1's: its fill id 0 when empty, else the last kept id of the input
    const long long id = cnt[L.B - 1] == 0 ? 0 : (long long)vals[s_last];
    *reinterpret_cast<long long*>(ws + L.last) = id;
  }
}

// Pass 3: scatter the kept ids to their filled positions (tile-local rank in entry order), the fill id 0 of each
// empty row, the row of every piece, and the tail copies of the last filled id.
template <typename V>
__global__ void __launch_bounds__(256) k_sparse_scatter(const long long* rows, const V* vals, SparseLayout L, int* ws,
                                                        long long* ids_f) {
  __shared__ int s_w[8];
  const int* cnt = ws + L.cnt;
  int* rowf = ws + L.rowf;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long t = blockIdx.x; t < L.NT; t += gridDim.x) {
    int base = ws[L.tbase + t];
    for (int q = 0; q < kSpTile / 256; ++q) {
      const long long i = t * kSpTile + q * 256 + threadIdx.x;
      long long r = -1;
      long long v = -1;
      if (i < L.nnz) {
        r = rows[i];
        v = (long long)vals[i];
      }
      const bool keep = r >= 0 && r < L.B && v >= 0;
      const unsigned km = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) s_w[warp] = __popc(km);
      __syncthreads();
      int wb = 0, tot = 0;
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        wb += u < warp ? s_w[u] : 0;
        tot += s_w[u];
      }
      if (keep) {
        const long long pos = base + wb + __popc(km & ((1u << lane) - 1)) + ws[L.ebef + r];
        ids_f[pos] = v;
        rowf[pos] = (int)r;
      }
      base += tot;
      __syncthreads();
    }
  }
  const long long stride = (long long)gridDim.x * blockDim.x;
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  for (long long b = g; b < L.B; b += stride) {
    const int c = cnt[b], o = ws[L.off + b], po = ws[L.poff + b], np = sp_pieces(c);
    if (c == 0) {
      ids_f[o] = 0;
      rowf[o] = -1;
    }
    for (int p = 0; p < np; ++p) ws[L.prow + po + p] = (int)b;
  }
  const long long kf = ws[L.off + L.B];
  const long long last = *reinterpret_cast<const long long*>(ws + L.last);
  for (long long j = kf + g; j < L.K; j += stride) {
    ids_f[j] = last;
    rowf[j] = -1;
  }
}

template <int VPT>
__device__ __forceinline__ void sp_scale_store(float* o, const float* x, int cnt, int combiner) {
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  float y[W];
  const float d = combiner == kSpMean ? (float)cnt : fsqrt((float)cnt);
#pragma unroll
  for (int e = 0; e < W; ++e) y[e] = cnt == 0 ? 0.f : combiner == kSpSum ? x[e] : fdiv(x[e], d);
  if (VPT == 0) o[0] = y[0];
  else {
#pragma unroll
    for (int v = 0; v < VPT; ++v) st_f4(o + 4 * v, *reinterpret_cast<float4*>(&y[4 * v]));
  }
}

// Combine forward: one warp per piece (<= kSpPiece filled entries of one row).  Lanes split as (entry slot, column
// chunk): CL lanes cover CL chunks of W floats, E = 32 / CL entries are read at once; each lane sums its entries in
// entry order, then the lanes of one chunk add through a fixed xor butterfly.  A row of one piece is scaled and
// stored; the pieces of a longer row store partials and the last piece to finish adds them in piece order and resets
// the row's arrival counter, so the combine can run again on the same workspace.  Every order is fixed, so two calls
// give the same bits; it is not strict entry order (see b200ps_sparse_combine).
template <int VPT>
__global__ void __launch_bounds__(256) k_sparse_combine(const float* __restrict__ bet, const int* __restrict__ inv,
                                                        SparseLayout L, int* ws, int dim, int combiner, float* out) {
  constexpr int W = VPT == 0 ? 1 : 4 * VPT;
  const int chunks = dim / W;
  int CL = 1;
  while (CL < chunks && CL < 32) CL <<= 1;
  const int E = 32 / CL;
  const int lane = threadIdx.x & 31;
  const int* off = ws + L.off;
  float* part = reinterpret_cast<float*>(ws + L.part);
  const long long npieces = ws[L.poff + L.B];
  const long long nwarps = (long long)gridDim.x * blockDim.x / 32;
  for (long long w = ((long long)blockIdx.x * blockDim.x + threadIdx.x) / 32; w < npieces; w += nwarps) {
    const int row = ws[L.prow + w];
    const int po = ws[L.poff + row], np = ws[L.poff + row + 1] - po, p = (int)(w - po);
    const int cnt = ws[L.cnt + row];
    const int s = off[row] + p * kSpPiece, e_end = min(s + kSpPiece, off[row + 1]);
    for (int cb = 0; cb < chunks; cb += CL) {
      const int c = cb + (lane & (CL - 1));
      const bool cok = c < chunks;
      float acc[W];
#pragma unroll
      for (int e = 0; e < W; ++e) acc[e] = 0.f;
      if (cok) {
        for (int j = s + lane / CL; j < e_end; j += E) {
          const float* src = bet + (long long)inv[j] * dim + c * W;
          if (VPT == 0) acc[0] = add(acc[0], __ldg(src));
          else {
#pragma unroll
            for (int v = 0; v < VPT; ++v) {
              const float4 x = __ldg(reinterpret_cast<const float4*>(src + 4 * v));
              acc[4 * v] = add(acc[4 * v], x.x); acc[4 * v + 1] = add(acc[4 * v + 1], x.y);
              acc[4 * v + 2] = add(acc[4 * v + 2], x.z); acc[4 * v + 3] = add(acc[4 * v + 3], x.w);
            }
          }
        }
      }
      for (int o = CL; o < 32; o <<= 1) {
#pragma unroll
        for (int e = 0; e < W; ++e) acc[e] = add(acc[e], __shfl_xor_sync(0xffffffffu, acc[e], o));
      }
      if (cok && lane < CL) {
        if (np == 1) sp_scale_store<VPT>(out + (long long)row * dim + c * W, acc, cnt, combiner);
        else {
          float* dst = part + ((long long)ws[L.moff + row] + p) * dim + c * W;
#pragma unroll
          for (int e = 0; e < W; ++e) dst[e] = acc[e];
        }
      }
    }
    if (np > 1) {
      __threadfence();
      __syncwarp();
      int done = 0;
      if (lane == 0) done = atomicAdd(ws + L.arrive + row, 1) == np - 1;
      done = __shfl_sync(0xffffffffu, done, 0);
      if (done) {
        __threadfence();
        if (lane == 0) ws[L.arrive + row] = 0;  // all np pieces have arrived: nothing else touches the counter
        const float* P = part + (long long)ws[L.moff + row] * dim;
        for (int c = lane; c < chunks; c += 32) {
          float acc[W];
#pragma unroll
          for (int e = 0; e < W; ++e) acc[e] = 0.f;
          for (int q = 0; q < np; ++q) {
#pragma unroll
            for (int e = 0; e < W; ++e) acc[e] = add(acc[e], __ldcg(P + (long long)q * dim + c * W + e));
          }
          sp_scale_store<VPT>(out + (long long)row * dim + c * W, acc, cnt, combiner);
        }
      }
    }
  }
}

// Combine backward load: entry j of the filled stream contributes s_row * gout[row, :] when it belongs to a non-empty
// row (rowf >= 0); the division is the one torch's autograd of out / counts (out / counts.sqrt()) performs.
template <int VPT>
struct SparseGradLoad {
  const float* G;
  const int* rowf;
  const int* cnt;
  int dim, combiner;
  __device__ __forceinline__ bool live(long long j) const { return rowf[j] >= 0; }
  __device__ __forceinline__ void load(long long j, int c, float* x) const {
    const int r = rowf[j];
    RowsLoad<VPT>{G, dim}.load(r, c, x);
    if (combiner != kSpSum) {
      constexpr int W = VPT == 0 ? 1 : 4 * VPT;
      const int n = cnt[r];
      const float d = combiner == kSpMean ? (float)n : fsqrt((float)n);
#pragma unroll
      for (int e = 0; e < W; ++e) x[e] = fdiv(x[e], d);
    }
  }
};

template <int VPT>
__global__ void __launch_bounds__(256) k_sparse_combine_grad(const float* gout, const int* inv, SparseLayout L,
                                                             const int* ws, int dim, int combiner, float* gbet) {
  const SparseGradLoad<VPT> ld{gout, ws + L.rowf, ws + L.cnt, dim, combiner};
  segment_sum_loop<VPT>(ld, inv, L.K, dim, gbet);
}

}  // namespace b200ps_impl
