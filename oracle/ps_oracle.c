/*
 * ps_oracle.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of the ElasticDL Go parameter-server data path, used only as
 * the parity checker (tests/, __graft_entry__.smoke()) and as the timed CPU
 * baseline (bench.py cpu_baseline / --impl reference).  Nothing under
 * elasticdl_b200/ may import, link or call this file.
 *
 * The reference's own native file (elasticdl/go/pkg/kernel/capi/kernel_api.cc)
 * includes <eigen3/Eigen/Dense> (kernel_api.cc:4) and Eigen is not in this
 * image; oracle/Makefile `ref` compiles it UNMODIFIED against a stand-in header
 * (oracle/eigen_shim) into oracle/_ref/libkernel_api_ref.so, and
 * tests/test_oracle_vs_ref.py checks that the dense kernels below agree with it
 * bit for bit (live, and through tests/golden/ref_kernel_vectors.npz which that
 * library produced).  The Go PS around the kernels needs go/protoc/grpc, absent
 * here, so the row loops, tables and control logic stay a restatement in plain
 * C with the same operation order, compiled -O3 -ffp-contract=off (the
 * reference is built `g++ -O3 -std=c++11` without -march,
 * elasticdl/Makefile:23-25, i.e. SSE2 and no FMA contraction), pinned by the
 * reference's golden vectors, see tests/test_oracle_golden.py.
 *
 * Every function cites the reference file:line it follows (paths relative to
 * /root/reference/elasticdl/).
 */
#define _GNU_SOURCE
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

/* ------------------------------------------------------------------ */
/* Dense kernels: go/pkg/kernel/capi/kernel_api.cc                     */
/* ------------------------------------------------------------------ */

/* kernel_api.cc:6-14   ep -= lr * eg */
void oracle_sgd(const float* grad, float* param, float lr, long long size) {
  for (long long i = 0; i < size; ++i) param[i] = param[i] - lr * grad[i];
}

/* kernel_api.cc:16-38  ev = mu*ev + eg ; nesterov ? ep -= lr*(eg + mu*ev)
 *                                                 : ep -= lr*ev */
void oracle_momentum(const float* grad, float* param, float* velocity,
                     float mu, int nesterov, float lr, long long size) {
  for (long long i = 0; i < size; ++i) {
    float v = mu * velocity[i] + grad[i];
    velocity[i] = v;
    if (nesterov)
      param[i] = param[i] - lr * (grad[i] + mu * v);
    else
      param[i] = param[i] - lr * v;
  }
}

/* kernel_api.cc:40-77.  (1.0 - beta) is evaluated in double and narrowed to
 * the array scalar (float) before the multiply (Eigen scalar promotion);
 * the bias correction is folded into lr in double (pow(float, long long)
 * promotes to double) and narrowed back to float by `lr *=`.  Epsilon is
 * outside the sqrt. */
void oracle_adam(const float* grad, float* param, float* m, float* v, float lr,
                 long long size, long long step, float beta1, float beta2,
                 float epsilon, float* max_square) {
  const float c1 = (float)(1.0 - (double)beta1);
  const float c2 = (float)(1.0 - (double)beta2);
  lr = (float)((double)lr * (sqrt(1.0 - pow((double)beta2, (double)step)) /
                             (1.0 - pow((double)beta1, (double)step))));
  for (long long i = 0; i < size; ++i) {
    float g = grad[i];
    float mi = beta1 * m[i] + c1 * g;      /* kernel_api.cc:63 */
    float vi = beta2 * v[i] + c2 * (g * g); /* kernel_api.cc:65 */
    m[i] = mi;
    v[i] = vi;
    if (max_square != NULL) {               /* kernel_api.cc:69-73 */
      float ms = max_square[i];
      ms = ms < vi ? vi : ms;
      max_square[i] = ms;
      param[i] = param[i] - (lr * mi) / (sqrtf(ms) + epsilon);
    } else {                                /* kernel_api.cc:75 */
      param[i] = param[i] - (lr * mi) / (sqrtf(vi) + epsilon);
    }
  }
}

/* kernel_api.cc:79-96   em += eg^2 ; ep -= lr*eg/(sqrt(em)+eps) */
void oracle_adagrad(const float* grad, float* param, float* m, float lr,
                    long long size, float epsilon) {
  for (long long i = 0; i < size; ++i) {
    float g = grad[i];
    float a = m[i] + g * g;
    m[i] = a;
    param[i] = param[i] - (lr * g) / (sqrtf(a) + epsilon);
  }
}

/* FTRL: NOT in the Go PS.  The reference reaches it only through
 * tf.keras.optimizers.Ftrl in the Python PS (python/ps/optimizer_wrapper.py:
 * 26,129-134); its arithmetic lives in tensorflow==2.5.2 (requirements.txt:6)
 * which is not under /root/reference -> PARITY UNPINNED.  Restated from TF's
 * documented ApplyFtrl (training_ops FtrlCompute), learning_rate_power = -0.5
 * fast path (rsqrt form), l2 already includes Keras' beta/(2*lr) term:
 *   g_shr      = g + 2*l2_shrinkage*var
 *   accum_new  = accum + g*g
 *   sigma      = (sqrt(accum_new) - sqrt(accum)) / lr
 *   linear    += (g_shr - sigma*var)
 *   quadratic  = sqrt(accum_new)/lr + 2*l2
 *   var        = |linear| > l1 ? (sign(linear)*l1 - linear)/quadratic : 0
 *   accum      = accum_new
 */
void oracle_ftrl(const float* grad, float* param, float* accum, float* linear,
                 float lr, long long size, float l1, float l2,
                 float l2_shrinkage) {
  for (long long i = 0; i < size; ++i) {
    float g = grad[i];
    float var = param[i];
    float g_shr = g + (2.0f * l2_shrinkage) * var;
    float a_old = accum[i];
    float a_new = a_old + g * g;
    float sigma = (sqrtf(a_new) - sqrtf(a_old)) / lr;
    float lin = linear[i] + (g_shr - sigma * var);
    float quad = sqrtf(a_new) / lr + 2.0f * l2;
    float sgn = lin > 0.0f ? 1.0f : (lin < 0.0f ? -1.0f : 0.0f);
    float out = fabsf(lin) > l1 ? (sgn * l1 - lin) / quad : 0.0f;
    linear[i] = lin;
    accum[i] = a_new;
    param[i] = out;
  }
}

/* ------------------------------------------------------------------ */
/* EmbeddingTable: go/pkg/common/embedding_table.go:22-88              */
/* map[int64]*Tensor + RWMutex, lazy row creation on first get.        */
/* ------------------------------------------------------------------ */

typedef struct {
  int64_t key;
  float* row;
} oslot_t;

typedef struct otable {
  int64_t dim;
  int init_uniform;    /* Initializer == "uniform" (embedding_table.go:51) */
  float init_constant; /* python slot tables: constant init (python/ps/embedding_table.py:135-136) */
  uint64_t seed;
  oslot_t* slots;
  size_t cap;  /* power of two */
  size_t size; /* len(EmbeddingVectors) */
  pthread_rwlock_t lock;
} otable_t;

static inline uint64_t mix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdULL;
  x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL;
  x ^= x >> 33; return x;
}

otable_t* otable_new(int64_t dim, int init_uniform, float init_constant,
                     uint64_t seed) {
  otable_t* t = (otable_t*)calloc(1, sizeof(otable_t));
  t->dim = dim;
  t->init_uniform = init_uniform;
  t->init_constant = init_constant;
  t->seed = seed;
  t->cap = 1024;
  t->slots = (oslot_t*)calloc(t->cap, sizeof(oslot_t));
  pthread_rwlock_init(&t->lock, NULL);
  return t;
}

void otable_free(otable_t* t) {
  if (!t) return;
  for (size_t i = 0; i < t->cap; ++i) free(t->slots[i].row);
  free(t->slots);
  pthread_rwlock_destroy(&t->lock);
  free(t);
}

int64_t otable_size(otable_t* t) { return (int64_t)t->size; }
int64_t otable_dim(otable_t* t) { return t->dim; }

static float* otable_find_nolock(otable_t* t, int64_t key) {
  size_t mask = t->cap - 1;
  size_t i = (size_t)mix64((uint64_t)key) & mask;
  while (t->slots[i].row) {
    if (t->slots[i].key == key) return t->slots[i].row;
    i = (i + 1) & mask;
  }
  return NULL;
}

static void otable_insert_nolock(otable_t* t, int64_t key, float* row) {
  if ((t->size + 1) * 2 > t->cap) {
    size_t ncap = t->cap * 2;
    oslot_t* ns = (oslot_t*)calloc(ncap, sizeof(oslot_t));
    for (size_t j = 0; j < t->cap; ++j) {
      if (!t->slots[j].row) continue;
      size_t i = (size_t)mix64((uint64_t)t->slots[j].key) & (ncap - 1);
      while (ns[i].row) i = (i + 1) & (ncap - 1);
      ns[i] = t->slots[j];
    }
    free(t->slots);
    t->slots = ns;
    t->cap = ncap;
  }
  size_t mask = t->cap - 1;
  size_t i = (size_t)mix64((uint64_t)key) & mask;
  while (t->slots[i].row) i = (i + 1) & mask;
  t->slots[i].key = key;
  t->slots[i].row = row;
  t->size++;
}

/* The GPU path's deterministic stand-in for the reference's lazy
 * RandomUniform(-0.05, 0.05, seed=len(map)) (embedding_table.go:51-54,
 * initializer.go:107-126).  The reference draws from Go's global math/rand
 * re-seeded with the current map size: insertion-order and race dependent, not
 * reproducible even Go-vs-Go, so it is excluded from parity (DESIGN.md).  The
 * oracle and the CUDA path share this counter-based generator instead: value =
 * f(seed, id, column), range and distribution as the reference. */
float oracle_uniform_init(uint64_t seed, int64_t id, int64_t col) {
  uint64_t h = mix64(seed ^ mix64((uint64_t)id * 0x9E3779B97F4A7C15ULL + (uint64_t)col));
  float u = (float)(h >> 40) * (1.0f / 16777216.0f); /* [0,1) 24 bit */
  return u * 0.1f + (-0.05f);                        /* initializer.go:116 */
}

/* embedding_table.go:41-58 GetEmbeddingVector: RLock probe; on miss allocate,
 * initialise (uniform or zeros) and insert under the write lock. */
float* otable_get_row(otable_t* t, int64_t id) {
  pthread_rwlock_rdlock(&t->lock);
  float* r = otable_find_nolock(t, id);
  pthread_rwlock_unlock(&t->lock);
  if (r) return r;
  float* nr = (float*)calloc((size_t)t->dim, sizeof(float));
  if (t->init_uniform) {
    for (int64_t c = 0; c < t->dim; ++c) nr[c] = oracle_uniform_init(t->seed, id, c);
  } else if (t->init_constant != 0.0f) {
    for (int64_t c = 0; c < t->dim; ++c) nr[c] = t->init_constant;
  }
  pthread_rwlock_wrlock(&t->lock);
  r = otable_find_nolock(t, id); /* another thread may have won (the Go code
                                    would overwrite; single-threaded identical) */
  if (!r) {
    otable_insert_nolock(t, id, nr);
    r = nr;
    nr = NULL;
  }
  pthread_rwlock_unlock(&t->lock);
  free(nr);
  return r;
}

/* embedding_table.go:61-68 GetEmbeddingVectors: COPIES of rows, in id order */
void otable_pull(otable_t* t, const int64_t* ids, int64_t n, float* out) {
  for (int64_t i = 0; i < n; ++i)
    memcpy(out + i * t->dim, otable_get_row(t, ids[i]), (size_t)t->dim * sizeof(float));
}

/* embedding_table.go:71-77 SetEmbeddingVectors */
void otable_set_rows(otable_t* t, const int64_t* ids, int64_t n, const float* values) {
  for (int64_t i = 0; i < n; ++i)
    memcpy(otable_get_row(t, ids[i]), values + i * t->dim, (size_t)t->dim * sizeof(float));
}

/* embedding_table.go:80-88 ToIndexedSlices: keys (map order is unspecified in
 * Go; here: table order) -- returns the ids, caller pulls rows. */
int64_t otable_keys(otable_t* t, int64_t* out, int64_t max) {
  int64_t n = 0;
  for (size_t i = 0; i < t->cap && n < max; ++i)
    if (t->slots[i].row) out[n++] = t->slots[i].key;
  return n;
}

/* ------------------------------------------------------------------ */
/* Sparse kernels (hash-table rows): go/pkg/kernel/kernel.go           */
/* Duplicated ids are applied SEQUENTIALLY, rows lazily created.       */
/* ------------------------------------------------------------------ */

/* kernel.go:35-45 */
void oracle_sparse_sgd(otable_t* p, const int64_t* ids, const float* grads, int64_t n, float lr) {
  for (int64_t i = 0; i < n; ++i)
    oracle_sgd(grads + i * p->dim, otable_get_row(p, ids[i]), lr, p->dim);
}
/* kernel.go:69-81 */
void oracle_sparse_momentum(otable_t* p, otable_t* vel, const int64_t* ids, const float* grads,
                            int64_t n, float mu, int nesterov, float lr) {
  for (int64_t i = 0; i < n; ++i)
    oracle_momentum(grads + i * p->dim, otable_get_row(p, ids[i]), otable_get_row(vel, ids[i]),
                    mu, nesterov, lr, p->dim);
}
/* Optional: the reference's OWN compiled Adam (kernel_api.h:20-30, from oracle/_ref/libkernel_api_ref.so =
 * kernel_api.cc built unmodified) for the per-row update, exactly as kernel.go:119-138 calls it through cgo.
 * Set by bench.py's CPU arm when oracle/_ref is present; NULL = the restatement above (bit-identical,
 * tests/test_oracle_vs_ref.py). */
typedef void (*ref_adam_fn)(float*, float*, float*, float*, float, long long, long long, float, float, float, float*);
static ref_adam_fn g_ref_adam = NULL;
void oracle_set_ref_adam(void* fn) { g_ref_adam = (ref_adam_fn)fn; }

/* kernel.go:119-138 */
void oracle_sparse_adam(otable_t* p, otable_t* m, otable_t* v, otable_t* ms, const int64_t* ids,
                        const float* grads, int64_t n, float lr, long long step, float beta1,
                        float beta2, float epsilon) {
  const ref_adam_fn ref = g_ref_adam;
  for (int64_t i = 0; i < n; ++i) {
    float* sp = otable_get_row(p, ids[i]);
    float* sm = otable_get_row(m, ids[i]);
    float* sv = otable_get_row(v, ids[i]);
    float* sms = ms ? otable_get_row(ms, ids[i]) : NULL;
    if (ref)
      ref((float*)(grads + i * p->dim), sp, sm, sv, lr, p->dim, step, beta1, beta2, epsilon, sms);
    else
      oracle_adam(grads + i * p->dim, sp, sm, sv, lr, p->dim, step, beta1, beta2, epsilon, sms);
  }
}
/* kernel.go:172-184 */
void oracle_sparse_adagrad(otable_t* p, otable_t* m, const int64_t* ids, const float* grads,
                           int64_t n, float lr, float epsilon) {
  for (int64_t i = 0; i < n; ++i)
    oracle_adagrad(grads + i * p->dim, otable_get_row(p, ids[i]), otable_get_row(m, ids[i]), lr,
                   p->dim, epsilon);
}
/* FTRL over table rows: python/ps/optimizer_wrapper.py:116-149 slot naming
 * ("accumulator" init initial_accumulator_value, "linear" init 0). */
void oracle_sparse_ftrl(otable_t* p, otable_t* accum, otable_t* linear, const int64_t* ids,
                        const float* grads, int64_t n, float lr, float l1, float l2, float l2s) {
  for (int64_t i = 0; i < n; ++i)
    oracle_ftrl(grads + i * p->dim, otable_get_row(p, ids[i]), otable_get_row(accum, ids[i]),
                otable_get_row(linear, ids[i]), lr, p->dim, l1, l2, l2s);
}

/* ------------------------------------------------------------------ */
/* Indexed kernels (rows of a dense [R,dim] matrix): kernel.go:48-55,  */
/* 84-96, 141-160, 187-199.  opt: 0 SGD 1 Momentum 2 Adam 3 AMSGrad    */
/* 4 Adagrad 5 FTRL.  s0..s2 are the same-shape slot matrices.         */
/* ------------------------------------------------------------------ */
void oracle_indexed_apply(int opt, float* param, float* s0, float* s1, float* s2, int64_t dim,
                          const int64_t* ids, const float* grads, int64_t n, float lr,
                          long long step, float h0, float h1, float h2, int flag) {
  for (int64_t i = 0; i < n; ++i) {
    int64_t r = ids[i];
    const float* g = grads + i * dim;
    switch (opt) {
      case 0: oracle_sgd(g, param + r * dim, lr, dim); break;
      case 1: oracle_momentum(g, param + r * dim, s0 + r * dim, h0, flag, lr, dim); break;
      case 2: oracle_adam(g, param + r * dim, s0 + r * dim, s1 + r * dim, lr, dim, step, h0, h1, h2, NULL); break;
      case 3: oracle_adam(g, param + r * dim, s0 + r * dim, s1 + r * dim, lr, dim, step, h0, h1, h2, s2 + r * dim); break;
      case 4: oracle_adagrad(g, param + r * dim, s0 + r * dim, lr, dim, h0); break;
      case 5: oracle_ftrl(g, param + r * dim, s0 + r * dim, s1 + r * dim, lr, dim, h0, h1, h2); break;
    }
  }
}

/* ------------------------------------------------------------------ */
/* deduplicate_indexed_slices: python/common/tensor_utils.py:39-60     */
/* Sum rows with equal index; output order = first occurrence;         */
/* accumulation order = occurrence order (in-place += on first row).   */
/* Returns number of unique ids.                                       */
/* ------------------------------------------------------------------ */
int64_t oracle_dedup(const float* values, const int64_t* indices, int64_t k, int64_t dim,
                     float* out_values, int64_t* out_indices) {
  size_t cap = 16;
  while (cap < (size_t)k * 2 + 2) cap <<= 1;
  int64_t* keys = (int64_t*)malloc(cap * sizeof(int64_t));
  int64_t* pos = (int64_t*)malloc(cap * sizeof(int64_t));
  for (size_t i = 0; i < cap; ++i) pos[i] = -1;
  int64_t u = 0;
  for (int64_t i = 0; i < k; ++i) {
    size_t s = (size_t)mix64((uint64_t)indices[i]) & (cap - 1);
    while (pos[s] >= 0 && keys[s] != indices[i]) s = (s + 1) & (cap - 1);
    if (pos[s] < 0) {
      keys[s] = indices[i];
      pos[s] = u;
      out_indices[u] = indices[i];
      memcpy(out_values + u * dim, values + i * dim, (size_t)dim * sizeof(float));
      ++u;
    } else {
      float* dst = out_values + pos[s] * dim;
      const float* src = values + i * dim;
      for (int64_t c = 0; c < dim; ++c) dst[c] = dst[c] + src[c];
    }
  }
  free(keys);
  free(pos);
  return u;
}

/* tf.unique as used by embedding_delegate.py:85: unique ids in first
 * occurrence order and the inverse index. */
int64_t oracle_unique(const int64_t* ids, int64_t k, int64_t* out_unique, int32_t* out_idx) {
  size_t cap = 16;
  while (cap < (size_t)k * 2 + 2) cap <<= 1;
  int64_t* keys = (int64_t*)malloc(cap * sizeof(int64_t));
  int64_t* pos = (int64_t*)malloc(cap * sizeof(int64_t));
  for (size_t i = 0; i < cap; ++i) pos[i] = -1;
  int64_t u = 0;
  for (int64_t i = 0; i < k; ++i) {
    size_t s = (size_t)mix64((uint64_t)ids[i]) & (cap - 1);
    while (pos[s] >= 0 && keys[s] != ids[i]) s = (s + 1) & (cap - 1);
    if (pos[s] < 0) {
      keys[s] = ids[i];
      pos[s] = u;
      out_unique[u++] = ids[i];
    }
    out_idx[i] = (int32_t)pos[s];
  }
  free(keys);
  free(pos);
  return u;
}

/* ------------------------------------------------------------------ */
/* Timed CPU baseline: T worker threads drive M in-process shards      */
/* through pull -> (caller-supplied grads) -> dedup -> scatter ->      */
/* SparseAdam, i.e. worker/ps_client.py:96-130,243-268 composed with   */
/* go/pkg/ps/server.go:163-206, with gRPC/protobuf removed (which      */
/* flatters the reference).                                            */
/* ------------------------------------------------------------------ */
typedef struct {
  int n_tables;       /* tables per family member (e.g. 38 groups) */
  int n_shards;
  otable_t** p;       /* [n_tables * n_shards] param tables  */
  otable_t** m;       /* Adam m  */
  otable_t** v;       /* Adam v  */
  const int64_t* ids; /* [n_threads][n_tables][batch] */
  const float* grads; /* [n_threads][n_tables][batch][dim] (per-occurrence BET grads) */
  int64_t batch;
  int64_t dim;
  float lr, beta1, beta2, eps;
  long long step0;
  int steps;
  int tid;
  double pulled_rows, pushed_rows;
} obench_arg_t;

static void* obench_thread(void* vp) {
  obench_arg_t* a = (obench_arg_t*)vp;
  const int64_t B = a->batch, D = a->dim;
  int64_t* uniq = (int64_t*)malloc(B * sizeof(int64_t));
  int32_t* idx = (int32_t*)malloc(B * sizeof(int32_t));
  float* bet = (float*)malloc(B * D * sizeof(float));
  float* gsum = (float*)malloc(B * D * sizeof(float));
  int64_t* gids = (int64_t*)malloc(B * sizeof(int64_t));
  int64_t* sid = (int64_t*)malloc(B * sizeof(int64_t));
  float* sg = (float*)malloc(B * D * sizeof(float));
  for (int s = 0; s < a->steps; ++s) {
    for (int t = 0; t < a->n_tables; ++t) {
      const int64_t* ids = a->ids + ((int64_t)a->tid * a->n_tables + t) * B;
      const float* g = a->grads + (((int64_t)a->tid * a->n_tables + t) * B) * D;
      /* embedding_delegate.py:85 unique, ps_client.py:96-130 pull per shard */
      int64_t u = oracle_unique(ids, B, uniq, idx);
      for (int sh = 0; sh < a->n_shards; ++sh) {
        int64_t c = 0;
        for (int64_t i = 0; i < u; ++i)
          if (uniq[i] % a->n_shards == sh) sid[c++] = uniq[i];
        otable_pull(a->p[t * a->n_shards + sh], sid, c, bet);
      }
      a->pulled_rows += (double)u;
      /* ps_client.py:255-268 dedup + scatter, server.go:176-206 apply */
      int64_t gu = oracle_dedup(g, ids, B, D, gsum, gids);
      for (int sh = 0; sh < a->n_shards; ++sh) {
        int64_t c = 0;
        for (int64_t i = 0; i < gu; ++i)
          if (gids[i] % a->n_shards == sh) {
            sid[c] = gids[i];
            memcpy(sg + c * D, gsum + i * D, (size_t)D * sizeof(float));
            ++c;
          }
        oracle_sparse_adam(a->p[t * a->n_shards + sh], a->m[t * a->n_shards + sh],
                           a->v[t * a->n_shards + sh], NULL, sid, sg, c, a->lr,
                           a->step0 + s + 1, a->beta1, a->beta2, a->eps);
      }
      a->pushed_rows += (double)gu;
    }
  }
  free(uniq); free(idx); free(bet); free(gsum); free(gids); free(sid); free(sg);
  return NULL;
}

/* Returns wall seconds for `steps` steps of every thread; rows_out[0..1] =
 * total pulled / pushed unique rows. */
double oracle_bench_ps(int n_threads, int n_tables, int n_shards, otable_t** p, otable_t** m,
                       otable_t** v, const int64_t* ids, const float* grads, int64_t batch,
                       int64_t dim, float lr, float beta1, float beta2, float eps, int steps,
                       double* rows_out) {
  pthread_t* th = (pthread_t*)malloc(sizeof(pthread_t) * n_threads);
  obench_arg_t* args = (obench_arg_t*)calloc(n_threads, sizeof(obench_arg_t));
  struct timespec t0, t1;
  clock_gettime(CLOCK_MONOTONIC, &t0);
  for (int i = 0; i < n_threads; ++i) {
    obench_arg_t a = {n_tables, n_shards, p, m, v, ids, grads, batch, dim, lr, beta1, beta2, eps, 0, steps, i, 0, 0};
    args[i] = a;
    pthread_create(&th[i], NULL, obench_thread, &args[i]);
  }
  double pr = 0, qr = 0;
  for (int i = 0; i < n_threads; ++i) {
    pthread_join(th[i], NULL);
    pr += args[i].pulled_rows;
    qr += args[i].pushed_rows;
  }
  clock_gettime(CLOCK_MONOTONIC, &t1);
  if (rows_out) { rows_out[0] = pr; rows_out[1] = qr; }
  free(th); free(args);
  return (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
}
