// Nearest-item retrieval over the embedding table: the serving step that follows Actor.forward in the
// reference (examples/streamlit_demo.py:189-215: faiss IndexFlatL2 / IndexFlatIP / cosine over the item
// matrix; recnn/data/db_con.py:45-56: MilvusConnection.search(search_vecs, topk)).
//
//   scores[q, j] = <query_q, item_j>            one [Q, D] x [D, n_items] contraction on the tensor cores
//                                               (wgmma 3xTF32, the update step's own GEMM kernel), in slabs
//                                               of query rows so that a slab of scores stays inside the 50 MB L2
//   key[q, j]    = |item_j|^2 - 2 scores        L2   (+ |query_q|^2 at the end: the squared distance faiss/Milvus report)
//                = -scores                      IP   (larger inner product = better)
//                = -scores / |item_j|           COS  (/ |query_q| at the end)
//   top-k smallest keys per query, ties broken towards the smaller item id (== a stable argsort of the keys).
//
// Top-k: every CTA owns one (query, column range); each thread keeps the best k of its strided share in a sorted
// register list (an element is compared with the list's worst first, so the insertion runs ~k ln(n/k) times);
// the CTA then merges its 256 sorted lists (block_merge, topk.cuh); a second tiny kernel merges the column ranges of a
// query (warp_merge) and reports the distances (metric_distance).  Everything is exact (no approximate search).
#include <float.h>
#include <string.h>

#include "common.cuh"
#include "distance.cuh"
#include "gemm_simt.cuh"
#include "tc_gemm.cuh"
#include "topk.cuh"

namespace recnn {

// per item: |t|^2 (L2) or 1/|t| (COS)
__global__ void __launch_bounds__(256)
item_norms_kernel(const float* __restrict__ table, long long n_items, int dim, int metric, float* __restrict__ out) {
  const long long row = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n_items) return;
  const float* t = table + row * dim;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s = fmaf(t[d], t[d], s);
  s = warp_sum(s);
  if (lane == 0) out[row] = metric == RECNN_METRIC_COS ? 1.0f / fmaxf(sqrtf(s), 1e-30f) : s;
}

// grid (splits, n_queries).  scores [n_queries, ld]; writes k candidates per (query, split), ascending.  Query q is
// row row0 + q of the call; with SETS its excluded set (ex) is tested only for a candidate that enters the thread's
// list (without, the kernel is the plain search, nothing staged).
template <int KMAX, bool SETS>
__global__ void __launch_bounds__(kTopkThreads)
topk_partial_kernel(const float* __restrict__ scores, long long ld, long long n_items, const float* __restrict__ norms,
                    int metric, int k, ItemSets ex, long long row0, int stage_cap, Cand* __restrict__ part) {
  extern __shared__ int s_set[];
  const int q = blockIdx.y, sp = blockIdx.x, splits = gridDim.x;
  const long long per = (n_items + splits - 1) / splits;
  const long long lo = sp * per, hi = min(n_items, lo + per);
  const float* row = scores + (long long)q * ld;
  SetView set = {nullptr, 0, true};
  if (SETS) {
    set = set_stage(ex, row0 + q, s_set, stage_cap);
    __syncthreads();
  }
  float keys[KMAX];
  int ids[KMAX];
  list_clear(keys, ids);
  for (long long j = lo + threadIdx.x; j < hi; j += blockDim.x) {
    const float key = metric_key(__ldcs(row + j), norms, j, metric);
    int id = (int)j;
    if (better(key, id, keys[KMAX - 1], ids[KMAX - 1]) && (!SETS || set.n == 0 || !set_has(set, s_set, id)))
      list_insert(keys, ids, key, id);
  }
  block_merge(keys, ids, k, part + ((long long)q * splits + sp) * k);
}

// one warp per query: merge `splits` <= 32 ascending lists of k candidates; finish the metric
__global__ void __launch_bounds__(128)
topk_merge_kernel(const Cand* __restrict__ part, int splits, int k, long long n_queries, int metric,
                  const float* __restrict__ queries, int dim, int64_t* __restrict__ ids_out, float* __restrict__ dist_out) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_queries) return;
  const float qn = warp_sq_norm(queries + q * dim, dim);
  const Cand* mine = part + q * (long long)splits * k;
  warp_merge<1>(k, [&](int l, int pos) {
    return l < splits && pos < k ? mine[(long long)l * k + pos] : Cand{FLT_MAX, kNoId};
  }, [&](int r, float key, int id, int) {
    if (lane == 0) {
      ids_out[q * k + r] = id == kNoId ? -1 : (int64_t)id;
      dist_out[q * k + r] = metric_distance(key, id, qn, metric);
    }
  });
}

// grid (splits, n_queries): rank[row0 + q] += the items of columns [lo, hi) that beat the query's target by
// metric_key (ties: the smaller id), minus the excluded ones (SETS).  The target's key is read from the same scores row,
// so every comparison is between the bits the search ranks.  A target outside [0, n_items) counts nothing.
template <bool SETS>
__global__ void __launch_bounds__(kTopkThreads)
rank_count_kernel(const float* __restrict__ scores, long long ld, long long n_items, const float* __restrict__ norms,
                  int metric, const long long* __restrict__ target, ItemSets ex, long long row0,
                  long long* __restrict__ rank) {
  __shared__ long long s_range[3];
  const int q = blockIdx.y, sp = blockIdx.x, splits = gridDim.x;
  const long long per = (n_items + splits - 1) / splits;
  const long long lo = sp * per, hi = min(n_items, lo + per);
  const long long t = target[row0 + q];
  if (t < 0 || t >= n_items) return;
  const float* row = scores + (long long)q * ld;
  const float kt = metric_key(row[t], norms, t, metric);
  int c = 0;
  for (long long j = lo + threadIdx.x; j < hi; j += blockDim.x)
    c += j != t && better(metric_key(__ldcs(row + j), norms, j, metric), (int)j, kt, (int)t);
  if (SETS)
    c -= excluded_beaters(ex, row0 + q, lo, hi, kt, (int)t,
                          [&](long long x) { return metric_key(row[x], norms, x, metric); }, s_range);
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c != 0)
    atomicAdd(reinterpret_cast<unsigned long long*>(rank + row0 + q), (unsigned long long)(long long)c);
}

// rank[q] <- 0, or -1 and *flag |= 1 for a target outside [0, n_items)
__global__ void rank_init_kernel(const long long* __restrict__ target, long long n, long long n_items,
                                 long long* __restrict__ rank, int* flag) {
  const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= n) return;
  const bool ok = target[q] >= 0 && target[q] < n_items;
  rank[q] = ok ? 0 : -1;
  if (!ok) atomicOr(flag, 1);
}

static int64_t slab_rows(int64_t n_items) {
  // a slab of scores should stay L2-resident between the GEMM that writes it and the top-k pass that reads it:
  // 32 MB of the H100's 50 MB L2, leaving room for the item table, its norms and the top-k partials
  const int64_t ld = round_up(n_items, 4);
  int64_t r = (32ll << 20) / (ld * 4);
  r = r / 128 * 128;
  return r < 128 ? 128 : (r > 4096 ? 4096 : r);
}

struct RetrieveWorkspace {
  int64_t slab, ld;    // query rows per slab; row pitch of the scores
  float* scores;       // [slab, ld]
  Cand* part;          // [slab, splits <= 32, k] candidates of every (query, column range)
  int64_t bytes;
};
static RetrieveWorkspace retrieve_carve(int64_t n_queries, int64_t n_items, int k, void* base) {
  RetrieveWorkspace w;
  Carve c(base);
  w.slab = n_queries < slab_rows(n_items) ? n_queries : slab_rows(n_items);
  w.ld = round_up(n_items, 4);
  w.scores = c.take(w.slab * w.ld);
  w.part = c.take<Cand>(w.slab * 32 * (int64_t)k);
  w.bytes = c.bytes();
  return w;
}

}  // namespace recnn

using namespace recnn;

extern "C" int recnn_item_norms(const float* table, int64_t n_items, int32_t dim, int32_t metric, float* out,
                                void* stream) {
  RECNN_REQUIRE(table && out && n_items > 0 && dim > 0, "table/out");
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_COS || metric == RECNN_METRIC_CORR,
                "norms exist for L2, COS and CORR");
  if (metric == RECNN_METRIC_CORR) {
    corr_stats_kernel<<<(unsigned)ceil_div(n_items, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(table, n_items,
                                                                                                       dim, out);
    RECNN_CHECK_LAUNCH("corr_stats_kernel");
    return RECNN_OK;
  }
  const int64_t blocks = ceil_div(n_items, 8);
  item_norms_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(table, n_items, dim, metric, out);
  RECNN_CHECK_LAUNCH("item_norms_kernel");
  return RECNN_OK;
}

extern "C" int64_t recnn_retrieve_workspace_bytes(int64_t n_queries, int64_t n_items, int32_t k) {
  if (n_queries <= 0 || n_items <= 0 || k <= 0) return 0;
  return retrieve_carve(n_queries, n_items, k, nullptr).bytes;
}

// The slab loop of every retrieval call: for each slab of up to w.slab query rows, scores[q, j] = <query q0 + q,
// item j> into w.scores for L2 / IP / COS (the tensor-core GEMM when the operands allow it, else the CUDA-core one: one
// choice per call), the distance of the pair for the other metrics (distance.cuh), then after(q0, nq) reads the slab.
// A search and a rank over the same queries see the same score bits.
template <class After>
static int retrieve_slabs(const float* queries, int64_t n_queries, int32_t dim, const float* table, int64_t n_items,
                          const float* norms, int32_t metric, const RetrieveWorkspace& w, cudaStream_t st,
                          After after) {
  const bool tc_ok = dim % 4 == 0 && (reinterpret_cast<uintptr_t>(queries) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(table) & 15) == 0;
  for (int64_t q0 = 0; q0 < n_queries; q0 += w.slab) {
    const int64_t nq = n_queries - q0 < w.slab ? n_queries - q0 : w.slab;
    const float* Q = queries + q0 * dim;
    if (metric >= RECNN_METRIC_L1) {
      RECNN_PROPAGATE(distance_slab(metric, Q, nq, table, n_items, dim, norms, w.scores, w.ld, st));
      RECNN_PROPAGATE(after(q0, nq));
      continue;
    }
    Epilogue e;
    memset(&e, 0, sizeof(e));
    e.out = w.scores;
    e.ldo = w.ld;
    if (tc_ok) {
      tc::Operand a0 = {Q, dim, 0, 0}, a1 = {nullptr, 0, 0, 0}, b = {table, dim, n_items, dim};
      tc::Problem p;
      memset(&p, 0, sizeof(p));
      p.M = (int)nq; p.N = (int)n_items; p.K0 = dim; p.b_k1_offset = dim;
      const int r = tc::launch<false, false, EPI_STORE>(a0, a1, b, p, 1, 128, e, st);
      if (r < 0) return r;
    } else {
      RECNN_PROPAGATE((launch_gemm_simt<true, true, EPI_STORE>(mat(Q, dim), mat(table, dim), (int)nq, (int)n_items, dim,
                                                                1, e, st)));
    }
    RECNN_PROPAGATE(after(q0, nq));
  }
  return RECNN_OK;
}

// the argument checks of every retrieval call
static int retrieve_check(const float* queries, int64_t n_queries, int32_t dim, const float* table, int64_t n_items,
                          const float* norms, int32_t metric, const void* workspace) {
  RECNN_REQUIRE(queries && table && workspace, "null pointer");
  RECNN_REQUIRE(n_queries >= 0 && n_items > 0 && dim > 0, "sizes");
  RECNN_REQUIRE(metric >= RECNN_METRIC_L2 && metric <= RECNN_METRIC_CORR, "metric");
  RECNN_REQUIRE(!(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_COS || metric == RECNN_METRIC_CORR) ||
                norms != nullptr, "L2 / COS / CORR need recnn_item_norms");
  RECNN_REQUIRE(n_items < (1ll << 31), "n_items must fit int32");
  return RECNN_OK;
}

// the checks of a search: the arguments, then the workspace carved at n_queries rows against workspace_bytes.  Every
// refusal comes before any device work (the *_sets forms zero the caller's flag and check the table only after it).
static int retrieve_topk_check(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                               int64_t n_items, const float* norms, int32_t metric, int32_t k, const int64_t* ids_out,
                               const float* dist_out, void* workspace, int64_t workspace_bytes, RetrieveWorkspace* w) {
  RECNN_PROPAGATE(retrieve_check(queries, n_queries, dim, table, n_items, norms, metric, workspace));
  RECNN_REQUIRE(ids_out && dist_out, "null pointer");
  RECNN_REQUIRE(k >= 1 && k <= 64 && k <= n_items, "1 <= k <= min(64, n_items)");
  if (n_queries == 0) return RECNN_OK;
  *w = retrieve_carve(n_queries, n_items, k, workspace);
  return check_workspace(w->bytes, workspace_bytes);
}

// the search behind both entry points, on a checked workspace; ex.ids NULL: no exclusion
static int retrieve(const float* queries, int64_t n_queries, int32_t dim, const float* table, int64_t n_items,
                    const float* norms, int32_t metric, int32_t k, const ItemSets& ex, int64_t* ids_out,
                    float* dist_out, const RetrieveWorkspace& w, cudaStream_t st) {
  if (n_queries == 0) return RECNN_OK;
  const int stage = set_stage_bytes(ex);
  auto kernel = k <= 16 ? (stage ? topk_partial_kernel<16, true> : topk_partial_kernel<16, false>)
                        : (stage ? topk_partial_kernel<64, true> : topk_partial_kernel<64, false>);
  return retrieve_slabs(queries, n_queries, dim, table, n_items, norms, metric, w, st, [&](int64_t q0, int64_t nq) {
    const float* Q = queries + q0 * dim;
    const int splits = topk_splits(nq, n_items, 32);
    dim3 grid((unsigned)splits, (unsigned)nq);
    kernel<<<grid, kTopkThreads, stage, st>>>(w.scores, w.ld, n_items, norms, metric, k, ex, q0,
                                              stage / (int)sizeof(int), w.part);
    RECNN_CHECK_LAUNCH("topk_partial_kernel");
    topk_merge_kernel<<<(unsigned)ceil_div(nq, 4), 128, 0, st>>>(w.part, splits, k, nq, metric, Q, dim,
                                                                  ids_out + q0 * k, dist_out + q0 * k);
    RECNN_CHECK_LAUNCH("topk_merge_kernel");
    return RECNN_OK;
  });
}

// the checks of a rank, as retrieve_topk_check
static int retrieve_rank_check(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                               int64_t n_items, const float* norms, int32_t metric, const int64_t* target,
                               const int64_t* rank_out, const int32_t* error_flag, void* workspace,
                               int64_t workspace_bytes, RetrieveWorkspace* w) {
  RECNN_PROPAGATE(retrieve_check(queries, n_queries, dim, table, n_items, norms, metric, workspace));
  RECNN_REQUIRE(target && rank_out && error_flag, "null pointer");
  if (n_queries == 0) return RECNN_OK;
  *w = retrieve_carve(n_queries, n_items, 0, workspace);
  return check_workspace(w->bytes, workspace_bytes);
}

// the rank behind both entry points, on a checked workspace: the slab's GEMM, then one count kernel per slab
static int retrieve_rank(const float* queries, int64_t n_queries, int32_t dim, const float* table, int64_t n_items,
                         const float* norms, int32_t metric, const int64_t* target, const ItemSets& ex,
                         int64_t* rank_out, int32_t* error_flag, const RetrieveWorkspace& w, cudaStream_t st) {
  if (n_queries == 0) return RECNN_OK;
  const long long* tgt = reinterpret_cast<const long long*>(target);
  long long* rank = reinterpret_cast<long long*>(rank_out);
  rank_init_kernel<<<(unsigned)ceil_div(n_queries, 256), 256, 0, st>>>(tgt, n_queries, n_items, rank, error_flag);
  RECNN_CHECK_LAUNCH("rank_init_kernel");
  auto kernel = ex.ids ? rank_count_kernel<true> : rank_count_kernel<false>;
  return retrieve_slabs(queries, n_queries, dim, table, n_items, norms, metric, w, st, [&](int64_t q0, int64_t nq) {
    dim3 grid((unsigned)topk_splits(nq, n_items, 32), (unsigned)nq);
    kernel<<<grid, kTopkThreads, 0, st>>>(w.scores, w.ld, n_items, norms, metric, tgt, ex, q0, rank);
    RECNN_CHECK_LAUNCH("rank_count_kernel");
    return RECNN_OK;
  });
}

extern "C" int recnn_retrieve_topk(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                   int64_t n_items, const float* norms, int32_t metric, int32_t k, int64_t* ids_out,
                                   float* dist_out, void* workspace, int64_t workspace_bytes, void* stream) {
  RetrieveWorkspace w{};
  RECNN_PROPAGATE(retrieve_topk_check(queries, n_queries, dim, table, n_items, norms, metric, k, ids_out, dist_out,
                                      workspace, workspace_bytes, &w));
  const ItemSets none = {nullptr, nullptr, nullptr, 0, 0, 0};
  return retrieve(queries, n_queries, dim, table, n_items, norms, metric, k, none, ids_out, dist_out, w,
                  static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_retrieve_topk_sets(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                        int64_t n_items, const float* norms, int32_t metric, int32_t k,
                                        const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                                        int64_t n_sets, const int64_t* row_set, int64_t* ids_out, float* dist_out,
                                        int32_t* error_flag, void* workspace, int64_t workspace_bytes, void* stream) {
  RetrieveWorkspace w{};
  RECNN_PROPAGATE(retrieve_topk_check(queries, n_queries, dim, table, n_items, norms, metric, k, ids_out, dist_out,
                                      workspace, workspace_bytes, &w));
  ItemSets ex;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_queries, error_flag, &ex));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  if (n_queries > 0) RECNN_PROPAGATE(item_sets_check(ex, n_queries, n_items, error_flag, st));
  return retrieve(queries, n_queries, dim, table, n_items, norms, metric, k, ex, ids_out, dist_out, w, st);
}

extern "C" int64_t recnn_retrieve_rank_workspace_bytes(int64_t n_queries, int64_t n_items) {
  if (n_queries <= 0 || n_items <= 0) return 0;
  return retrieve_carve(n_queries, n_items, 0, nullptr).bytes;
}

extern "C" int recnn_retrieve_rank(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                   int64_t n_items, const float* norms, int32_t metric, const int64_t* target,
                                   int64_t* rank_out, int32_t* error_flag, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  RetrieveWorkspace w{};
  RECNN_PROPAGATE(retrieve_rank_check(queries, n_queries, dim, table, n_items, norms, metric, target, rank_out,
                                      error_flag, workspace, workspace_bytes, &w));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  const ItemSets none = {nullptr, nullptr, nullptr, 0, 0, 0};
  return retrieve_rank(queries, n_queries, dim, table, n_items, norms, metric, target, none, rank_out, error_flag, w,
                       st);
}

extern "C" int recnn_retrieve_rank_sets(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                        int64_t n_items, const float* norms, int32_t metric, const int64_t* target,
                                        const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                                        int64_t n_sets, const int64_t* row_set, int64_t* rank_out,
                                        int32_t* error_flag, void* workspace, int64_t workspace_bytes, void* stream) {
  RetrieveWorkspace w{};
  RECNN_PROPAGATE(retrieve_rank_check(queries, n_queries, dim, table, n_items, norms, metric, target, rank_out,
                                      error_flag, workspace, workspace_bytes, &w));
  ItemSets ex;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_queries, error_flag, &ex));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  if (n_queries > 0) RECNN_PROPAGATE(item_sets_check(ex, n_queries, n_items, error_flag, st));
  return retrieve_rank(queries, n_queries, dim, table, n_items, norms, metric, target, ex, rank_out, error_flag, w, st);
}
