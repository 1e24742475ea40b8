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
// the CTA then merges its 256 sorted lists by k rounds of a block arg-min over the list heads; a second tiny
// kernel merges the column ranges of a query the same way.  Everything is exact (no approximate search).
#include <float.h>
#include <string.h>

#include "common.cuh"
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

// grid (splits, n_queries).  scores [n_queries, ld]; writes k candidates per (query, split), ascending.
template <int KMAX>
__global__ void __launch_bounds__(kTopkThreads)
topk_partial_kernel(const float* __restrict__ scores, long long ld, long long n_items, const float* __restrict__ norms,
                    int metric, int k, Cand* __restrict__ part) {
  __shared__ float s_key[32];
  __shared__ int s_id[32], s_owner[32];
  const int q = blockIdx.y, sp = blockIdx.x, splits = gridDim.x;
  const long long per = (n_items + splits - 1) / splits;
  const long long lo = sp * per, hi = min(n_items, lo + per);
  const float* row = scores + (long long)q * ld;
  float keys[KMAX];
  int ids[KMAX];
  list_clear(keys, ids);
  for (long long j = lo + threadIdx.x; j < hi; j += blockDim.x) {
    const float s = __ldcs(row + j);
    float key = metric == RECNN_METRIC_L2 ? fmaf(-2.0f, s, __ldg(norms + j))
              : metric == RECNN_METRIC_COS ? -s * __ldg(norms + j) : -s;
    if (!(key == key)) key = FLT_MAX;                 // NaN scores rank last
    int id = (int)j;
    if (better(key, id, keys[KMAX - 1], ids[KMAX - 1])) list_insert(keys, ids, key, id);
  }
  // merge the 256 sorted lists: k rounds of arg-min over the heads
  int head = 0;
  Cand* out = part + ((long long)q * splits + sp) * k;
  for (int r = 0; r < k; ++r) {
    float hk; int hid;
    list_at(keys, ids, head, hk, hid);
    float wk; int wi, wo;
    block_argmin(hk, hid, s_key, s_id, s_owner, wk, wi, wo);
    if ((int)threadIdx.x == wo) ++head;
    if (threadIdx.x == 0) { out[r].key = wk; out[r].id = wi; }
  }
}

// one warp per query: merge `splits` ascending lists of k candidates; finish the metric
__global__ void __launch_bounds__(128)
topk_merge_kernel(const Cand* __restrict__ part, int splits, int k, long long n_queries, int metric,
                  const float* __restrict__ queries, int dim, int64_t* __restrict__ ids_out, float* __restrict__ dist_out) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_queries) return;
  float qn = 0.f;
  for (int d = lane; d < dim; d += 32) { const float v = queries[q * dim + d]; qn = fmaf(v, v, qn); }
  qn = warp_sum(qn);
  const Cand* mine = part + q * (long long)splits * k;
  // lane l walks lists l, l+32, ...: keeps one head per owned list in a small loop (splits <= 32 in practice)
  int head = 0;                                      // lane's position in list `lane` (splits <= 32)
  for (int r = 0; r < k; ++r) {
    float key = FLT_MAX; int id = kNoId;
    if (lane < splits && head < k) { key = mine[(long long)lane * k + head].key; id = mine[(long long)lane * k + head].id; }
    int owner = lane;
    warp_argmin(key, id, owner);
    if (lane == owner) ++head;
    if (lane == 0) {
      float d;
      if (metric == RECNN_METRIC_L2) d = fmaxf(key + qn, 0.f);                 // squared L2 distance
      else if (metric == RECNN_METRIC_COS) d = -key / fmaxf(sqrtf(qn), 1e-30f);  // cosine similarity
      else d = -key;                                                           // inner product
      ids_out[q * k + r] = id == kNoId ? -1 : (int64_t)id;
      dist_out[q * k + r] = d;
    }
  }
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
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_COS, "norms exist for L2 and COS");
  const int64_t blocks = ceil_div(n_items, 8);
  item_norms_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(table, n_items, dim, metric, out);
  RECNN_CHECK_LAUNCH("item_norms_kernel");
  return RECNN_OK;
}

extern "C" int64_t recnn_retrieve_workspace_bytes(int64_t n_queries, int64_t n_items, int32_t k) {
  if (n_queries <= 0 || n_items <= 0 || k <= 0) return 0;
  return retrieve_carve(n_queries, n_items, k, nullptr).bytes;
}

extern "C" int recnn_retrieve_topk(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                   int64_t n_items, const float* norms, int32_t metric, int32_t k, int64_t* ids_out,
                                   float* dist_out, void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(queries && table && ids_out && dist_out && workspace, "null pointer");
  RECNN_REQUIRE(n_queries >= 0 && n_items > 0 && dim > 0, "sizes");
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_IP || metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(metric == RECNN_METRIC_IP || norms != nullptr, "L2 / COS need recnn_item_norms");
  RECNN_REQUIRE(k >= 1 && k <= 64 && k <= n_items, "1 <= k <= min(64, n_items)");
  RECNN_REQUIRE(n_items < (1ll << 31), "n_items must fit int32");
  if (n_queries == 0) return RECNN_OK;
  const RetrieveWorkspace w = retrieve_carve(n_queries, n_items, k, workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t ld = w.ld, slab = w.slab;
  float* scores = w.scores;
  Cand* part = w.part;
  const bool tc_ok = dim % 4 == 0 && (reinterpret_cast<uintptr_t>(queries) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(table) & 15) == 0;
  for (int64_t q0 = 0; q0 < n_queries; q0 += slab) {
    const int64_t nq = n_queries - q0 < slab ? n_queries - q0 : slab;
    const float* Q = queries + q0 * dim;
    Epilogue e;
    memset(&e, 0, sizeof(e));
    e.out = scores;
    e.ldo = ld;
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
    const int splits = topk_splits(nq, n_items, 32);
    dim3 grid((unsigned)splits, (unsigned)nq);
    if (k <= 16)
      topk_partial_kernel<16><<<grid, kTopkThreads, 0, st>>>(scores, ld, n_items, norms, metric, k, part);
    else
      topk_partial_kernel<64><<<grid, kTopkThreads, 0, st>>>(scores, ld, n_items, norms, metric, k, part);
    RECNN_CHECK_LAUNCH("topk_partial_kernel");
    topk_merge_kernel<<<(unsigned)ceil_div(nq, 4), 128, 0, st>>>(part, splits, k, nq, metric, Q, dim, ids_out + q0 * k,
                                                                  dist_out + q0 * k);
    RECNN_CHECK_LAUNCH("topk_merge_kernel");
  }
  return RECNN_OK;
}
