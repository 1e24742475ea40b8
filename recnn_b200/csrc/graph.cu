// A proximity-graph index over the embedding table in the style of CAGRA (Ootomo et al., arXiv:2308.15136; Milvus's
// GPU_CAGRA), built and searched on the device.  The index is n_items x degree int32 neighbour ids plus a few hundred
// entry points; it reads the resident table and keeps no copy of it.
//
// Build (recnn_graph_build), from the k-NN lists N(u) = [v_0 .. v_{D-1}] of every item (the host computes them with
// the exact or the IVF search):
//   prune      a warp per node, N(u) staged in shared memory: c_j = #{i < j : v_j is in N(v_i) at a position p < j}
//              (CAGRA's detour count); P(u) = the first d positions in (c_j, j) order
//   reverse    every kept edge u -> v at rank r of P(u) becomes the 64-bit key (v << 6 | r) with value u; CUB's stable
//              radix sort orders them by (v, r, u), so each node's reverse candidates come in (r, u) order
//   merge      a warp per node: the first d/2 of P(v), then its reverse candidates, then the rest of P(v), each
//              skipping ids already present, until d are held
// Every step is a function of the k-NN ids only, with integer counts and no float atomics: a build is bit-reproducible.
//
// Search (recnn_graph_search), one CTA per query, everything in shared memory:
//   buffer     T (key, id, explored) entries sorted by (key, id), starting empty {FLT_MAX, kNoId}
//   iteration  0: the first W * d entry points are the candidates; then each iteration takes the W best unexplored
//              entries as parents and their out-lists as the candidates
//   visited    a shared hash of every id keyed so far drops repeats (a candidate already in the buffer, or a copy
//              within the iteration); once half full it is cleared and refilled with the buffer's ids.  An id that
//              left the buffer, or never entered it, is worse than the T-th entry, which never gets worse, so keying
//              it again could not change the buffer: the result is the one an exact "in the buffer" check gives.
//   keys       a warp scores four candidate rows at a time, straight from the table: lane l accumulates
//              q[t] * x[t] for t = l, l + 32, ... by fp32 fma in ascending t, then warp_sum and lane 0's value, then
//              metric_key (topk.cuh).  A key's bits depend only on the query, the item and dim.
//   merge      the candidates are bitonic-sorted in shared memory, then merged with the buffer by rank (each entry's
//              position is its index plus its count of smaller entries in the other list); the best T stay
// A second kernel (a warp per query) drops the excluded items from the final buffer and reports the k best eligible
// ones through metric_distance, as the flat search does.
#include <float.h>
#include <stddef.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>

#include "common.cuh"
#include "topk.cuh"

namespace recnn {

constexpr int kGraphMaxDim = 512;      // a lane keeps at most 16 elements of a row in flight
constexpr int kGraphMaxKnn = 64;       // D: the k-NN lists come from a k <= 64 search
constexpr int kGraphMaxEntry = 512;    // entry points stored with the index
constexpr int kGraphMaxCand = 512;     // W * d
constexpr int kGraphThreads = 256;     // a search CTA
constexpr int kGraphRows = 4;          // candidate rows a warp scores at once
constexpr int kGraphHash = 4096;       // visited-hash slots (a power of two)
constexpr int kGraphHashFill = 2048;   // the hash is cleared before an iteration would take it past this
constexpr int kGraphRevBits = 6;       // rank bits of a reverse-edge key: r < d <= 64

// ------------------------------------------------------------------------------------------------------------ build
// A warp per node u (4 per CTA).  flag |= 1 for a k-NN id outside [0, n), |= 2 for u itself or a repeated id in N(u);
// such a row still gets a graph row, but one no search should use.
__global__ void __launch_bounds__(128)
graph_prune_kernel(const long long* __restrict__ knn, int D, long long n, int d, int* __restrict__ pruned,
                   int* __restrict__ flag) {
  __shared__ int s_v[4][kGraphMaxKnn], s_sid[4][kGraphMaxKnn], s_spos[4][kGraphMaxKnn], s_c[4][kGraphMaxKnn];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long u = (long long)blockIdx.x * 4 + w;
  if (u >= n) return;
  int *v = s_v[w], *sid = s_sid[w], *spos = s_spos[w], *c = s_c[w];
  int bad = 0;
  for (int j = lane; j < D; j += 32) {
    const long long x = knn[u * D + j];
    const bool in = x >= 0 && x < n;
    bad |= in ? (x == u ? 2 : 0) : 1;
    v[j] = in ? (int)x : -1;
    c[j] = 0;
  }
  __syncwarp();
  // N(u) sorted by id (rank by counting; a repeated id is reported and keeps distinct ranks), for the lookups below
  for (int j = lane; j < D; j += 32) {
    const int x = v[j];
    int r = 0;
    for (int t = 0; t < D; ++t) {
      const int y = v[t];
      r += y < x || (y == x && t < j);
      if (y == x && t != j) bad |= 2;
    }
    sid[r] = x;
    spos[r] = j;
  }
  bad = __reduce_or_sync(0xffffffffu, bad);
  if (lane == 0 && bad) atomicOr(flag, bad);
  __syncwarp();
  // detours: for each i, the entries p < D - 1 of N(v_i) that sit in N(u) at a position j > max(i, p)
  for (int i = 0; i < D - 1; ++i) {
    const int vi = v[i];
    if (vi < 0) continue;                                   // the same decision in every lane
    const long long* row = knn + (long long)vi * D;
    for (int p = lane; p < D - 1; p += 32) {
      const long long x = __ldg(row + p);
      if (x < 0 || x >= n) continue;
      int lo = 0, hi = D;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (sid[mid] < (int)x) lo = mid + 1; else hi = mid;
      }
      if (lo < D && sid[lo] == (int)x) {
        const int j = spos[lo];
        if (j > i && p < j) atomicAdd(c + j, 1);
      }
    }
  }
  __syncwarp();
  // P(u): the positions in (c_j, j) order, the first d of them
  for (int j = lane; j < D; j += 32) {
    const int cj = c[j];
    int r = 0;
    for (int t = 0; t < D; ++t) r += c[t] < cj || (c[t] == cj && t < j);
    if (r < d) pruned[u * d + r] = v[j];
  }
}

// the sort's input: key = (v << 6 | r) for the kept edge u -> v at rank r, value = u; input order (u, r)
__global__ void graph_rev_keys_kernel(const int* __restrict__ pruned, long long edges, int d,
                                      unsigned long long* __restrict__ keys, int* __restrict__ vals) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= edges) return;
  const int v = pruned[e];
  keys[e] = ((unsigned long long)(v < 0 ? 0 : v) << kGraphRevBits) | (unsigned long long)(e % d);
  vals[e] = (int)(e / d);
}

// offs[v] = the first sorted position whose node is >= v, v in [0, n]
__global__ void graph_rev_offsets_kernel(const unsigned long long* __restrict__ keys, long long edges, long long n,
                                         long long* __restrict__ offs) {
  const long long v = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (v > n) return;
  long long lo = 0, hi = edges;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if ((long long)(keys[mid] >> kGraphRevBits) < v) lo = mid + 1; else hi = mid;
  }
  offs[v] = lo;
}

// A warp per node v: out = P(v)[0, d/2), then the reverse candidates in (r, u) order, then P(v)[d/2, d), each id
// appended when not already present, until d are held
__global__ void __launch_bounds__(128)
graph_merge_kernel(const int* __restrict__ pruned, int d, long long n, const long long* __restrict__ offs,
                   const int* __restrict__ rev, int* __restrict__ graph) {
  __shared__ int s_out[4][kGraphMaxKnn];
  const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long v = (long long)blockIdx.x * 4 + w;
  if (v >= n) return;
  int* out = s_out[w];
  const int* P = pruned + v * d;
  const int half = d / 2;
  for (int j = lane; j < half; j += 32) out[j] = P[j];
  int cnt = half;
  __syncwarp();
  auto offer = [&](int x) {                                 // every lane, the same x
    bool dup = false;
    for (int t = lane; t < cnt; t += 32) dup |= out[t] == x;
    if (!__any_sync(0xffffffffu, dup)) {
      if (lane == 0) out[cnt] = x;
      ++cnt;
      __syncwarp();
    }
  };
  for (long long e = offs[v]; e < offs[v + 1] && cnt < d; ++e) offer(rev[e]);
  for (int j = half; j < d && cnt < d; ++j) offer(P[j]);
  __syncwarp();
  for (int j = lane; j < d; j += 32) graph[v * d + j] = out[j];
}

// ----------------------------------------------------------------------------------------------------------- search
struct GraphView {
  const float* table;
  const float* norms;
  const int* graph;
  const int* entry;
  long long n;
  int dim, metric, degree, n_entry;
};

// insert id into the shared open-addressing hash; true when it was absent
__device__ __forceinline__ bool hash_insert(int* h, int id) {
  unsigned s = ((unsigned)id * 0x9E3779B1u) >> 20;          // 12 bits: kGraphHash slots
  for (;;) {
    const int prev = atomicCAS(h + s, -1, id);
    if (prev == -1) return true;
    if (prev == id) return false;
    s = (s + 1) & (kGraphHash - 1);
  }
}

__device__ __forceinline__ bool cand_le(float ka, int ia, float kb, int ib) {
  return better(ka, ia, kb, ib) || (ka == kb && ia == ib);
}

// One CTA per query.  Writes the final buffer, sorted by (key, id), to buf_out[q * T .. + T) and the number of
// iterations after iteration 0 to iters_out[q] (when given).
__global__ void __launch_bounds__(kGraphThreads)
graph_search_kernel(const float* __restrict__ queries, GraphView g, int T, int W, int max_iter, int C,
                    Cand* __restrict__ buf_out, int* __restrict__ iters_out) {
  extern __shared__ __align__(16) unsigned char smem[];
  __shared__ int s_par[8];
  __shared__ int s_np, s_fill;
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
  const int dim = g.dim, d = g.degree;
  float* s_q = reinterpret_cast<float*>(smem);                       // [dim rounded up to 4]
  // the buffer (keys, ids, explored) and the merge's output, swapped after every merge
  float* bk = s_q + ((dim + 3) & ~3);
  int* bi = reinterpret_cast<int*>(bk + T);
  int* be = bi + T;
  float* nk = reinterpret_cast<float*>(be + T);
  int* ni = reinterpret_cast<int*>(nk + T);
  int* ne = ni + T;
  float* s_ck = reinterpret_cast<float*>(ne + T);                // candidates [C]
  int* s_ci = reinterpret_cast<int*>(s_ck + C);
  int* s_hash = s_ci + C;                                             // [kGraphHash]

  for (int t = tid; t < dim; t += blockDim.x) s_q[t] = queries[q * dim + t];
  for (int t = tid; t < T; t += blockDim.x) { bk[t] = FLT_MAX; bi[t] = kNoId; be[t] = 0; }
  for (int t = tid; t < kGraphHash; t += blockDim.x) s_hash[t] = -1;
  if (tid == 0) s_fill = 0;
  int it = 0;
  int nc = min(W * d, g.n_entry);
  int fill = 0;                      // s_fill as of the last merge, read where no thread can be adding to it
  __syncthreads();

  for (;;) {
    // the hash is cleared and refilled with the buffer's ids before this iteration could overfill it (fill is the
    // same register value in every thread, so every thread takes the same branch and meets the same barriers)
    if (fill + nc > kGraphHashFill) {
      for (int t = tid; t < kGraphHash; t += blockDim.x) s_hash[t] = -1;
      __syncthreads();
      if (tid == 0) s_fill = 0;
      __syncthreads();
      for (int t = tid; t < T; t += blockDim.x)
        if (bi[t] != kNoId && hash_insert(s_hash, bi[t])) atomicAdd(&s_fill, 1);
      __syncthreads();
    }
    // 1. the candidates' ids; a repeat becomes an empty slot
    for (int c = tid; c < C; c += blockDim.x) {
      int id = kNoId;
      if (c < nc) {
        id = it == 0 ? __ldg(g.entry + c) : __ldg(g.graph + (long long)s_par[c / d] * d + c % d);
        if (hash_insert(s_hash, id)) atomicAdd(&s_fill, 1);
        else id = kNoId;
      }
      s_ci[c] = id;
      s_ck[c] = FLT_MAX;
    }
    __syncthreads();
    // 2. keys: a warp scores kGraphRows candidates at once
    for (int c0 = warp * kGraphRows; c0 < nc; c0 += nw * kGraphRows) {
      int ids[kGraphRows];
      float acc[kGraphRows];
#pragma unroll
      for (int r = 0; r < kGraphRows; ++r) {
        ids[r] = c0 + r < nc ? s_ci[c0 + r] : kNoId;
        acc[r] = 0.f;
      }
      // every load first (up to 64 per lane in flight), then the sums in ascending t
      float x[kGraphMaxDim / 32][kGraphRows];
#pragma unroll
      for (int i = 0; i < kGraphMaxDim / 32; ++i) {
        const int t = lane + 32 * i;
#pragma unroll
        for (int r = 0; r < kGraphRows; ++r)
          x[i][r] = t < dim && ids[r] != kNoId ? __ldg(g.table + (long long)ids[r] * dim + t) : 0.f;
      }
#pragma unroll
      for (int i = 0; i < kGraphMaxDim / 32; ++i) {
        const int t = lane + 32 * i;
        if (t < dim) {
          const float qv = s_q[t];
#pragma unroll
          for (int r = 0; r < kGraphRows; ++r) acc[r] = fmaf(qv, x[i][r], acc[r]);
        }
      }
#pragma unroll
      for (int r = 0; r < kGraphRows; ++r) {
        const float s = warp_sum(acc[r]);
        if (lane == 0 && ids[r] != kNoId) s_ck[c0 + r] = metric_key(s, g.norms, ids[r], g.metric);
      }
    }
    __syncthreads();
    // 3. bitonic sort of the C candidates by (key, id)
    for (int size = 2; size <= C; size <<= 1) {
      for (int stride = size >> 1; stride > 0; stride >>= 1) {
        for (int p = tid; p < C / 2; p += blockDim.x) {
          const int lo = 2 * stride * (p / stride) + (p % stride), hi = lo + stride;
          const bool up = (lo & size) == 0;
          const float ka = s_ck[lo], kb = s_ck[hi];
          const int ia = s_ci[lo], ib = s_ci[hi];
          if (better(kb, ib, ka, ia) == up) { s_ck[lo] = kb; s_ci[lo] = ib; s_ck[hi] = ka; s_ci[hi] = ia; }
        }
        __syncthreads();
      }
    }
    // 4. merge by rank into the other buffer: the best T of buffer + candidates (buffer entries first on a tie,
    // which only empty slots can make)
    for (int t = tid; t < T + C; t += blockDim.x) {
      float k; int id, ex, pos;
      if (t < T) {
        k = bk[t]; id = bi[t]; ex = be[t];
        int lo = 0, hi = C;                                 // candidates strictly before it
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (better(s_ck[mid], s_ci[mid], k, id)) lo = mid + 1; else hi = mid;
        }
        pos = t + lo;
      } else {
        const int c = t - T;
        k = s_ck[c]; id = s_ci[c]; ex = 0;
        int lo = 0, hi = T;                                 // buffer entries at or before it
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (cand_le(bk[mid], bi[mid], k, id)) lo = mid + 1; else hi = mid;
        }
        pos = c + lo;
      }
      if (pos < T) { nk[pos] = k; ni[pos] = id; ne[pos] = ex; }
    }
    __syncthreads();
    fill = s_fill;                   // step 1's inserts are behind the barriers above, the next ones behind the next
    { float* t = bk; bk = nk; nk = t; }
    { int* t = bi; bi = ni; ni = t; }
    { int* t = be; be = ne; ne = t; }
    if (max_iter > 0 && it >= max_iter) break;
    // 5. parents: the W best unexplored entries, marked explored
    if (warp == 0) {
      int np = 0;
      for (int base = 0; base < T && np < W; base += 32) {
        const int t = base + lane;
        const bool un = be[t] == 0 && bi[t] != kNoId;
        const unsigned m = __ballot_sync(0xffffffffu, un);
        const int before = __popc(m & ((1u << lane) - 1u));
        if (un && np + before < W) {
          s_par[np + before] = bi[t];
          be[t] = 1;
        }
        np += __popc(m);
      }
      if (lane == 0) s_np = min(np, W);
    }
    __syncthreads();
    if (s_np == 0) break;
    nc = s_np * d;
    ++it;
  }
  for (int t = tid; t < T; t += blockDim.x) buf_out[q * T + t] = Cand{bk[t], bi[t]};
  if (iters_out && tid == 0) iters_out[q] = it;
}

// A warp per query: the k best eligible entries of the final buffer, reported as the flat search reports them; fewer
// than k eligible ones end in id -1 and the metric's pad distance
__global__ void __launch_bounds__(128)
graph_finish_kernel(const Cand* __restrict__ buf, int T, int k, long long n_queries, int metric,
                    const float* __restrict__ queries, int dim, ItemSets ex, int64_t* __restrict__ ids_out,
                    float* __restrict__ dist_out) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_queries) return;
  const float qn = warp_sq_norm(queries + q * dim, dim);
  SetView set = {nullptr, 0, false};
  if (ex.ids) {
    long long a, b;
    set_segment(ex, q, a, b);
    set.g = ex.ids + a;
    set.n = b - a;
  }
  int written = 0;
  for (int base = 0; base < T && written < k; base += 32) {
    const Cand c = buf[q * T + base + lane];
    const bool ok = c.id != kNoId && (set.n == 0 || !set_has(set, nullptr, c.id));
    const unsigned m = __ballot_sync(0xffffffffu, ok);
    const int pos = written + __popc(m & ((1u << lane) - 1u));
    if (ok && pos < k) {
      ids_out[q * k + pos] = c.id;
      dist_out[q * k + pos] = metric_distance(c.key, c.id, qn, metric);
    }
    written += __popc(m);
  }
  for (int r = min(written, k) + lane; r < k; r += 32) {
    ids_out[q * k + r] = -1;
    dist_out[q * k + r] = metric_distance(FLT_MAX, kNoId, qn, metric);
  }
}

// ------------------------------------------------------------------------------------------------------- workspaces
static int rev_end_bit(int64_t n) {
  int b = 1;
  while ((1ll << b) < n) ++b;
  return b + kGraphRevBits;
}

struct GraphBuildWorkspace {
  int* pruned;                      // [n, d] P(u)
  unsigned long long *keys_in, *keys_out;
  int *vals_in, *vals_out;          // [n * d] each
  long long* offs;                  // [n + 1] reverse-candidate ranges
  void* sort_tmp;
  size_t sort_bytes;
  int64_t bytes;
};

static GraphBuildWorkspace build_carve(int64_t n, int d, void* base) {
  GraphBuildWorkspace w;
  Carve c(base);
  const int64_t edges = n * d;
  w.pruned = c.take<int>(edges);
  w.keys_in = c.take<unsigned long long>(edges);
  w.keys_out = c.take<unsigned long long>(edges);
  w.vals_in = c.take<int>(edges);
  w.vals_out = c.take<int>(edges);
  w.offs = c.take<long long>(n + 1);
  w.sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, w.sort_bytes, (const unsigned long long*)nullptr,
                                  (unsigned long long*)nullptr, (const int*)nullptr, (int*)nullptr, (int)edges, 0,
                                  rev_end_bit(n));
  w.sort_tmp = c.take<char>((int64_t)w.sort_bytes);
  w.bytes = c.bytes();
  return w;
}

struct GraphSearchWorkspace {
  Cand* buf;          // [n_queries, T] the final buffers
  int64_t bytes;
};

static GraphSearchWorkspace search_carve(int64_t n_queries, int T, void* base) {
  GraphSearchWorkspace w;
  Carve c(base);
  w.buf = c.take<Cand>(n_queries * T);
  w.bytes = c.bytes();
  return w;
}

static int pow2_at_least(int x) {
  int p = 1;
  while (p < x) p <<= 1;
  return p;
}

static int graph_smem_bytes(int dim, int T, int C) {
  return (int)sizeof(float) * ((dim + 3) / 4 * 4 + 6 * T + 2 * C + kGraphHash);
}

static bool graph_degree_ok(int d) { return d == 16 || d == 32 || d == 64; }

static int graph_index_check(const recnn_graph_index& x) {
  RECNN_REQUIRE(x.table && x.graph && x.entry, "null pointer");
  RECNN_REQUIRE(x.metric == RECNN_METRIC_L2 || x.metric == RECNN_METRIC_IP || x.metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(x.metric == RECNN_METRIC_IP || x.norms, "L2 / COS need the norms");
  RECNN_REQUIRE(graph_degree_ok(x.degree), "degree in {16, 32, 64}");
  RECNN_REQUIRE(x.n_items > x.degree && x.n_items < (1ll << 31), "degree < n_items < 2^31");
  RECNN_REQUIRE(x.dim >= 1 && x.dim <= kGraphMaxDim, "1 <= dim <= 512");
  RECNN_REQUIRE(x.n_entry >= 1 && x.n_entry <= kGraphMaxEntry && x.n_entry <= x.n_items,
                "1 <= n_entry <= min(512, n_items)");
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

extern "C" int64_t recnn_graph_build_workspace_bytes(int64_t n_items, int32_t degree) {
  if (!graph_degree_ok(degree) || n_items <= degree || n_items >= (1ll << 31) || n_items * degree >= (1ll << 31))
    return 0;
  return build_carve(n_items, degree, nullptr).bytes;
}

extern "C" int64_t recnn_graph_search_workspace_bytes(int64_t n_queries, int32_t itopk) {
  if (n_queries <= 0 || itopk < 32 || itopk > 256 || itopk % 32 != 0) return 0;
  return search_carve(n_queries, itopk, nullptr).bytes;
}

extern "C" int64_t recnn_sizeof_graph_index(void) { return (int64_t)sizeof(recnn_graph_index); }
extern "C" int64_t recnn_sizeof_graph_build_args(void) { return (int64_t)sizeof(recnn_graph_build_args); }
extern "C" int64_t recnn_sizeof_graph_search_args(void) { return (int64_t)sizeof(recnn_graph_search_args); }

extern "C" int64_t recnn_offsetof_graph_build_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_graph_build_args, index);
    case 1: return offsetof(recnn_graph_build_args, knn);
    case 2: return offsetof(recnn_graph_build_args, knn_degree);
    case 3: return offsetof(recnn_graph_build_args, error_flag);
    case 4: return offsetof(recnn_graph_build_args, workspace);
    case 5: return offsetof(recnn_graph_build_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int64_t recnn_offsetof_graph_search_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_graph_search_args, index);
    case 1: return offsetof(recnn_graph_search_args, queries);
    case 2: return offsetof(recnn_graph_search_args, n_queries);
    case 3: return offsetof(recnn_graph_search_args, k);
    case 4: return offsetof(recnn_graph_search_args, itopk);
    case 5: return offsetof(recnn_graph_search_args, search_width);
    case 6: return offsetof(recnn_graph_search_args, max_iterations);
    case 7: return offsetof(recnn_graph_search_args, set_ids);
    case 8: return offsetof(recnn_graph_search_args, n_set_ids);
    case 9: return offsetof(recnn_graph_search_args, set_offsets);
    case 10: return offsetof(recnn_graph_search_args, n_sets);
    case 11: return offsetof(recnn_graph_search_args, row_set);
    case 12: return offsetof(recnn_graph_search_args, ids_out);
    case 13: return offsetof(recnn_graph_search_args, dist_out);
    case 14: return offsetof(recnn_graph_search_args, iterations_out);
    case 15: return offsetof(recnn_graph_search_args, error_flag);
    case 16: return offsetof(recnn_graph_search_args, workspace);
    case 17: return offsetof(recnn_graph_search_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int recnn_graph_build(const recnn_graph_build_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_graph_index& x = a->index;
  RECNN_REQUIRE(x.graph && a->knn && a->error_flag && a->workspace, "null pointer");
  RECNN_REQUIRE(graph_degree_ok(x.degree), "degree in {16, 32, 64}");
  RECNN_REQUIRE(a->knn_degree >= x.degree && a->knn_degree <= kGraphMaxKnn, "degree <= knn_degree <= 64");
  RECNN_REQUIRE(x.n_items > a->knn_degree, "knn_degree < n_items");
  RECNN_REQUIRE(x.n_items < (1ll << 31) && x.n_items * x.degree < (1ll << 31),
                "n_items * degree < 2^31: the reverse-edge sort counts in int32");
  const int64_t n = x.n_items;
  const int d = x.degree, D = a->knn_degree;
  const GraphBuildWorkspace w = build_carve(n, d, a->workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, a->workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(a->error_flag, 0, sizeof(int32_t), st));
  const unsigned warps4 = (unsigned)ceil_div(n, 4);
  graph_prune_kernel<<<warps4, 128, 0, st>>>(reinterpret_cast<const long long*>(a->knn), D, n, d, w.pruned,
                                             a->error_flag);
  RECNN_CHECK_LAUNCH("graph_prune_kernel");
  const int64_t edges = n * d;
  graph_rev_keys_kernel<<<(unsigned)ceil_div(edges, 256), 256, 0, st>>>(w.pruned, edges, d, w.keys_in, w.vals_in);
  RECNN_CHECK_LAUNCH("graph_rev_keys_kernel");
  size_t bytes = w.sort_bytes;
  RECNN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out,
                                                   (int)edges, 0, rev_end_bit(n), st));
  count_launch();
  graph_rev_offsets_kernel<<<(unsigned)ceil_div(n + 1, 256), 256, 0, st>>>(w.keys_out, edges, n, w.offs);
  RECNN_CHECK_LAUNCH("graph_rev_offsets_kernel");
  graph_merge_kernel<<<warps4, 128, 0, st>>>(w.pruned, d, n, w.offs, w.vals_out, x.graph);
  RECNN_CHECK_LAUNCH("graph_merge_kernel");
  return RECNN_OK;
}

extern "C" int recnn_graph_search(const recnn_graph_search_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_graph_index& x = a->index;
  RECNN_PROPAGATE(graph_index_check(x));
  RECNN_REQUIRE(a->queries && a->ids_out && a->dist_out && a->workspace, "null pointer");
  RECNN_REQUIRE(a->n_queries >= 0, "n_queries >= 0");
  const int T = a->itopk, W = a->search_width, k = a->k;
  RECNN_REQUIRE(T >= 32 && T <= 256 && T % 32 == 0, "itopk a multiple of 32 in [32, 256]");
  RECNN_REQUIRE(k >= 1 && k <= 64 && k <= T, "1 <= k <= min(64, itopk)");
  RECNN_REQUIRE(W >= 1 && W <= 8 && W * x.degree <= kGraphMaxCand, "1 <= search_width <= 8, search_width * degree <= 512");
  RECNN_REQUIRE(a->max_iterations >= 0, "max_iterations >= 0");
  if (a->n_queries == 0) return RECNN_OK;
  RECNN_REQUIRE(a->n_queries < (1ll << 31), "n_queries < 2^31");
  const GraphSearchWorkspace w = search_carve(a->n_queries, T, a->workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, a->workspace_bytes));
  ItemSets ex = {nullptr, nullptr, nullptr, 0, 0, 0};
  const bool sets = a->set_offsets != nullptr;
  if (sets)
    RECNN_PROPAGATE(item_sets_args(a->set_ids, a->n_set_ids, a->set_offsets, a->n_sets, a->row_set, a->n_queries,
                                   a->error_flag, &ex));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (sets) {
    RECNN_CHECK_CUDA(cudaMemsetAsync(a->error_flag, 0, sizeof(int32_t), st));
    RECNN_PROPAGATE(item_sets_check(ex, a->n_queries, x.n_items, a->error_flag, st));
  }
  const GraphView g = {x.table, x.norms, x.graph, x.entry, x.n_items, x.dim, x.metric, x.degree, x.n_entry};
  const int C = pow2_at_least(W * x.degree);
  graph_search_kernel<<<(unsigned)a->n_queries, kGraphThreads, graph_smem_bytes(x.dim, T, C), st>>>(
      a->queries, g, T, W, a->max_iterations, C, w.buf, a->iterations_out);
  RECNN_CHECK_LAUNCH("graph_search_kernel");
  graph_finish_kernel<<<(unsigned)ceil_div(a->n_queries, 4), 128, 0, st>>>(w.buf, T, k, a->n_queries, x.metric,
                                                                           a->queries, x.dim, ex, a->ids_out,
                                                                           a->dist_out);
  RECNN_CHECK_LAUNCH("graph_finish_kernel");
  return RECNN_OK;
}
