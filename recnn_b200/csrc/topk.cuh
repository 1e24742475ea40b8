// Exact top-k building blocks shared by every selector: nearest-item retrieval (retrieval.cu, ivf.cu, ivf_pq.cu), the
// REINFORCE policy's top-k and sampled slates (reinforce.cuh) and Q-scored critic serving (critic_serve.cuh).  A
// candidate is (key, id), smaller key first, ties towards the smaller id (== a stable argsort of the keys); an empty
// slot is {FLT_MAX, kNoId}.  Every selector builds its keys through finite_key (NaN and +inf rank as FLT_MAX), and the
// retrieval ones through metric_key, so that a flat search, an IVF search probing every list and a rank see the same
// key bits.  Each thread keeps the best KMAX of its share in a sorted register list; a CTA merges its lists with
// block_merge, and a warp merges sorted lists in memory (the CTAs' outputs) with warp_merge.  The retrieval merges
// report a key as a distance through metric_distance.
#pragma once

#include <float.h>
#include <limits.h>

#include "common.cuh"

namespace recnn {

struct Cand {
  float key;
  int id;
};
constexpr int kNoId = 0x7fffffff;     // the id of an empty slot (key FLT_MAX): worse than every real candidate
constexpr int kTopkThreads = 256;     // threads of a CTA that keeps register lists

// column ranges per row of a [n_rows, n_items] score block: enough CTAs for two waves when rows are few, at least
// 4 * kTopkThreads columns per range, at most `cap` ranges (the merge gives each range a lane of one warp)
static inline int topk_splits(int64_t n_rows, int64_t n_items, int cap) {
  int64_t s = ceil_div(2 * kNumSMs, n_rows);
  const int64_t max_by_items = ceil_div(n_items, 4 * kTopkThreads);
  if (s > max_by_items) s = max_by_items;
  if (s > cap) s = cap;
  return (int)(s < 1 ? 1 : s);
}

__device__ __forceinline__ bool better(float ka, int ia, float kb, int ib) { return ka < kb || (ka == kb && ia < ib); }

// A ranking key as every selector stores it: NaN and +inf become FLT_MAX (fminf returns the other operand of a NaN), so
// such an item ranks after every finite key, ties by id, and still before an empty slot {FLT_MAX, kNoId}: it is
// returned before any "fewer than k eligible items" pad.  -inf stays the best key.
__device__ __forceinline__ float finite_key(float key) { return fminf(key, FLT_MAX); }

// block arg-min over one candidate per thread; returns the winner's (key, id, owner thread) to every thread
__device__ __forceinline__ void block_argmin(float key, int id, float* s_key, int* s_id, int* s_owner, float& wk,
                                             int& wi, int& wo) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int owner = threadIdx.x;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float k2 = __shfl_xor_sync(0xffffffffu, key, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, id, o);
    const int o2 = __shfl_xor_sync(0xffffffffu, owner, o);
    if (better(k2, i2, key, id)) { key = k2; id = i2; owner = o2; }
  }
  __syncthreads();
  if (lane == 0) { s_key[warp] = key; s_id[warp] = id; s_owner[warp] = owner; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    key = lane < nw ? s_key[lane] : FLT_MAX;
    id = lane < nw ? s_id[lane] : kNoId;
    owner = lane < nw ? s_owner[lane] : -1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float k2 = __shfl_xor_sync(0xffffffffu, key, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, id, o);
      const int o2 = __shfl_xor_sync(0xffffffffu, owner, o);
      if (better(k2, i2, key, id)) { key = k2; id = i2; owner = o2; }
    }
    if (lane == 0) { s_key[0] = key; s_id[0] = id; s_owner[0] = owner; }
  }
  __syncthreads();
  wk = s_key[0]; wi = s_id[0]; wo = s_owner[0];
}

// warp arg-min: the winner's (key, id, owner lane) in every lane
__device__ __forceinline__ void warp_argmin(float& key, int& id, int& owner) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float k2 = __shfl_xor_sync(0xffffffffu, key, o);
    const int i2 = __shfl_xor_sync(0xffffffffu, id, o);
    const int o2 = __shfl_xor_sync(0xffffffffu, owner, o);
    if (better(k2, i2, key, id)) { key = k2; id = i2; owner = o2; }
  }
}

template <int KMAX>
__device__ __forceinline__ void list_clear(float (&keys)[KMAX], int (&ids)[KMAX]) {
#pragma unroll
  for (int i = 0; i < KMAX; ++i) { keys[i] = FLT_MAX; ids[i] = kNoId; }
}

// sorted insertion of (key, id) by a chain of compare-exchanges (fully unrolled: the list stays in registers).  The
// caller has checked that the candidate beats the list's worst, keys[KMAX - 1].
template <int KMAX>
__device__ __forceinline__ void list_insert(float (&keys)[KMAX], int (&ids)[KMAX], float key, int id) {
#pragma unroll
  for (int i = 0; i < KMAX; ++i) {
    if (better(key, id, keys[i], ids[i])) {
      const float tk = keys[i]; const int ti = ids[i];
      keys[i] = key; ids[i] = id;
      key = tk; id = ti;
    }
  }
}

// entry `head` of a register list (an unrolled select: a dynamic index would move the list to local memory)
template <int KMAX>
__device__ __forceinline__ void list_at(const float (&keys)[KMAX], const int (&ids)[KMAX], int head, float& k, int& id) {
  k = FLT_MAX; id = kNoId;
#pragma unroll
  for (int i = 0; i < KMAX; ++i) if (i == head) { k = keys[i]; id = ids[i]; }
}

// Called by every thread of the CTA: merges the threads' sorted register lists into out[0, k), ascending, by rounds of
// block_argmin over the list heads; thread 0 writes each winner.  Once a round's winner is an empty slot every list is
// exhausted (a real candidate, NaN-keyed included, has a real id), so the rounds stop there and the rest of out is
// padded with empty slots: the bytes k rounds would write.
template <int KMAX>
__device__ __forceinline__ void block_merge(const float (&keys)[KMAX], const int (&ids)[KMAX], int k, Cand* out) {
  __shared__ float s_key[32];
  __shared__ int s_id[32], s_owner[32];
  int head = 0, i = 0;
  for (; i < k; ++i) {
    float hk, wk;
    int hid, wi, wo;
    list_at(keys, ids, head, hk, hid);
    block_argmin(hk, hid, s_key, s_id, s_owner, wk, wi, wo);
    if (wi == kNoId) break;                               // the same decision in every thread
    if ((int)threadIdx.x == wo) ++head;
    if (threadIdx.x == 0) out[i] = Cand{wk, wi};
  }
  for (int j = i + threadIdx.x; j < k; j += blockDim.x) out[j] = Cand{FLT_MAX, kNoId};
}

// Called by a whole warp: the k best of up to 32 * LISTS sorted candidate lists, lane l owning lists l, l + 32, ...
// read(list, pos) returns entry pos of a list, {FLT_MAX, kNoId} past its end or for a list that does not exist; it is
// called once per list a lane owns in every round, before the round's arg-min.  emit(i, key, id, owner) runs in every
// lane for the i-th best, i = 0 .. k - 1, owner being the lane whose list held it.
template <int LISTS, class Read, class Emit>
__device__ __forceinline__ void warp_merge(int k, Read read, Emit emit) {
  const int lane = threadIdx.x & 31;
  int head[LISTS];
#pragma unroll
  for (int l = 0; l < LISTS; ++l) head[l] = 0;
  for (int i = 0; i < k; ++i) {
    Cand c = read(lane, head[0]);
    int from = 0;
#pragma unroll
    for (int l = 1; l < LISTS; ++l) {
      const Cand o = read(lane + 32 * l, head[l]);
      if (better(o.key, o.id, c.key, c.id)) { c = o; from = l; }
    }
    int owner = lane;
    warp_argmin(c.key, c.id, owner);
#pragma unroll
    for (int l = 0; l < LISTS; ++l) if (lane == owner && l == from) ++head[l];
    emit(i, c.key, c.id, owner);
  }
}

// The ranking key of item j with inner product s under a retrieval metric: |t_j|^2 - 2 s (L2, norms[j] = |t_j|^2),
// -s / |t_j| (COS, norms[j] = 1 / |t_j|), -s (IP: norms is not read and may be NULL); for the metrics from L1 on, s is
// already the distance (distance.cuh) and is its own key.  Every retrieval search and rank keys its items here, so
// their results agree bit for bit.
__device__ __forceinline__ float metric_key(float s, const float* __restrict__ norms, long long j, int metric) {
  return finite_key(metric == RECNN_METRIC_L2 ? fmaf(-2.0f, s, __ldg(norms + j))
                    : metric == RECNN_METRIC_COS ? -s * __ldg(norms + j)
                    : metric == RECNN_METRIC_IP ? -s : s);
}

// Called by a whole warp: |row|^2, lane l summing d = l, l + 32, ... by fma, then the butterfly sum; in every lane
__device__ __forceinline__ float warp_sq_norm(const float* row, int dim) {
  float s = 0.f;
  for (int d = threadIdx.x & 31; d < dim; d += 32) { const float v = row[d]; s = fmaf(v, v, s); }
  return warp_sum(s);
}

// The distance a search reports for a metric_key key, qn = |query|^2: the squared L2 distance, the inner product, the
// cosine similarity, or the key itself for the metrics from L1 on; an empty slot (fewer than k eligible items) reports
// -FLT_MAX (IP, COS) or FLT_MAX (the others).
__device__ __forceinline__ float metric_distance(float key, int id, float qn, int metric) {
  float d;
  if (metric == RECNN_METRIC_L2) d = fmaxf(key + qn, 0.f);
  else if (metric == RECNN_METRIC_COS) d = -key / fmaxf(sqrtf(qn), 1e-30f);
  else if (metric == RECNN_METRIC_IP) d = -key;
  else d = key;
  if (id == kNoId) d = metric == RECNN_METRIC_IP || metric == RECNN_METRIC_COS ? -FLT_MAX : FLT_MAX;
  return d;
}

// ---- Item-set exclusion: the ids a row must never return ----------------------------------------------------------
// A table of segments: segment s is ids[offsets[s] : offsets[s + 1]], ascending (duplicates allowed); row r of a call
// excludes segment row_set[r] (-1: nothing).  Many rows can share one segment, e.g. every window of one user.  Two
// defaults describe the dense [n_rows, E] form: offsets NULL (segment s is ids[s * stride, (s + 1) * stride)) and
// row_set NULL (row r -> segment r).  ids NULL: no exclusion.
struct ItemSets {
  const long long* ids;
  const long long* offsets;
  const long long* row_set;
  long long total, n_sets;
  int stride;
};

// Segments of up to kSetStage ids are staged in shared memory as int32 (16 KB: the select kernels are register bound
// at 256 threads, so the stage never costs a CTA per SM), longer ones are searched in global memory.
constexpr int kSetStage = 4096;

// [lo, hi) of row r's segment; empty for -1 and, defensively, for anything out of range (the call's check kernel
// reports those, and no read here leaves the table)
__device__ __forceinline__ void set_segment(const ItemSets& s, long long r, long long& lo, long long& hi) {
  lo = hi = 0;
  if (!s.ids) return;
  const long long seg = s.row_set ? s.row_set[r] : r;
  if (seg < 0 || seg >= s.n_sets) return;
  long long a = s.offsets ? s.offsets[seg] : seg * s.stride, b = s.offsets ? s.offsets[seg + 1] : a + s.stride;
  a = a < 0 ? 0 : (a > s.total ? s.total : a);
  b = b < a ? a : (b > s.total ? s.total : b);
  lo = a; hi = b;
}

// a staged id: monotone in the int64 id (sorted stays sorted), and no candidate id (0 <= id < kNoId) is lost
__device__ __forceinline__ int set_stage_id(long long x) { return x < 0 ? -1 : (x >= kNoId ? kNoId : (int)x); }

// The CTA's view of one row's segment.  set_stage is called by every thread, then __syncthreads before set_has.
struct SetView {
  const long long* g;   // the segment in global memory, when it is not staged
  long long n;
  bool staged;
};
__device__ __forceinline__ SetView set_stage(const ItemSets& s, long long r, int* s_ids, int cap) {
  long long lo, hi;
  set_segment(s, r, lo, hi);
  SetView v = {s.ids ? s.ids + lo : nullptr, hi - lo, hi - lo <= cap};
  if (v.staged)
    for (long long e = threadIdx.x; e < v.n; e += blockDim.x) s_ids[e] = set_stage_id(v.g[e]);
  return v;
}

// id in the segment: binary search (lower bound) in shared or global memory
__device__ __forceinline__ bool set_has(const SetView& v, const int* s_ids, int id) {
  long long lo = 0, hi = v.n;
  if (v.staged) {
    while (lo < hi) {
      const long long mid = (lo + hi) >> 1;
      if (s_ids[mid] < id) lo = mid + 1; else hi = mid;
    }
    return lo < v.n && s_ids[lo] == id;
  }
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(v.g + mid) < id) lo = mid + 1; else hi = mid;
  }
  return lo < v.n && __ldg(v.g + lo) == id;
}

// ---- Exact rank of a row's target: the number of eligible items that the row's top-k would put before it ----------
// A rank pass counts every id j != t of a column block whose (key, id) beats the target's, then subtracts the excluded
// ones: the distinct ids of the row's segment inside the block that beat it, t itself never (a target is not
// excluded).  A sorted segment is cut to the block by two binary searches, so exclusion costs one read per excluded id
// of the block, not a search per beating item.

// first index of segment ids[0, n) holding an id >= x
__device__ __forceinline__ long long seg_lower_bound(const long long* ids, long long n, long long x) {
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(ids + mid) < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Called by every thread of the CTA: this thread's share of the excluded ids of row r inside [id_lo, id_hi) that beat
// (kt, t); key_at(id) is the key of an id of the block.  A repeated id counts once; an id outside the block (only in a
// malformed table, which the call's check kernel reports) is skipped, so no read leaves the block.
template <class KeyAt>
__device__ int excluded_beaters(const ItemSets& s, long long r, long long id_lo, long long id_hi, float kt, int t,
                                KeyAt key_at, long long* s_range) {
  if (threadIdx.x == 0) {
    long long lo, hi;
    set_segment(s, r, lo, hi);
    s_range[0] = lo;
    s_range[1] = lo + seg_lower_bound(s.ids + lo, hi - lo, id_lo);
    s_range[2] = lo + seg_lower_bound(s.ids + lo, hi - lo, id_hi);
  }
  __syncthreads();
  const long long first = s_range[0], a = s_range[1], b = s_range[2];
  int c = 0;
  for (long long e = a + threadIdx.x; e < b; e += blockDim.x) {
    const long long x = __ldg(s.ids + e);
    if (x < id_lo || x >= id_hi || x == t || (e > first && __ldg(s.ids + e - 1) == x)) continue;
    if (better(key_at(x), (int)x, kt, t)) ++c;
  }
  __syncthreads();                                          // s_range is rewritten for the next row
  return c;
}

// One thread per row: *flag |= 1 for a target outside [0, items)
static __global__ void rank_target_check_kernel(const long long* __restrict__ target, long long n, long long items,
                                                int* flag) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r < n && (target[r] < 0 || target[r] >= items)) atomicOr(flag, 1);
}

static inline int rank_target_check(const long long* target, int64_t n, int64_t items, int* flag, cudaStream_t st) {
  rank_target_check_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(target, n, items, flag);
  RECNN_CHECK_LAUNCH("rank_target_check_kernel");
  return RECNN_OK;
}

// One warp per row of the call: *flag |= 4 for a row_set outside [-1, n_sets), offsets out of [0, total] or
// decreasing, or a descending pair in the row's segment; |= 1 for an id outside [0, items).  Only the segments the rows
// reference are read.
static __global__ void __launch_bounds__(128)
item_sets_check_kernel(ItemSets s, long long n_rows, long long items, int* flag) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n_rows) return;
  const long long seg = s.row_set ? s.row_set[r] : r;
  if (seg < -1 || seg >= s.n_sets) {
    if (lane == 0) atomicOr(flag, 4);
    return;
  }
  if (seg < 0) return;
  const long long a = s.offsets ? s.offsets[seg] : seg * s.stride, b = s.offsets ? s.offsets[seg + 1] : a + s.stride;
  if (a < 0 || b < a || b > s.total) {
    if (lane == 0) atomicOr(flag, 4);
    return;
  }
  int bits = 0;
  for (long long e = a + lane; e < b; e += 32) {
    const long long x = s.ids[e];
    if (x < 0 || x >= items) bits |= 1;
    if (e > a && s.ids[e - 1] > x) bits |= 4;
  }
  bits = __reduce_or_sync(0xffffffffu, bits);
  if (lane == 0 && bits) atomicOr(flag, bits);
}

// One CTA per row of a dense [n_rows, n_ex] list (n_ex <= blockDim.x, a power of two): the row sorted ascending into
// out, so that the dense form is searched like a table segment
static __global__ void __launch_bounds__(256)
exclude_sort_kernel(const long long* __restrict__ ex, int n_ex, long long* __restrict__ out) {
  __shared__ long long s[256];
  const long long r = blockIdx.x;
  const int t = threadIdx.x, n = blockDim.x;
  s[t] = t < n_ex ? ex[r * n_ex + t] : LLONG_MAX;
  __syncthreads();
  for (int size = 2; size <= n; size <<= 1) {            // bitonic sort of n keys, one per thread
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      const int p = t ^ stride;
      if (p > t) {
        const long long a = s[t], b = s[p];
        const bool up = (t & size) == 0;
        if ((a > b) == up) { s[t] = b; s[p] = a; }
      }
      __syncthreads();
    }
  }
  if (t < n_ex) out[r * n_ex + t] = s[t];
}

static inline int pow2_threads(int n) {
  int t = 32;
  while (t < n) t <<= 1;
  return t;
}

// the shared-memory stage of a select kernel: none without exclusion
static inline int set_stage_bytes(const ItemSets& s) { return s.ids ? kSetStage * (int)sizeof(int) : 0; }

// The host checks of a table passed to a *_sets entry point (its contents are checked on the device); row_set NULL
// maps row r to segment r and then needs n_sets == n_rows.
static inline int item_sets_args(const int64_t* ids, int64_t total, const int64_t* offsets, int64_t n_sets,
                                 const int64_t* row_set, int64_t n_rows, const int32_t* error_flag, ItemSets* out) {
  RECNN_REQUIRE(error_flag && offsets && (ids || total == 0), "null pointer");
  RECNN_REQUIRE(total >= 0 && n_sets >= 0, "n_set_ids >= 0, n_sets >= 0");
  RECNN_REQUIRE(row_set || n_sets == n_rows, "without row_set, row r excludes set r: n_sets == n_rows");
  out->ids = reinterpret_cast<const long long*>(ids);
  out->offsets = reinterpret_cast<const long long*>(offsets);
  out->row_set = reinterpret_cast<const long long*>(row_set);
  out->total = total;
  out->n_sets = n_sets;
  out->stride = 0;                                         // ids NULL (an empty table): every segment is empty
  return RECNN_OK;
}

static inline int item_sets_check(const ItemSets& s, int64_t n_rows, int64_t items, int* flag, cudaStream_t st) {
  item_sets_check_kernel<<<(unsigned)ceil_div(n_rows, 4), 128, 0, st>>>(s, n_rows, items, flag);
  RECNN_CHECK_LAUNCH("item_sets_check_kernel");
  return RECNN_OK;
}

}  // namespace recnn
