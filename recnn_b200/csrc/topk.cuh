// Exact top-k building blocks shared by nearest-item retrieval (retrieval.cu) and the REINFORCE policy's top-k
// (reinforce.cuh): a candidate is (key, id), smaller key first, ties towards the smaller id (== a stable argsort of the
// keys).  Each thread keeps the best KMAX of its share in a sorted register list; a CTA merges its lists by rounds of a
// block arg-min over the list heads.
#pragma once

#include <float.h>

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

}  // namespace recnn
