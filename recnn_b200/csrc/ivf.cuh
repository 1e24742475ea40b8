// The pieces of the IVF index that IVF_FLAT (ivf.cu) and IVF_PQ (ivf_pq.cu) share: the coarse build (Lloyd k-means and
// the inverted lists), the probe inversion of a search and the bulk copy that streams list storage.  The host functions
// live in ivf.cu; one copy of each.  Both merge a query's probed lists with topk.cuh's warp_merge.
#pragma once

#include <stddef.h>

#include "common.cuh"
#include "tc_gemm.cuh"
#include "topk.cuh"

namespace recnn {

constexpr int kIvfTileQ = 32;          // queries of an IVF_FLAT fine-scan work unit: one per lane
constexpr int kIvfMaxDim = 512;        // the query tile and both row buffers fit shared memory up to here

// The buffers of one Lloyd k-means over n points into k centroids (carved by kmeans_carve).
struct IvfKmeans {
  float* cnorm;       // [k] |c|^2 for the L2 assignment
  float* count;       // [k] member counts (the split halves them)
  int64_t* assign;    // [n] nearest centroid of each point
  float* adist;       // [n]
  void* coarse;       // the assignment search's own workspace
  int64_t coarse_bytes;
  int *keys_in, *vals_in, *keys_out, *vals_out;   // [n] each
  long long* offs;    // [k + 1] training lists
  void* sort_tmp;
  size_t sort_bytes;
};

// the k-means buffers for n points and k centroids; the assignment search is sized for n_other points as well
IvfKmeans kmeans_carve(Carve& c, int64_t n, int64_t n_other, int k);

// Lloyd rounds over the points train [n, dim] (unit rows when spherical) from the centroids [k, dim] in place: every
// point to its nearest centroid in L2 (recnn_retrieve_topk, ties to the smaller id), each centroid the mean of its members
// summed in fp64 in ascending point order, faiss's deterministic split of empty lists, and (spherical) renormalisation.
// km must be carved for at least n points and k centroids.
int ivf_lloyd(const IvfKmeans& km, const float* train, int64_t n, int dim, float* centroids, int k, int n_iter,
              bool spherical, cudaStream_t st);

// warp per row: dst[r, :dim] = src[idx[r], :] (scaled to unit length when `unit`), dst[r, dim:ld_dst] = 0
int ivf_gather(const float* src, int dim, const long long* idx, long long n, bool unit, float* dst, int ld_dst,
               cudaStream_t st);

// The coarse half of an IVF build, shared by IVF_FLAT and IVF_PQ: k-means on the sample, then every item to its nearest
// centroid, written as centroids, centroid norms (L2 / COS), list_offsets and list_ids.  The workspace is carved by
// ivf_build_lists_bytes' layout; on return the final assignment of every item is left in assign_out [n_items]
// (a pointer into the workspace).
int64_t ivf_build_lists_bytes(int64_t n_items, int dim, int nlist, int64_t n_sample);
int ivf_build_lists(const float* table, int64_t n_items, int dim, int metric, const int64_t* sample_ids,
                    int64_t n_sample, const int64_t* init, int nlist, int n_iter, float* centroids_out,
                    float* centroid_norms_out, int64_t* list_offsets_out, int64_t* list_ids_out, void* workspace,
                    const int64_t** assign_out, cudaStream_t st);

// The search's probe step: each query's nprobe best lists (recnn_retrieve_topk over the centroids), regrouped per list
// into work units of `tile` queries.  group[list_start[l] + i] is the output slot (q * nprobe + j) of the i-th pair
// probing list l; list l's units are unit_start[l] .. unit_start[l + 1].
struct IvfProbes {
  int64_t* probe;     // [n, p] the coarse step's lists
  float* pdist;       // [n, p]
  void* coarse;
  int64_t coarse_bytes;
  int *cnt, *list_start, *unit_start;   // [nlist], [nlist + 1], [nlist + 1]
  int* group;         // [n * p] output slots grouped by list
};
IvfProbes ivf_probes_carve(Carve& c, int64_t n, int nlist, int nprobe);
int ivf_probe(const IvfProbes& w, const float* queries, int64_t n, int dim, const float* centroids,
              const float* centroid_norms, int nlist, int metric, int nprobe, int tile, cudaStream_t st);

// the list l and the first group entry g0 / query count nq of work unit u (device side of ivf_probe's units)
__device__ __forceinline__ int ivf_unit_list(const int* __restrict__ unit_start, int nlist, int u) {
  int lo = 0, hi = nlist;                              // the largest l with unit_start[l] <= u (< nlist)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (unit_start[mid] <= u) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ void bulk_copy(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(src)), "r"(bytes), "r"(bar)
               : "memory");
}

}  // namespace recnn
