// IVF_FLAT over the embedding table: the inverted-file index that MilvusConnection.search's {"nprobe": 16} addresses in
// the reference (recnn/data/db_con.py:45-56), built and searched on the device.
//
// Build (recnn_ivf_build): Lloyd k-means on a host-chosen sample (COS: unit rows, spherical), then every item goes to
// its nearest final centroid and the lists are laid out as a CSR with a list-ordered copy of the table.
//   assignment   recnn_retrieve_topk(points, centroids, L2, k = 1): the exact search itself, ties to the smaller id
//   grouping     a stable radix sort of (centroid, point) pairs: each list's members in ascending point order
//   update       one CTA per centroid sums its members in that order (fp64), so a build is bit-reproducible
//   empty lists  faiss's split, made deterministic: each empty list, in ascending id, takes the centroid of the list
//                with the largest count (ties: smaller id) with faiss's +-1/1024 perturbation; both counts halve
//
// Search (recnn_ivf_search), for n queries, nprobe p and k:
//   coarse       recnn_retrieve_topk(queries, centroids, metric, k = p): each query's p best lists
//   inversion    the [n, p] (query, list) pairs regrouped per list: a count, a scan into work units of 32 queries, a
//                scatter of each pair's output slot (q * p + j)
//   fine scan    one CTA per (list, tile of <= 32 queries probing it): the tile's queries staged in shared memory,
//                the list's contiguous rows streamed through two cp.async.bulk buffers; lane = query, each thread keeps
//                a register top-k list; fp32 fma dot products in ascending d; keys by metric_key (topk.cuh)
//   merge        one warp per query merges its p sorted lists (warp_merge, a lane owns lists lane and lane + 32) and
//                reports the distances through metric_distance, as the flat search does
// A (query, item) key is computed by the same instructions in the same order wherever it lands, so the result at
// nprobe p is the exact top-k, by (key, id), over the union of the p probed lists, whatever else shares the call.
#include <float.h>
#include <stddef.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>

#include "ivf.cuh"

namespace recnn {

constexpr int kIvfWarps = 4;           // warps of a fine-scan CTA: each takes 4 rows of a 16-row chunk
constexpr int kIvfChunk = 16;          // list rows per bulk copy
constexpr float kSplitEps = 1.0f / 1024.0f;

static inline int ivf_pitch(int dim) { return (int)round_up(dim, 4); }   // list-table row pitch: 16-byte rows

// ---------------------------------------------------------------------------------------------------- build kernels
// warp per row: dst[r, :dim] = src[idx[r], :] (scaled to unit length when `unit`), dst[r, dim:ld_dst] = 0; norms_out[r]
// (optional) = |row|^2 (L2) or 1/|row| (COS) by the instructions of item_norms_kernel, so the bits match
// recnn_item_norms of the table
__global__ void __launch_bounds__(256)
ivf_gather_kernel(const float* __restrict__ src, int dim, const long long* __restrict__ idx, long long n, bool unit,
                  float* __restrict__ dst, int ld_dst, int metric, float* __restrict__ norms_out) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* t = src + idx[r] * dim;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s = fmaf(t[d], t[d], s);
  s = warp_sum(s);
  const float scale = unit ? 1.0f / fmaxf(sqrtf(s), 1e-30f) : 1.0f;
  float* o = dst + r * ld_dst;
  for (int d = lane; d < ld_dst; d += 32) o[d] = d < dim ? (unit ? t[d] * scale : t[d]) : 0.f;
  if (norms_out && lane == 0) norms_out[r] = metric == RECNN_METRIC_COS ? 1.0f / fmaxf(sqrtf(s), 1e-30f) : s;
}

// the sort's input: key = the point's centroid, value = the point's index (ascending, so the sort keeps it so per list)
__global__ void ivf_keys_kernel(const int64_t* __restrict__ assign, long long n, int* __restrict__ keys,
                                int* __restrict__ vals) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = (int)assign[i];
  vals[i] = (int)i;
}

// offs[l] = the first position of the sorted keys holding a key >= l, l in [0, nlist]
__global__ void ivf_offsets_kernel(const int* __restrict__ keys, long long n, int nlist, long long* __restrict__ offs) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l > nlist) return;
  long long lo = 0, hi = n;
  while (lo < hi) {
    const long long mid = (lo + hi) >> 1;
    if (keys[mid] < l) lo = mid + 1; else hi = mid;
  }
  offs[l] = lo;
}

// one CTA per centroid: the mean of its members, summed in fp64 in ascending member order; an empty list keeps its
// centroid (the split rewrites it).  count[l] <- the member count.
__global__ void __launch_bounds__(128)
ivf_update_kernel(const float* __restrict__ points, int dim, const int* __restrict__ members,
                  const long long* __restrict__ offs, float* __restrict__ centroids, float* __restrict__ count) {
  const int l = blockIdx.x;
  const long long a = offs[l], b = offs[l + 1];
  if (threadIdx.x == 0) count[l] = (float)(b - a);
  if (a == b) return;
  for (int d = threadIdx.x; d < dim; d += blockDim.x) {
    double s = 0.0;
    for (long long m = a; m < b; ++m) s += (double)points[(long long)members[m] * dim + d];
    centroids[(long long)l * dim + d] = (float)(s / (double)(b - a));
  }
}

// one CTA: faiss's split of empty clusters (faiss/Clustering.cpp split_clusters) with the random donor replaced by the
// largest count (ties: the smaller id).  Empty lists are visited in ascending id; each takes the donor's centroid with
// even dims * (1 + eps) and odd dims * (1 - eps), the donor gets the opposite; the donor's count is split in halves
// between the two, as faiss does, before the next donor is chosen.
__global__ void __launch_bounds__(256)
ivf_split_kernel(float* __restrict__ centroids, int dim, float* __restrict__ count, int nlist) {
  __shared__ float s_key[32];
  __shared__ int s_id[32], s_owner[32];
  for (int i = 0; i < nlist; ++i) {
    if (count[i] != 0.f) continue;                     // uniform: every thread reads the same word
    // arg-max of the counts as an arg-min of -count, ties to the smaller id
    float best = FLT_MAX; int bid = kNoId;
    for (int j = threadIdx.x; j < nlist; j += blockDim.x)
      if (better(-count[j], j, best, bid)) { best = -count[j]; bid = j; }
    float wk; int donor, wo;
    block_argmin(best, bid, s_key, s_id, s_owner, wk, donor, wo);
    float* ci = centroids + (long long)i * dim;
    float* cj = centroids + (long long)donor * dim;
    for (int d = threadIdx.x; d < dim; d += blockDim.x) {
      const float v = cj[d];
      ci[d] = v * ((d & 1) ? 1.0f - kSplitEps : 1.0f + kSplitEps);
      cj[d] = v * ((d & 1) ? 1.0f + kSplitEps : 1.0f - kSplitEps);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      const float half = count[donor] * 0.5f;
      count[i] = half;
      count[donor] = count[donor] - half;
    }
    __syncthreads();
  }
}

// warp per centroid: scale to unit length (spherical k-means for COS)
__global__ void __launch_bounds__(256)
ivf_normalize_kernel(float* __restrict__ centroids, int nlist, int dim) {
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= nlist) return;
  float* c = centroids + (long long)r * dim;
  float s = 0.f;
  for (int d = lane; d < dim; d += 32) s = fmaf(c[d], c[d], s);
  s = warp_sum(s);
  const float inv = 1.0f / fmaxf(sqrtf(s), 1e-30f);
  for (int d = lane; d < dim; d += 32) c[d] *= inv;
}

__global__ void ivf_widen_kernel(const int* __restrict__ v, long long n, int64_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = v[i];
}

// --------------------------------------------------------------------------------------------------- search kernels
// the (query, list) pairs of the coarse step, counted per list
__global__ void ivf_count_kernel(const int64_t* __restrict__ probe, long long pairs, int* __restrict__ cnt) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < pairs) atomicAdd(cnt + probe[i], 1);
}

// one CTA, in order over chunks of 1024 lists: list_start = exclusive scan of the counts, unit_start = exclusive scan of
// the work units ceil(count / tile); the counts are zeroed for the scatter that follows (they become its fill cursors)
__global__ void __launch_bounds__(1024)
ivf_scan_kernel(int* __restrict__ cnt, int nlist, int tile, int* __restrict__ list_start, int* __restrict__ unit_start) {
  __shared__ int s_a[32], s_b[32];
  __shared__ int s_carry[2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) { s_carry[0] = 0; s_carry[1] = 0; }
  __syncthreads();
  for (int base = 0; base < nlist; base += 1024) {
    const int l = base + threadIdx.x;
    const int c = l < nlist ? cnt[l] : 0;
    const int u = (c + tile - 1) / tile;
    int a = c, b = u;                                  // inclusive warp scans
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int a2 = __shfl_up_sync(0xffffffffu, a, o), b2 = __shfl_up_sync(0xffffffffu, b, o);
      if (lane >= o) { a += a2; b += b2; }
    }
    if (lane == 31) { s_a[warp] = a; s_b[warp] = b; }
    __syncthreads();
    if (warp == 0) {
      int x = s_a[lane], y = s_b[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int x2 = __shfl_up_sync(0xffffffffu, x, o), y2 = __shfl_up_sync(0xffffffffu, y, o);
        if (lane >= o) { x += x2; y += y2; }
      }
      s_a[lane] = x; s_b[lane] = y;
    }
    __syncthreads();
    const int ca = s_carry[0], cb = s_carry[1];
    const int wa = warp ? s_a[warp - 1] : 0, wb = warp ? s_b[warp - 1] : 0;
    if (l < nlist) {
      list_start[l] = ca + wa + a - c;
      unit_start[l] = cb + wb + b - u;
      cnt[l] = 0;
    }
    __syncthreads();
    if (threadIdx.x == 0) { s_carry[0] = ca + s_a[31]; s_carry[1] = cb + s_b[31]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) { list_start[nlist] = s_carry[0]; unit_start[nlist] = s_carry[1]; }
}

// group[list_start[l] + i] = the output slot (q * p + j) of the i-th pair probing list l (order within a list is free:
// every key of a pair is computed the same wherever the pair lands)
__global__ void ivf_scatter_kernel(const int64_t* __restrict__ probe, long long pairs, const int* __restrict__ list_start,
                                   int* __restrict__ fill, int* __restrict__ group) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= pairs) return;
  const int l = (int)probe[i];
  group[list_start[l] + atomicAdd(fill + l, 1)] = (int)i;
}

struct IvfLists {
  const long long* offsets;   // [nlist + 1]
  const float* table;         // [n_items, pitch], list order
  const float* norms;         // [n_items], list order (NULL for IP)
  const long long* ids;       // [n_items], list order
};

// One CTA per work unit (list l, tile t of the queries probing l); blockIdx.x past the last unit exits.  Lane i of every
// warp holds query i of the tile; warp w scores rows 4w .. 4w + 3 of each 16-row chunk, so each query has four partial
// lists, merged through shared memory at the end.  Writes k candidates, ascending, to part[slot * k].
template <int KMAX, bool SETS>
__global__ void __launch_bounds__(kIvfWarps * 32)
ivf_scan_lists_kernel(const float* __restrict__ queries, int dim, int pitch, int nprobe, int nlist,
                      const int* __restrict__ list_start, const int* __restrict__ unit_start,
                      const int* __restrict__ group, IvfLists L, int metric, int k, ItemSets ex,
                      Cand* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int u = blockIdx.x;
  if (u >= unit_start[nlist]) return;
  const int l = ivf_unit_list(unit_start, nlist, u);
  const int g0 = list_start[l] + (u - unit_start[l]) * kIvfTileQ;
  const int nq = min(kIvfTileQ, list_start[l + 1] - g0);
  const long long r0 = L.offsets[l], n_rows = L.offsets[l + 1] - r0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ldq = pitch + 4;                           // 4-float skew: the lanes' 16-byte reads hit distinct banks

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  float* s_q = reinterpret_cast<float*>(smem + 128);
  float* s_rows = s_q + kIvfTileQ * ldq;               // [2][kIvfChunk][pitch], later the merge scratch
  const uint32_t bar0 = tc::smem_u32(bars), bar1 = tc::smem_u32(bars + 1);
  const long long chunks = (n_rows + kIvfChunk - 1) / kIvfChunk;
  auto issue = [&](long long c) {
    const uint32_t bar = (c & 1) ? bar1 : bar0;
    const long long rows = min((long long)kIvfChunk, n_rows - c * kIvfChunk);
    const uint32_t bytes = (uint32_t)(rows * pitch * 4);
    tc::mbar_expect_tx(bar, bytes);
    bulk_copy(tc::smem_u32(s_rows + (c & 1) * kIvfChunk * pitch), L.table + (r0 + c * kIvfChunk) * pitch, bytes, bar);
  };
  if (threadIdx.x == 0) {
    tc::mbar_init(bar0, 1);
    tc::mbar_init(bar1, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (chunks > 0) issue(0);
    if (chunks > 1) issue(1);
  }
  // the tile's queries, zero-padded to the pitch (and zero rows past nq)
  for (int i = 0; i < kIvfTileQ; ++i) {
    const long long q = i < nq ? group[g0 + i] / nprobe : -1;
    for (int d = threadIdx.x; d < pitch; d += blockDim.x)
      s_q[i * ldq + d] = q >= 0 && d < dim ? queries[q * dim + d] : 0.f;
  }
  const bool live = lane < nq;
  const int slot = live ? group[g0 + lane] : 0;
  SetView set = {nullptr, 0, false};
  if (SETS && live) {
    long long a, b;
    set_segment(ex, slot / nprobe, a, b);
    set.g = ex.ids + a;
    set.n = b - a;
  }
  __syncthreads();

  float keys[KMAX];
  int ids[KMAX];
  list_clear(keys, ids);
  const float* qrow = s_q + lane * ldq;
  for (long long c = 0; c < chunks; ++c) {
    tc::mbar_wait((c & 1) ? bar1 : bar0, (uint32_t)((c >> 1) & 1));
    const int rows = (int)min((long long)kIvfChunk, n_rows - c * kIvfChunk);
    const int rw = warp * 4;                           // this warp's rows of the chunk
    if (rw < rows) {
      const float* rbase = s_rows + ((c & 1) * kIvfChunk + rw) * pitch;
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      for (int d = 0; d < pitch; d += 4) {
        const float4 qv = *reinterpret_cast<const float4*>(qrow + d);
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const float4 rv = *reinterpret_cast<const float4*>(rbase + r * pitch + d);
          acc[r] = fmaf(qv.x, rv.x, acc[r]);
          acc[r] = fmaf(qv.y, rv.y, acc[r]);
          acc[r] = fmaf(qv.z, rv.z, acc[r]);
          acc[r] = fmaf(qv.w, rv.w, acc[r]);
        }
      }
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        if (!live || rw + r >= rows) continue;
        const long long row = r0 + c * kIvfChunk + rw + r;
        const float key = metric_key(acc[r], L.norms, row, metric);
        const int id = (int)__ldg(L.ids + row);
        if (better(key, id, keys[KMAX - 1], ids[KMAX - 1]) && (!SETS || set.n == 0 || !set_has(set, nullptr, id)))
          list_insert(keys, ids, key, id);
      }
    }
    __syncthreads();                                   // every warp is done with this buffer
    if (threadIdx.x == 0 && c + 2 < chunks) issue(c + 2);
  }

  // merge the four partial lists of each query: warps 2, 3 -> 0, 1, then warp 1 -> 0
  Cand* s_m = reinterpret_cast<Cand*>(s_rows);         // [2][32][KMAX]
  for (int step = 2; step >= 1; step >>= 1) {
    if (warp >= step && warp < 2 * step) {
      Cand* mine = s_m + ((warp - step) * kIvfTileQ + lane) * KMAX;
#pragma unroll
      for (int i = 0; i < KMAX; ++i) if (i < k) { mine[i].key = keys[i]; mine[i].id = ids[i]; }
    }
    __syncthreads();
    if (warp < step) {
      const Cand* other = s_m + (warp * kIvfTileQ + lane) * KMAX;
      for (int i = 0; i < k; ++i) {
        const Cand o = other[i];
        if (!better(o.key, o.id, keys[KMAX - 1], ids[KMAX - 1])) break;
        list_insert(keys, ids, o.key, o.id);
      }
    }
    __syncthreads();
  }
  if (warp == 0 && live) {
    Cand* out = part + (long long)slot * k;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) if (i < k) { out[i].key = keys[i]; out[i].id = ids[i]; }
  }
}

// one warp per query: merge its nprobe <= 64 ascending lists of k (lane owns lists lane and lane + 32) and report the
// distances, as the flat search does (metric_distance)
__global__ void __launch_bounds__(128)
ivf_merge_kernel(const Cand* __restrict__ part, int nprobe, int k, long long n_queries, int metric,
                 const float* __restrict__ queries, int dim, int64_t* __restrict__ ids_out, float* __restrict__ dist_out) {
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_queries) return;
  const float qn = warp_sq_norm(queries + q * dim, dim);
  const Cand* mine = part + q * (long long)nprobe * k;
  warp_merge<2>(k, [&](int l, int pos) {
    return l < nprobe && pos < k ? mine[(long long)l * k + pos] : Cand{FLT_MAX, kNoId};
  }, [&](int r, float key, int id, int) {
    if (lane == 0) {
      ids_out[q * k + r] = id == kNoId ? -1 : (int64_t)id;
      dist_out[q * k + r] = metric_distance(key, id, qn, metric);
    }
  });
}

// ------------------------------------------------------------------------------------------------------- workspaces
static int sort_end_bit(int nlist) {
  int b = 1;
  while ((1ll << b) < nlist) ++b;
  return b;
}

static size_t sort_temp_bytes(int64_t n, int nlist) {
  size_t bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, bytes, (const int*)nullptr, (int*)nullptr, (const int*)nullptr,
                                  (int*)nullptr, (int)n, 0, sort_end_bit(nlist));
  return bytes;
}

struct IvfBuildWorkspace {
  float* train;       // [n_sample, dim] the sample (COS: unit rows)
  IvfKmeans km;       // for n_items points: the training rounds and the final assignment
  int64_t bytes;
};

// the k-means buffers for n points and k centroids; the assignment search is sized for n_other points as well
IvfKmeans kmeans_carve(Carve& c, int64_t n, int64_t n_other, int k) {
  IvfKmeans w;
  w.cnorm = c.take(k);
  w.count = c.take(k);
  w.assign = c.take<int64_t>(n);
  w.adist = c.take(n);
  const int64_t a = recnn_retrieve_workspace_bytes(n_other, k, 1), b = recnn_retrieve_workspace_bytes(n, k, 1);
  w.coarse_bytes = a > b ? a : b;
  w.coarse = c.take<char>(w.coarse_bytes);
  w.keys_in = c.take<int>(n);
  w.vals_in = c.take<int>(n);
  w.keys_out = c.take<int>(n);
  w.vals_out = c.take<int>(n);
  w.offs = c.take<long long>(k + 1);
  w.sort_bytes = sort_temp_bytes(n, k);
  w.sort_tmp = c.take<char>((int64_t)w.sort_bytes);
  return w;
}

static IvfBuildWorkspace build_carve(int64_t n_items, int dim, int nlist, int64_t n_sample, void* base) {
  IvfBuildWorkspace w;
  Carve c(base);
  w.train = c.take(n_sample * dim);
  w.km = kmeans_carve(c, n_items, n_sample, nlist);
  w.bytes = c.bytes();
  return w;
}

int64_t ivf_build_lists_bytes(int64_t n_items, int dim, int nlist, int64_t n_sample) {
  return build_carve(n_items, dim, nlist, n_sample, nullptr).bytes;
}

IvfProbes ivf_probes_carve(Carve& c, int64_t n, int nlist, int p) {
  IvfProbes w;
  w.probe = c.take<int64_t>(n * p);
  w.pdist = c.take(n * p);
  w.coarse_bytes = recnn_retrieve_workspace_bytes(n, nlist, p);
  w.coarse = c.take<char>(w.coarse_bytes);
  w.cnt = c.take<int>(nlist);
  w.list_start = c.take<int>(nlist + 1);
  w.unit_start = c.take<int>(nlist + 1);
  w.group = c.take<int>(n * p);
  return w;
}

struct IvfSearchWorkspace {
  IvfProbes pr;
  Cand* part;         // [n * p, k]
  int64_t bytes;
};

static IvfSearchWorkspace search_carve(int64_t n, int nlist, int p, int k, void* base) {
  IvfSearchWorkspace w;
  Carve c(base);
  w.pr = ivf_probes_carve(c, n, nlist, p);
  w.part = c.take<Cand>(n * p * k);
  w.bytes = c.bytes();
  return w;
}

static int ivf_smem_bytes(int dim, int kmax) {
  const int pitch = ivf_pitch(dim);
  const int rows = 2 * kIvfChunk * pitch * 4, merge = 2 * kIvfTileQ * kmax * (int)sizeof(Cand);
  return 128 + kIvfTileQ * (pitch + 4) * 4 + (rows > merge ? rows : merge);
}

// sorted (centroid, point) pairs of `assign` -> vals_out grouped by list, ascending inside; offs [nlist + 1]
static int group_by_list(const IvfKmeans& w, int64_t n, int nlist, long long* offs, cudaStream_t st) {
  ivf_keys_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(w.assign, n, w.keys_in, w.vals_in);
  RECNN_CHECK_LAUNCH("ivf_keys_kernel");
  size_t bytes = w.sort_bytes;
  RECNN_CHECK_CUDA(cub::DeviceRadixSort::SortPairs(w.sort_tmp, bytes, w.keys_in, w.keys_out, w.vals_in, w.vals_out,
                                                   (int)n, 0, sort_end_bit(nlist), st));
  count_launch();
  ivf_offsets_kernel<<<(unsigned)ceil_div(nlist + 1, 256), 256, 0, st>>>(w.keys_out, n, nlist, offs);
  RECNN_CHECK_LAUNCH("ivf_offsets_kernel");
  return RECNN_OK;
}

int ivf_gather(const float* src, int dim, const long long* idx, long long n, bool unit, float* dst, int ld_dst,
               cudaStream_t st) {
  ivf_gather_kernel<<<(unsigned)ceil_div(n, 8), 256, 0, st>>>(src, dim, idx, n, unit, dst, ld_dst, RECNN_METRIC_L2,
                                                              nullptr);
  RECNN_CHECK_LAUNCH("ivf_gather_kernel");
  return RECNN_OK;
}

int ivf_lloyd(const IvfKmeans& w, const float* train, int64_t n, int dim, float* centroids, int k, int n_iter,
              bool spherical, cudaStream_t st) {
  for (int it = 0; it < n_iter; ++it) {
    RECNN_PROPAGATE(recnn_item_norms(centroids, k, dim, RECNN_METRIC_L2, w.cnorm, st));
    RECNN_PROPAGATE(recnn_retrieve_topk(train, n, dim, centroids, k, w.cnorm, RECNN_METRIC_L2, 1, w.assign, w.adist,
                                        w.coarse, w.coarse_bytes, st));
    RECNN_PROPAGATE(group_by_list(w, n, k, w.offs, st));
    ivf_update_kernel<<<(unsigned)k, 128, 0, st>>>(train, dim, w.vals_out, w.offs, centroids, w.count);
    RECNN_CHECK_LAUNCH("ivf_update_kernel");
    ivf_split_kernel<<<1, 256, 0, st>>>(centroids, dim, w.count, k);
    RECNN_CHECK_LAUNCH("ivf_split_kernel");
    if (spherical) {
      ivf_normalize_kernel<<<(unsigned)ceil_div(k, 8), 256, 0, st>>>(centroids, k, dim);
      RECNN_CHECK_LAUNCH("ivf_normalize_kernel");
    }
  }
  return RECNN_OK;
}

int ivf_build_lists(const float* table, int64_t n_items, int dim, int metric, const int64_t* sample_ids,
                    int64_t n_sample, const int64_t* init, int nlist, int n_iter, float* centroids_out,
                    float* centroid_norms_out, int64_t* list_offsets_out, int64_t* list_ids_out, void* workspace,
                    const int64_t** assign_out, cudaStream_t st) {
  const IvfBuildWorkspace w = build_carve(n_items, dim, nlist, n_sample, workspace);
  const bool cos = metric == RECNN_METRIC_COS;
  RECNN_PROPAGATE(ivf_gather(table, dim, reinterpret_cast<const long long*>(sample_ids), n_sample, cos, w.train, dim,
                             st));
  RECNN_PROPAGATE(ivf_gather(w.train, dim, reinterpret_cast<const long long*>(init), nlist, false, centroids_out, dim,
                             st));
  RECNN_PROPAGATE(ivf_lloyd(w.km, w.train, n_sample, dim, centroids_out, nlist, n_iter, cos, st));
  // final lists: every item to its nearest centroid (L2 on the raw rows; COS: the largest cosine, i.e. L2 on unit
  // rows).  The centroid norms of L2 and COS are the search's coarse norms too; IP's coarse step needs none.
  const int assign_metric = cos ? RECNN_METRIC_COS : RECNN_METRIC_L2;
  float* cnorm = metric == RECNN_METRIC_IP ? w.km.cnorm : centroid_norms_out;
  RECNN_PROPAGATE(recnn_item_norms(centroids_out, nlist, dim, assign_metric, cnorm, st));
  RECNN_PROPAGATE(recnn_retrieve_topk(table, n_items, dim, centroids_out, nlist, cnorm, assign_metric, 1, w.km.assign,
                                      w.km.adist, w.km.coarse, w.km.coarse_bytes, st));
  RECNN_PROPAGATE(group_by_list(w.km, n_items, nlist, reinterpret_cast<long long*>(list_offsets_out), st));
  ivf_widen_kernel<<<(unsigned)ceil_div(n_items, 256), 256, 0, st>>>(w.km.vals_out, n_items, list_ids_out);
  RECNN_CHECK_LAUNCH("ivf_widen_kernel");
  if (assign_out) *assign_out = w.km.assign;
  return RECNN_OK;
}

int ivf_probe(const IvfProbes& w, const float* queries, int64_t n, int dim, const float* centroids,
              const float* centroid_norms, int nlist, int metric, int nprobe, int tile, cudaStream_t st) {
  // 1. coarse: the nprobe best centroids of each query under the index's metric
  RECNN_PROPAGATE(recnn_retrieve_topk(queries, n, dim, centroids, nlist, centroid_norms, metric, nprobe, w.probe,
                                      w.pdist, w.coarse, w.coarse_bytes, st));
  // 2. probe inversion
  const long long pairs = n * nprobe;
  RECNN_CHECK_CUDA(cudaMemsetAsync(w.cnt, 0, sizeof(int) * nlist, st));
  ivf_count_kernel<<<(unsigned)ceil_div(pairs, 256), 256, 0, st>>>(w.probe, pairs, w.cnt);
  RECNN_CHECK_LAUNCH("ivf_count_kernel");
  ivf_scan_kernel<<<1, 1024, 0, st>>>(w.cnt, nlist, tile, w.list_start, w.unit_start);
  RECNN_CHECK_LAUNCH("ivf_scan_kernel");
  ivf_scatter_kernel<<<(unsigned)ceil_div(pairs, 256), 256, 0, st>>>(w.probe, pairs, w.list_start, w.cnt, w.group);
  RECNN_CHECK_LAUNCH("ivf_scatter_kernel");
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

extern "C" int64_t recnn_ivf_build_workspace_bytes(int64_t n_items, int32_t dim, int32_t nlist, int64_t n_sample) {
  if (n_items <= 0 || dim <= 0 || nlist <= 0 || n_sample < nlist || n_sample > n_items || n_items >= (1ll << 31))
    return 0;
  return build_carve(n_items, dim, nlist, n_sample, nullptr).bytes;
}

extern "C" int recnn_ivf_list_table(const float* table, int64_t n_items, int32_t dim, int32_t metric,
                                    const int64_t* list_ids, float* list_table_out, float* list_norms_out,
                                    void* stream) {
  RECNN_REQUIRE(table && list_ids && list_table_out && n_items > 0 && dim > 0, "null pointer / sizes");
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_IP || metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(metric == RECNN_METRIC_IP || list_norms_out, "L2 / COS need list_norms_out");
  ivf_gather_kernel<<<(unsigned)ceil_div(n_items, 8), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      table, dim, reinterpret_cast<const long long*>(list_ids), n_items, false, list_table_out, ivf_pitch(dim), metric,
      metric == RECNN_METRIC_IP ? nullptr : list_norms_out);
  RECNN_CHECK_LAUNCH("ivf_gather_kernel");
  return RECNN_OK;
}

static int ivf_build(const float* table, int64_t n_items, int32_t dim, int32_t metric,
                               const int64_t* sample_ids, int64_t n_sample, const int64_t* init, int32_t nlist,
                               int32_t n_iter, float* centroids_out, float* centroid_norms_out,
                               int64_t* list_offsets_out, int64_t* list_ids_out, float* list_table_out,
                               float* list_norms_out, void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(table && sample_ids && init && centroids_out && list_offsets_out && list_ids_out && list_table_out &&
                workspace, "null pointer");
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_IP || metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(metric == RECNN_METRIC_IP || (centroid_norms_out && list_norms_out), "L2 / COS need the norms outputs");
  RECNN_REQUIRE(n_items > 0 && n_items < (1ll << 31) && dim > 0, "0 < n_items < 2^31, dim > 0");
  RECNN_REQUIRE(nlist >= 1 && nlist <= n_sample && n_sample <= n_items, "1 <= nlist <= n_sample <= n_items");
  RECNN_REQUIRE(n_iter >= 0, "n_iter >= 0");
  const IvfBuildWorkspace w = build_carve(n_items, dim, nlist, n_sample, workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, workspace_bytes));
  RECNN_PROPAGATE(ivf_build_lists(table, n_items, dim, metric, sample_ids, n_sample, init, nlist, n_iter, centroids_out,
                                  centroid_norms_out, list_offsets_out, list_ids_out, workspace, nullptr,
                                  static_cast<cudaStream_t>(stream)));
  return recnn_ivf_list_table(table, n_items, dim, metric, list_ids_out, list_table_out, list_norms_out, stream);
}

extern "C" int64_t recnn_ivf_search_workspace_bytes(int64_t n_queries, int32_t nlist, int32_t nprobe, int32_t k) {
  if (n_queries <= 0 || nlist <= 0 || nprobe <= 0 || nprobe > nlist || k <= 0) return 0;
  return search_carve(n_queries, nlist, nprobe, k, nullptr).bytes;
}

static int ivf_search(const float* queries, int64_t n_queries, int32_t dim, const float* centroids,
                                const float* centroid_norms, int32_t nlist, const int64_t* list_offsets,
                                const float* list_table, const float* list_norms, const int64_t* list_ids,
                                int64_t n_items, int32_t metric, int32_t nprobe, int32_t k, const int64_t* set_ids,
                                int64_t n_set_ids, const int64_t* set_offsets, int64_t n_sets, const int64_t* row_set,
                                int64_t* ids_out, float* dist_out, int32_t* error_flag, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(queries && centroids && list_offsets && list_table && list_ids && ids_out && dist_out && workspace,
                "null pointer");
  RECNN_REQUIRE(metric == RECNN_METRIC_L2 || metric == RECNN_METRIC_IP || metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(metric == RECNN_METRIC_IP || (centroid_norms && list_norms), "L2 / COS need the norms");
  RECNN_REQUIRE(n_queries >= 0 && n_items > 0 && n_items < (1ll << 31), "sizes");
  RECNN_REQUIRE(dim > 0 && dim <= kIvfMaxDim, "1 <= dim <= 512");
  RECNN_REQUIRE(nlist >= 1 && nlist <= n_items, "1 <= nlist <= n_items");
  RECNN_REQUIRE(nprobe >= 1 && nprobe <= 64 && nprobe <= nlist, "1 <= nprobe <= min(nlist, 64)");
  RECNN_REQUIRE(k >= 1 && k <= 64 && k <= n_items, "1 <= k <= min(64, n_items)");
  RECNN_REQUIRE(n_queries * nprobe < (1ll << 31), "n_queries * nprobe must fit int32");
  RECNN_REQUIRE((reinterpret_cast<uintptr_t>(list_table) & 15) == 0, "list_table must be 16-byte aligned");
  ItemSets ex = {nullptr, nullptr, nullptr, 0, 0, 0};
  const bool sets = set_offsets != nullptr;
  if (n_queries == 0) return RECNN_OK;
  const IvfSearchWorkspace w = search_carve(n_queries, nlist, nprobe, k, workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, workspace_bytes));
  if (sets) RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_queries, error_flag, &ex));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (sets) {
    RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
    RECNN_PROPAGATE(item_sets_check(ex, n_queries, n_items, error_flag, st));
  }
  // 1, 2. coarse step and probe inversion
  RECNN_PROPAGATE(ivf_probe(w.pr, queries, n_queries, dim, centroids, centroid_norms, nlist, metric, nprobe, kIvfTileQ,
                            st));
  const long long pairs = n_queries * nprobe;
  // 3. fine scan: at most ceil(pairs / 32) + min(nlist, pairs) units; the surplus CTAs exit at once
  const int kmax = k <= 16 ? 16 : 64;
  auto kernel = k <= 16 ? (sets ? ivf_scan_lists_kernel<16, true> : ivf_scan_lists_kernel<16, false>)
                        : (sets ? ivf_scan_lists_kernel<64, true> : ivf_scan_lists_kernel<64, false>);
  const int smem = ivf_smem_bytes(dim, kmax);
  RECNN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long units = ceil_div(pairs, kIvfTileQ) + (pairs < nlist ? pairs : nlist);
  const IvfLists L = {reinterpret_cast<const long long*>(list_offsets), list_table, list_norms,
                      reinterpret_cast<const long long*>(list_ids)};
  kernel<<<(unsigned)units, kIvfWarps * 32, smem, st>>>(queries, dim, ivf_pitch(dim), nprobe, nlist, w.pr.list_start,
                                                        w.pr.unit_start, w.pr.group, L, metric, k, ex, w.part);
  RECNN_CHECK_LAUNCH("ivf_scan_lists_kernel");
  // 4. merge the nprobe lists of each query
  ivf_merge_kernel<<<(unsigned)ceil_div(n_queries, 4), 128, 0, st>>>(w.part, nprobe, k, n_queries, metric, queries, dim,
                                                                     ids_out, dist_out);
  RECNN_CHECK_LAUNCH("ivf_merge_kernel");
  return RECNN_OK;
}

// ---- the struct-argument entry points (recnn_ivf_index, recnn_ivf_build_args, recnn_ivf_search_args) --------------
extern "C" int64_t recnn_sizeof_ivf_index(void) { return (int64_t)sizeof(recnn_ivf_index); }
extern "C" int64_t recnn_sizeof_ivf_build_args(void) { return (int64_t)sizeof(recnn_ivf_build_args); }
extern "C" int64_t recnn_sizeof_ivf_search_args(void) { return (int64_t)sizeof(recnn_ivf_search_args); }

extern "C" int64_t recnn_offsetof_ivf_build_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_ivf_build_args, index);
    case 1: return offsetof(recnn_ivf_build_args, table);
    case 2: return offsetof(recnn_ivf_build_args, sample_ids);
    case 3: return offsetof(recnn_ivf_build_args, n_sample);
    case 4: return offsetof(recnn_ivf_build_args, init);
    case 5: return offsetof(recnn_ivf_build_args, n_iter);
    case 6: return offsetof(recnn_ivf_build_args, workspace);
    case 7: return offsetof(recnn_ivf_build_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int64_t recnn_offsetof_ivf_search_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_ivf_search_args, index);
    case 1: return offsetof(recnn_ivf_search_args, queries);
    case 2: return offsetof(recnn_ivf_search_args, n_queries);
    case 3: return offsetof(recnn_ivf_search_args, nprobe);
    case 4: return offsetof(recnn_ivf_search_args, k);
    case 5: return offsetof(recnn_ivf_search_args, set_ids);
    case 6: return offsetof(recnn_ivf_search_args, n_set_ids);
    case 7: return offsetof(recnn_ivf_search_args, set_offsets);
    case 8: return offsetof(recnn_ivf_search_args, n_sets);
    case 9: return offsetof(recnn_ivf_search_args, row_set);
    case 10: return offsetof(recnn_ivf_search_args, ids_out);
    case 11: return offsetof(recnn_ivf_search_args, dist_out);
    case 12: return offsetof(recnn_ivf_search_args, error_flag);
    case 13: return offsetof(recnn_ivf_search_args, workspace);
    case 14: return offsetof(recnn_ivf_search_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int recnn_ivf_build(const recnn_ivf_build_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_ivf_index& x = a->index;
  return ivf_build(a->table, x.n_items, x.dim, x.metric, a->sample_ids, a->n_sample, a->init, x.nlist, a->n_iter,
                   x.centroids, x.centroid_norms, x.list_offsets, x.list_ids, x.list_table, x.list_norms, a->workspace,
                   a->workspace_bytes, stream);
}

extern "C" int recnn_ivf_search(const recnn_ivf_search_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_ivf_index& x = a->index;
  return ivf_search(a->queries, a->n_queries, x.dim, x.centroids, x.centroid_norms, x.nlist, x.list_offsets,
                    x.list_table, x.list_norms, x.list_ids, x.n_items, x.metric, a->nprobe, a->k, a->set_ids,
                    a->n_set_ids, a->set_offsets, a->n_sets, a->row_set, a->ids_out, a->dist_out, a->error_flag,
                    a->workspace, a->workspace_bytes, stream);
}
