// IVF_PQ over the embedding table: the coarse lists of IVF_FLAT (ivf.cu, the same build code) with each item stored as
// m one-byte codes of its residual from its list's centroid, the index type Milvus and faiss offer next to IVF_FLAT.
//
// Build (recnn_ivf_pq_build):
//   lists        ivf_build_lists, the code recnn_ivf_build runs: the same centroids, offsets and ids, bit for bit
//   codebooks    per subspace j (dims [j * dsub, (j + 1) * dsub)), Lloyd k-means into 256 codewords on the residuals
//                of the first min(n_sample, 65536) sample points, through ivf_lloyd (the coarse build's rounds)
//   codes        recnn_ivf_pq_encode: residuals in slabs of 65,536 list positions, then a warp per (position,
//                subspace) takes the argmin over the 256 codewords
//
// Search (recnn_ivf_pq_search), for n queries, nprobe p, k and k' = max(1, refine) * k:
//   coarse, inversion   ivf_probe, in work units of TQ queries (8 / 4 / 2 for m <= 16 / 32 / 64)
//   ADC scan     one CTA per (list, tile of <= TQ queries): each query's lookup table [m][256] built in shared memory
//                from the query, the centroid and the codebooks; the list's codes streamed through two cp.async.bulk
//                buffers; 256 / TQ threads per query, each with a register top-k' list, merged in shared memory
//   merge        one warp per query merges its p lists of k'; with refine it re-scores the k' candidates exactly from
//                the table by the instructions of ivf.cu's fine scan and merge, and keeps k
// A (query, item) key depends on the query, the item's list and codes only, so a query's result does not depend on the
// other queries of the call.
#include <float.h>
#include <stddef.h>
#include <stdint.h>

#include "ivf.cuh"

namespace recnn {

constexpr int kPqCodewords = 256;
constexpr int kPqMaxM = 64;
constexpr int kPqThreads = 256;        // ADC scan CTA
constexpr int kPqChunk = 256;          // list items per bulk copy
constexpr int64_t kPqTrainMax = 65536; // codebook training points
constexpr int64_t kPqSlab = 65536;     // list positions per encode slab

static inline int pq_code_pitch(int m) { return (int)round_up(m, 16); }
// queries of an ADC work unit: their tables (TQ * m * 1 KB) fit in 128 KB
static inline int pq_tile(int m) { return m <= 16 ? 8 : (m <= 32 ? 4 : 2); }

// ---------------------------------------------------------------------------------------------------- build kernels
// warp per row r < n: out[j][r][t] = x[j * dsub + t] - c_l[j * dsub + t] (x scaled to unit length when `unit`, by
// ivf_gather_kernel's instructions).  Sample mode (assign != NULL): x = table[items[r]], l = assign[items[r]].  List mode:
// x = table[items[p0 + r]] and l the list holding position p0 + r of offsets.
__global__ void __launch_bounds__(256)
pq_residual_kernel(const float* __restrict__ table, int dim, int dsub, const long long* __restrict__ items,
                   const int64_t* __restrict__ assign, const long long* __restrict__ offsets, int nlist, long long p0,
                   long long n, bool unit, const float* __restrict__ centroids, float* __restrict__ out) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  long long item;
  int l;
  if (assign) {
    item = items[r];
    l = (int)assign[item];
  } else {
    const long long p = p0 + r;
    item = items[p];
    int lo = 0, hi = nlist;                            // the largest l with offsets[l] <= p: the list holding p
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (offsets[mid] <= p) lo = mid; else hi = mid;
    }
    l = lo;
  }
  const float* x = table + item * dim;
  const float* c = centroids + (long long)l * dim;
  float scale = 1.0f;
  if (unit) {
    float s = 0.f;
    for (int d = lane; d < dim; d += 32) s = fmaf(x[d], x[d], s);
    s = warp_sum(s);
    scale = 1.0f / fmaxf(sqrtf(s), 1e-30f);
  }
  for (int d = lane; d < dim; d += 32) {
    const int j = d / dsub;
    // __fmul_rn: the unit row is rounded before the centroid is subtracted, as ivf_gather_kernel rounds it
    out[((long long)j * n + r) * dsub + (d - j * dsub)] = (unit ? __fmul_rn(x[d], scale) : x[d]) - c[d];
  }
}

// grid (rows / 8, code pitch), warp per (row r, subspace j): codes[(p0 + r) * pitch + j] = the argmin over the 256
// codewords of sum_t (res_t - B_j[c]_t)^2 (fp32 fma, ascending t, ties to the smaller code); pad bytes j >= m get 0
__global__ void __launch_bounds__(256)
pq_encode_kernel(const float* __restrict__ res, long long n, int dsub, int m, const float* __restrict__ codebooks,
                 uint8_t* __restrict__ codes, int pitch, long long p0) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, j = blockIdx.y;
  if (r >= n) return;
  uint8_t* out = codes + (p0 + r) * pitch + j;
  if (j >= m) {
    if (lane == 0) *out = 0;
    return;
  }
  const float* x = res + ((long long)j * n + r) * dsub;
  const float* B = codebooks + (long long)j * kPqCodewords * dsub;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int t = 0; t < dsub; ++t) {
    const float v = x[t];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float d = v - __ldg(B + (lane + 32 * i) * dsub + t);
      acc[i] = fmaf(d, d, acc[i]);
    }
  }
  float key = acc[0];
  int id = lane;
#pragma unroll
  for (int i = 1; i < 8; ++i) if (acc[i] < key) { key = acc[i]; id = lane + 32 * i; }
  int owner = lane;
  warp_argmin(key, id, owner);
  if (lane == 0) *out = (uint8_t)id;
}

// --------------------------------------------------------------------------------------------------- search kernels
struct PqLists {
  const long long* offsets;   // [nlist + 1]
  const long long* ids;       // [n_items], list order
  const uint8_t* codes;       // [n_items, pitch], list order
  const float* centroids;     // [nlist, dim]
  const float* codebooks;     // [m, 256, dsub]
  int m, dsub, pitch;
};

static int pq_smem_layout(int dim, int m, int kmax, int* off_q, int* off_lut) {
  const int tq = pq_tile(m);
  const int codes = 2 * kPqChunk * pq_code_pitch(m);
  *off_q = 128 + codes + 32;                           // barriers, code buffers, the tile's <q, c_l> terms
  *off_lut = (int)round_up(*off_q + tq * dim * 4, 16);
  const int lut = tq * m * kPqCodewords * 4, merge = kPqThreads / 2 * kmax * (int)sizeof(Cand);
  return *off_lut + (lut > merge ? lut : merge);
}

// One CTA per work unit (list l, tile of <= TQ queries probing l); blockIdx.x past the last unit exits.  Threads
// [qi * S, (qi + 1) * S), S = 256 / TQ, serve query qi of the tile: thread s of them scores items s, s + S, ... of each
// chunk.  Their S lists are merged by halving through shared memory; writes k' candidates, ascending, to part[slot * k'].
template <int KMAX, bool SETS>
__global__ void __launch_bounds__(kPqThreads)
pq_scan_lists_kernel(const float* __restrict__ queries, int dim, int nprobe, int nlist, int tq,
                     const int* __restrict__ list_start, const int* __restrict__ unit_start,
                     const int* __restrict__ group, PqLists P, int metric, int kp, ItemSets ex, int off_q, int off_lut,
                     Cand* __restrict__ part) {
  extern __shared__ __align__(128) unsigned char smem[];
  const int u = blockIdx.x;
  if (u >= unit_start[nlist]) return;
  const int l = ivf_unit_list(unit_start, nlist, u);
  const int g0 = list_start[l] + (u - unit_start[l]) * tq;
  const int nq = min(tq, list_start[l + 1] - g0);
  const long long r0 = P.offsets[l], n_rows = P.offsets[l + 1] - r0;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int S = kPqThreads / tq, qi = threadIdx.x / S, slot_in = threadIdx.x % S;
  const int m = P.m, dsub = P.dsub, pitch = P.pitch;
  const bool l2 = metric == RECNN_METRIC_L2;

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem);
  uint8_t* s_codes = smem + 128;                       // [2][kPqChunk][pitch]
  float* s_c = reinterpret_cast<float*>(smem + off_q - 32);   // [tq] <q, c_l> (IP / COS)
  float* s_q = reinterpret_cast<float*>(smem + off_q);        // [tq][dim] L2: q - c_l; IP: q; COS: q / |q|
  float* s_lut = reinterpret_cast<float*>(smem + off_lut);    // [tq][m][256], later the merge scratch
  const uint32_t bar0 = tc::smem_u32(bars), bar1 = tc::smem_u32(bars + 1);
  const long long chunks = (n_rows + kPqChunk - 1) / kPqChunk;
  auto issue = [&](long long c) {
    const uint32_t bar = (c & 1) ? bar1 : bar0;
    const long long rows = min((long long)kPqChunk, n_rows - c * kPqChunk);
    const uint32_t bytes = (uint32_t)(rows * pitch);
    tc::mbar_expect_tx(bar, bytes);
    bulk_copy(tc::smem_u32(s_codes + (c & 1) * kPqChunk * pitch), P.codes + (r0 + c * kPqChunk) * pitch, bytes, bar);
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
  // warp w < tq stages query w of the tile (zeros past nq)
  const float* cl = P.centroids + (long long)l * dim;
  if (warp < tq) {
    const long long q = warp < nq ? group[g0 + warp] / nprobe : -1;
    const float* qrow = queries + (q < 0 ? 0 : q) * dim;
    float inv = 1.0f;
    if (metric == RECNN_METRIC_COS && q >= 0) inv = 1.0f / fmaxf(sqrtf(warp_sq_norm(qrow, dim)), 1e-30f);
    float* sq = s_q + warp * dim;
    for (int d = lane; d < dim; d += 32)
      sq[d] = q < 0 ? 0.f : (l2 ? qrow[d] - cl[d] : (metric == RECNN_METRIC_COS ? qrow[d] * inv : qrow[d]));
    __syncwarp();
    if (!l2 && lane == 0) {
      float s = 0.f;
      for (int d = 0; d < dim; ++d) s = fmaf(sq[d], cl[d], s);
      s_c[warp] = s;
    }
  }
  __syncthreads();
  // the tables: entry (j, c) of every query of the tile per thread, so each codeword is read once per CTA
  for (int e = threadIdx.x; e < m * kPqCodewords; e += kPqThreads) {
    const int j = e / kPqCodewords;
    const float* b = P.codebooks + (long long)e * dsub;
    const float* q0 = s_q + j * dsub;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int t = 0; t < dsub; ++t) {
      const float bv = __ldg(b + t);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (i < tq) {
          const float v = q0[i * dim + t];
          if (l2) { const float d = v - bv; acc[i] = fmaf(d, d, acc[i]); }
          else acc[i] = fmaf(v, bv, acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) if (i < tq) s_lut[i * m * kPqCodewords + e] = acc[i];
  }
  const bool live = qi < nq;
  const int slot = live ? group[g0 + qi] : 0;
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
  // the k'-th entry: the bar a candidate must beat (entries past k' are never read, so they need not be kept exact)
  float bar_k = FLT_MAX;
  int bar_i = kNoId;
  const float* T = s_lut + qi * m * kPqCodewords;
  const float base = (l2 || !live) ? 0.f : s_c[qi];
  for (long long c = 0; c < chunks; ++c) {
    tc::mbar_wait((c & 1) ? bar1 : bar0, (uint32_t)((c >> 1) & 1));
    const int rows = (int)min((long long)kPqChunk, n_rows - c * kPqChunk);
    if (live) {
      for (int i = slot_in; i < rows; i += S) {
        const uint8_t* crow = s_codes + ((c & 1) * kPqChunk + i) * pitch;
        float s = base;
        for (int j0 = 0; j0 < m; j0 += 16) {
          const uint4 w = *reinterpret_cast<const uint4*>(crow + j0);
          const uint32_t wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
          for (int b = 0; b < 16; ++b) {
            const int j = j0 + b;
            if (j < m) s += T[j * kPqCodewords + ((wv[b >> 2] >> (8 * (b & 3))) & 255u)];
          }
        }
        const float key = finite_key(l2 ? s : -s);
        const long long row = r0 + c * kPqChunk + i;
        const int id = (int)__ldg(P.ids + row);
        if (better(key, id, bar_k, bar_i) && (!SETS || set.n == 0 || !set_has(set, nullptr, id))) {
          list_insert(keys, ids, key, id);
          list_at(keys, ids, kp - 1, bar_k, bar_i);
        }
      }
    }
    __syncthreads();                                   // every thread is done with this buffer
    if (threadIdx.x == 0 && c + 2 < chunks) issue(c + 2);
  }

  // merge the S lists of each query by halving: threads [step, 2 step) of the query's range hand theirs to [0, step).
  // The scratch is entry-major ([KMAX][tq * S / 2]), so the 32 lanes of a warp touch consecutive slots, not one bank.
  constexpr int kLists = kPqThreads / 2;
  Cand* s_m = reinterpret_cast<Cand*>(s_lut);
  for (int step = S >> 1; step >= 1; step >>= 1) {
    if (slot_in >= step && slot_in < 2 * step) {
      Cand* mine = s_m + qi * (S >> 1) + slot_in - step;
#pragma unroll
      for (int i = 0; i < KMAX; ++i) if (i < kp) { mine[i * kLists].key = keys[i]; mine[i * kLists].id = ids[i]; }
    }
    __syncthreads();
    if (slot_in < step) {
      const Cand* other = s_m + qi * (S >> 1) + slot_in;
      for (int i = 0; i < kp; ++i) {
        const Cand o = other[i * kLists];
        if (!better(o.key, o.id, bar_k, bar_i)) break;
        list_insert(keys, ids, o.key, o.id);
        list_at(keys, ids, kp - 1, bar_k, bar_i);
      }
    }
    __syncthreads();
  }
  if (slot_in == 0 && live) {
    Cand* out = part + (long long)slot * kp;
#pragma unroll
    for (int i = 0; i < KMAX; ++i) if (i < kp) { out[i].key = keys[i]; out[i].id = ids[i]; }
  }
}

// the exact key of (query row q, item id) by the instructions of ivf_scan_lists_kernel: an fp32 fma dot product in
// ascending d, then metric_key with the item's norm
__device__ __forceinline__ float pq_exact_key(const float* __restrict__ q, const float* __restrict__ table, int dim,
                                              const float* __restrict__ norms, int metric, int id) {
  const float* x = table + (long long)id * dim;
  float s = 0.f;
  for (int d = 0; d < dim; ++d) s = fmaf(q[d], __ldg(x + d), s);
  return metric_key(s, norms, id, metric);
}

// one warp per query: merge its nprobe <= 64 ascending lists of k' into the k' best (warp_merge, two lists per lane).
// Without refine the first k are written with their ADC distances; with refine the k' are re-scored exactly and the
// best k reported as the flat search reports them (metric_distance).
__global__ void __launch_bounds__(128)
pq_merge_kernel(const Cand* __restrict__ part, int nprobe, int kp, int k, bool refine, long long n_queries, int metric,
                const float* __restrict__ queries, int dim, const float* __restrict__ table,
                const float* __restrict__ norms, int64_t* __restrict__ ids_out, float* __restrict__ dist_out) {
  __shared__ Cand s_best[4][64];
  const long long q = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (q >= n_queries) return;
  Cand* best = s_best[threadIdx.x >> 5];
  const Cand* mine = part + q * (long long)nprobe * kp;
  warp_merge<2>(kp, [&](int l, int pos) {
    return l < nprobe && pos < kp ? mine[(long long)l * kp + pos] : Cand{FLT_MAX, kNoId};
  }, [&](int r, float key, int id, int) {
    if (lane == 0) { best[r].key = key; best[r].id = id; }
  });
  __syncwarp();
  const float pad = metric == RECNN_METRIC_L2 ? FLT_MAX : -FLT_MAX;
  if (!refine) {
    for (int r = lane; r < k; r += 32) {
      const Cand c = best[r];
      ids_out[q * k + r] = c.id == kNoId ? -1 : (int64_t)c.id;
      dist_out[q * k + r] = c.id == kNoId ? pad : (metric == RECNN_METRIC_L2 ? c.key : -c.key);
    }
    return;
  }
  const float* qrow = queries + q * dim;
  const float qn = warp_sq_norm(qrow, dim);
  float k0 = FLT_MAX, k1 = FLT_MAX;
  int i0 = kNoId, i1 = kNoId;
  if (lane < kp && best[lane].id != kNoId) { i0 = best[lane].id; k0 = pq_exact_key(qrow, table, dim, norms, metric, i0); }
  if (lane + 32 < kp && best[lane + 32].id != kNoId) {
    i1 = best[lane + 32].id;
    k1 = pq_exact_key(qrow, table, dim, norms, metric, i1);
  }
  for (int r = 0; r < k; ++r) {
    const bool second = better(k1, i1, k0, i0);
    float key = second ? k1 : k0;
    int id = second ? i1 : i0, owner = lane;
    warp_argmin(key, id, owner);
    if (lane == owner) {
      if (second) { k1 = FLT_MAX; i1 = kNoId; } else { k0 = FLT_MAX; i0 = kNoId; }
    }
    if (lane == 0) {
      ids_out[q * k + r] = id == kNoId ? -1 : (int64_t)id;
      dist_out[q * k + r] = metric_distance(key, id, qn, metric);
    }
  }
}

// ------------------------------------------------------------------------------------------------------- workspaces
static int64_t pq_slab_rows(int64_t n_items) { return n_items < kPqSlab ? n_items : kPqSlab; }
static int64_t pq_train_rows(int64_t n_sample) { return n_sample < kPqTrainMax ? n_sample : kPqTrainMax; }

struct PqBuildWorkspace {
  void* lists;        // ivf_build_lists' workspace
  float* res;         // [m][n_train][dsub] training residuals
  IvfKmeans km;       // n_train points, 256 codewords
  float* slab;        // the encode slab
  int64_t bytes;
};

static PqBuildWorkspace pq_build_carve(int64_t n_items, int dim, int nlist, int64_t n_sample, void* base) {
  PqBuildWorkspace w;
  Carve c(base);
  const int64_t n_train = pq_train_rows(n_sample);
  w.lists = c.take<char>(ivf_build_lists_bytes(n_items, dim, nlist, n_sample));
  w.res = c.take(n_train * dim);
  w.km = kmeans_carve(c, n_train, n_train, kPqCodewords);
  w.slab = c.take(pq_slab_rows(n_items) * dim);
  w.bytes = c.bytes();
  return w;
}

static int64_t pq_encode_bytes(int64_t n_items, int dim, float** slab, void* base) {
  Carve c(base);
  *slab = c.take(pq_slab_rows(n_items) * dim);
  return c.bytes();
}

struct PqSearchWorkspace {
  IvfProbes pr;
  Cand* part;         // [n * p, k']
  int64_t bytes;
};

static PqSearchWorkspace pq_search_carve(int64_t n, int nlist, int p, int kp, void* base) {
  PqSearchWorkspace w;
  Carve c(base);
  w.pr = ivf_probes_carve(c, n, nlist, p);
  w.part = c.take<Cand>(n * p * kp);
  w.bytes = c.bytes();
  return w;
}

static int pq_index_args(const recnn_ivf_pq_index& x) {
  RECNN_REQUIRE(x.centroids && x.list_offsets && x.list_ids && x.codebooks && x.codes, "null pointer");
  RECNN_REQUIRE(x.metric == RECNN_METRIC_L2 || x.metric == RECNN_METRIC_IP || x.metric == RECNN_METRIC_COS, "metric");
  RECNN_REQUIRE(x.metric == RECNN_METRIC_IP || x.centroid_norms, "L2 / COS need centroid_norms");
  RECNN_REQUIRE(x.n_items >= kPqCodewords && x.n_items < (1ll << 31), "256 <= n_items < 2^31");
  RECNN_REQUIRE(x.dim > 0 && x.dim <= kIvfMaxDim, "1 <= dim <= 512");
  RECNN_REQUIRE(x.m >= 1 && x.m <= kPqMaxM && x.dim % x.m == 0, "1 <= m <= 64, m divides dim");
  RECNN_REQUIRE(x.nlist >= 1 && x.nlist <= x.n_items, "1 <= nlist <= n_items");
  RECNN_REQUIRE((reinterpret_cast<uintptr_t>(x.codes) & 15) == 0, "codes must be 16-byte aligned");
  return RECNN_OK;
}

// the codes of every list position, slab by slab
static int pq_encode(const recnn_ivf_pq_index& x, const float* table, float* slab, cudaStream_t st) {
  const int dsub = x.dim / x.m, pitch = pq_code_pitch(x.m);
  const int64_t rows_max = pq_slab_rows(x.n_items);
  const long long* ids = reinterpret_cast<const long long*>(x.list_ids);
  for (int64_t p0 = 0; p0 < x.n_items; p0 += rows_max) {
    const int64_t rows = x.n_items - p0 < rows_max ? x.n_items - p0 : rows_max;
    pq_residual_kernel<<<(unsigned)ceil_div(rows, 8), 256, 0, st>>>(
        table, x.dim, dsub, ids, nullptr, reinterpret_cast<const long long*>(x.list_offsets), x.nlist, p0, rows,
        x.metric == RECNN_METRIC_COS, x.centroids, slab);
    RECNN_CHECK_LAUNCH("pq_residual_kernel");
    pq_encode_kernel<<<dim3((unsigned)ceil_div(rows, 8), (unsigned)pitch), 256, 0, st>>>(slab, rows, dsub, x.m,
                                                                                      x.codebooks, x.codes, pitch, p0);
    RECNN_CHECK_LAUNCH("pq_encode_kernel");
  }
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

extern "C" int64_t recnn_ivf_pq_build_workspace_bytes(int64_t n_items, int32_t dim, int32_t nlist, int64_t n_sample,
                                                      int32_t m) {
  if (n_items < kPqCodewords || n_items >= (1ll << 31) || dim <= 0 || dim > kIvfMaxDim || nlist <= 0 ||
      n_sample < nlist || n_sample > n_items || pq_train_rows(n_sample) < kPqCodewords || m < 1 || m > kPqMaxM ||
      dim % m != 0)
    return 0;
  return pq_build_carve(n_items, dim, nlist, n_sample, nullptr).bytes;
}

extern "C" int64_t recnn_ivf_pq_encode_workspace_bytes(int64_t n_items, int32_t dim) {
  if (n_items <= 0 || dim <= 0) return 0;
  float* slab;
  return pq_encode_bytes(n_items, dim, &slab, nullptr);
}

extern "C" int64_t recnn_ivf_pq_search_workspace_bytes(int64_t n_queries, int32_t nlist, int32_t nprobe, int32_t k,
                                                       int32_t refine) {
  if (n_queries <= 0 || nlist <= 0 || nprobe <= 0 || nprobe > nlist || k <= 0 || refine < 0) return 0;
  return pq_search_carve(n_queries, nlist, nprobe, (refine > 1 ? refine : 1) * k, nullptr).bytes;
}

extern "C" int recnn_ivf_pq_build(const recnn_ivf_pq_build_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_ivf_pq_index& x = a->index;
  RECNN_PROPAGATE(pq_index_args(x));
  RECNN_REQUIRE(a->table && a->sample_ids && a->init && a->pq_init && a->workspace, "null pointer");
  RECNN_REQUIRE(x.nlist <= a->n_sample && a->n_sample <= x.n_items, "1 <= nlist <= n_sample <= n_items");
  RECNN_REQUIRE(pq_train_rows(a->n_sample) >= kPqCodewords, "min(n_sample, 65536) >= 256");
  RECNN_REQUIRE(a->n_iter >= 0, "n_iter >= 0");
  const PqBuildWorkspace w = pq_build_carve(x.n_items, x.dim, x.nlist, a->n_sample, a->workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, a->workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t* assign = nullptr;
  RECNN_PROPAGATE(ivf_build_lists(a->table, x.n_items, x.dim, x.metric, a->sample_ids, a->n_sample, a->init, x.nlist,
                                  a->n_iter, x.centroids, x.centroid_norms, x.list_offsets, x.list_ids, w.lists,
                                  &assign, st));
  const int64_t n_train = pq_train_rows(a->n_sample);
  const int dsub = x.dim / x.m;
  pq_residual_kernel<<<(unsigned)ceil_div(n_train, 8), 256, 0, st>>>(
      a->table, x.dim, dsub, reinterpret_cast<const long long*>(a->sample_ids), assign, nullptr, x.nlist, 0, n_train,
      x.metric == RECNN_METRIC_COS, x.centroids, w.res);
  RECNN_CHECK_LAUNCH("pq_residual_kernel");
  for (int j = 0; j < x.m; ++j) {
    float* book = x.codebooks + (int64_t)j * kPqCodewords * dsub;
    const float* train = w.res + j * n_train * dsub;
    RECNN_PROPAGATE(ivf_gather(train, dsub, reinterpret_cast<const long long*>(a->pq_init), kPqCodewords, false, book,
                               dsub, st));
    RECNN_PROPAGATE(ivf_lloyd(w.km, train, n_train, dsub, book, kPqCodewords, a->n_iter, false, st));
  }
  return pq_encode(x, a->table, w.slab, st);
}

extern "C" int recnn_ivf_pq_encode(const recnn_ivf_pq_encode_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  RECNN_PROPAGATE(pq_index_args(a->index));
  RECNN_REQUIRE(a->table && a->workspace, "null pointer");
  float* slab;
  RECNN_PROPAGATE(check_workspace(pq_encode_bytes(a->index.n_items, a->index.dim, &slab, a->workspace),
                                  a->workspace_bytes));
  return pq_encode(a->index, a->table, slab, static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_ivf_pq_search(const recnn_ivf_pq_search_args* a, void* stream) {
  RECNN_REQUIRE(a, "null pointer");
  const recnn_ivf_pq_index& x = a->index;
  RECNN_PROPAGATE(pq_index_args(x));
  RECNN_REQUIRE(a->queries && a->ids_out && a->dist_out && a->workspace, "null pointer");
  RECNN_REQUIRE(a->n_queries >= 0, "n_queries >= 0");
  RECNN_REQUIRE(a->nprobe >= 1 && a->nprobe <= 64 && a->nprobe <= x.nlist, "1 <= nprobe <= min(nlist, 64)");
  RECNN_REQUIRE(a->k >= 1 && a->k <= 64 && a->k <= x.n_items, "1 <= k <= min(64, n_items)");
  RECNN_REQUIRE(a->refine >= 0 && (int64_t)(a->refine > 1 ? a->refine : 1) * a->k <= 64, "refine >= 0, refine * k <= 64");
  RECNN_REQUIRE(a->refine == 0 || (a->table && (x.metric == RECNN_METRIC_IP || a->norms)), "refine needs the table "
                "(and its norms for L2 / COS)");
  RECNN_REQUIRE(a->n_queries * a->nprobe < (1ll << 31), "n_queries * nprobe must fit int32");
  ItemSets ex = {nullptr, nullptr, nullptr, 0, 0, 0};
  const bool sets = a->set_offsets != nullptr;
  if (a->n_queries == 0) return RECNN_OK;
  const int kp = (a->refine > 1 ? a->refine : 1) * a->k;
  const PqSearchWorkspace w = pq_search_carve(a->n_queries, x.nlist, a->nprobe, kp, a->workspace);
  RECNN_PROPAGATE(check_workspace(w.bytes, a->workspace_bytes));
  if (sets)
    RECNN_PROPAGATE(item_sets_args(a->set_ids, a->n_set_ids, a->set_offsets, a->n_sets, a->row_set, a->n_queries,
                                   a->error_flag, &ex));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (sets) {
    RECNN_CHECK_CUDA(cudaMemsetAsync(a->error_flag, 0, sizeof(int32_t), st));
    RECNN_PROPAGATE(item_sets_check(ex, a->n_queries, x.n_items, a->error_flag, st));
  }
  const int tq = pq_tile(x.m);
  RECNN_PROPAGATE(ivf_probe(w.pr, a->queries, a->n_queries, x.dim, x.centroids, x.centroid_norms, x.nlist, x.metric,
                            a->nprobe, tq, st));
  const long long pairs = a->n_queries * a->nprobe;
  const int kmax = kp <= 16 ? 16 : 64;
  auto kernel = kp <= 16 ? (sets ? pq_scan_lists_kernel<16, true> : pq_scan_lists_kernel<16, false>)
                         : (sets ? pq_scan_lists_kernel<64, true> : pq_scan_lists_kernel<64, false>);
  int off_q, off_lut;
  const int smem = pq_smem_layout(x.dim, x.m, kmax, &off_q, &off_lut);
  RECNN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  const long long units = ceil_div(pairs, tq) + (pairs < x.nlist ? pairs : x.nlist);
  const PqLists P = {reinterpret_cast<const long long*>(x.list_offsets), reinterpret_cast<const long long*>(x.list_ids),
                     x.codes, x.centroids, x.codebooks, x.m, x.dim / x.m, pq_code_pitch(x.m)};
  kernel<<<(unsigned)units, kPqThreads, smem, st>>>(a->queries, x.dim, a->nprobe, x.nlist, tq, w.pr.list_start,
                                                    w.pr.unit_start, w.pr.group, P, x.metric, kp, ex, off_q, off_lut,
                                                    w.part);
  RECNN_CHECK_LAUNCH("pq_scan_lists_kernel");
  pq_merge_kernel<<<(unsigned)ceil_div(a->n_queries, 4), 128, 0, st>>>(
      w.part, a->nprobe, kp, a->k, a->refine > 0, a->n_queries, x.metric, a->queries, x.dim, a->table, a->norms,
      a->ids_out, a->dist_out);
  RECNN_CHECK_LAUNCH("pq_merge_kernel");
  return RECNN_OK;
}

// ---- struct probes -------------------------------------------------------------------------------------------------
extern "C" int64_t recnn_sizeof_ivf_pq_index(void) { return (int64_t)sizeof(recnn_ivf_pq_index); }
extern "C" int64_t recnn_sizeof_ivf_pq_build_args(void) { return (int64_t)sizeof(recnn_ivf_pq_build_args); }
extern "C" int64_t recnn_sizeof_ivf_pq_encode_args(void) { return (int64_t)sizeof(recnn_ivf_pq_encode_args); }
extern "C" int64_t recnn_sizeof_ivf_pq_search_args(void) { return (int64_t)sizeof(recnn_ivf_pq_search_args); }

extern "C" int64_t recnn_offsetof_ivf_pq_build_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_ivf_pq_build_args, index);
    case 1: return offsetof(recnn_ivf_pq_build_args, table);
    case 2: return offsetof(recnn_ivf_pq_build_args, sample_ids);
    case 3: return offsetof(recnn_ivf_pq_build_args, n_sample);
    case 4: return offsetof(recnn_ivf_pq_build_args, init);
    case 5: return offsetof(recnn_ivf_pq_build_args, pq_init);
    case 6: return offsetof(recnn_ivf_pq_build_args, n_iter);
    case 7: return offsetof(recnn_ivf_pq_build_args, workspace);
    case 8: return offsetof(recnn_ivf_pq_build_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int64_t recnn_offsetof_ivf_pq_encode_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_ivf_pq_encode_args, index);
    case 1: return offsetof(recnn_ivf_pq_encode_args, table);
    case 2: return offsetof(recnn_ivf_pq_encode_args, workspace);
    case 3: return offsetof(recnn_ivf_pq_encode_args, workspace_bytes);
    default: return -1;
  }
}

extern "C" int64_t recnn_offsetof_ivf_pq_search_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_ivf_pq_search_args, index);
    case 1: return offsetof(recnn_ivf_pq_search_args, table);
    case 2: return offsetof(recnn_ivf_pq_search_args, norms);
    case 3: return offsetof(recnn_ivf_pq_search_args, queries);
    case 4: return offsetof(recnn_ivf_pq_search_args, n_queries);
    case 5: return offsetof(recnn_ivf_pq_search_args, nprobe);
    case 6: return offsetof(recnn_ivf_pq_search_args, k);
    case 7: return offsetof(recnn_ivf_pq_search_args, refine);
    case 8: return offsetof(recnn_ivf_pq_search_args, set_ids);
    case 9: return offsetof(recnn_ivf_pq_search_args, n_set_ids);
    case 10: return offsetof(recnn_ivf_pq_search_args, set_offsets);
    case 11: return offsetof(recnn_ivf_pq_search_args, n_sets);
    case 12: return offsetof(recnn_ivf_pq_search_args, row_set);
    case 13: return offsetof(recnn_ivf_pq_search_args, ids_out);
    case 14: return offsetof(recnn_ivf_pq_search_args, dist_out);
    case 15: return offsetof(recnn_ivf_pq_search_args, error_flag);
    case 16: return offsetof(recnn_ivf_pq_search_args, workspace);
    case 17: return offsetof(recnn_ivf_pq_search_args, workspace_bytes);
    default: return -1;
  }
}
