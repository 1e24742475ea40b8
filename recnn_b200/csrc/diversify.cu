// Diversified re-ranking of served candidate pools against the resident embedding table: greedy MMR (Carbonell &
// Goldstein, 1998) and greedy DPP MAP inference (Chen, Zhang & Zhou, NeurIPS 2018), k steps per pool row.
//
// A pool row is served by a group of warps.  Its candidates' item vectors are read from the table once, staged in
// shared memory (cp.async when every row is 16-byte aligned, scalar loads otherwise) together with each candidate's id,
// score, squared norm and greedy state (the running max similarity for MMR; d^2 and the Cholesky c-vector for the DPP).
// Every step then reads shared memory only: each live candidate is dotted with the item chosen last, its state is
// updated, and the group takes a deterministic argmax (larger objective, then smaller id, then smaller column).
//
// Pools larger than one CTA's shared memory are split over a thread-block cluster of C = 2, 4 or 8 CTAs, each owning
// m_loc = ceil(m / C) consecutive columns.  Each step's per-warp bests are exchanged through distributed shared memory
// and every CTA reduces all of them to the same winner; the chosen row and, for the DPP, its c-vector are then copied
// out of the owner CTA's shared memory.  No global workspace, and no candidate is read twice from L2 / HBM.  Small
// pools pack several rows per CTA, one warp group each.
//
// Dot products (and the squared norms, in the same fma order, so a repeated item has similarity exactly 1) are formed
// by an octet of 8 lanes: lane q accumulates the float4 chunks q, q + 8, ... sequentially, then a fixed xor tree adds
// the 8 partials.  That order depends on dim only; the c-vector dots likewise depend on the step only.  With the total
// order of the argmax, a row's outputs are the same bits whatever the cluster size, rows per CTA, batch or padding.
#include <cooperative_groups.h>
#include <float.h>
#include <math.h>
#include <string.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace recnn {

constexpr int kDivMaxPool = 256, kDivMaxK = 64, kDivMaxDim = 1024;
constexpr int kDivThreads = 256;                  // threads per CTA: up to 8 warps per pool row
constexpr int kDivMaxWarps = kDivThreads / 32;
constexpr int64_t kDivSmemCap = 112 * 1024;       // beyond this the pool is split over a cluster: 2 CTAs per SM
constexpr int64_t kDivSmemPacked = 48 * 1024;     // packing several rows into one CTA stops here
constexpr float kDppEps = 1e-4f;                  // the DPP stops when the chosen item's d^2 falls below this

struct DivBest {
  float obj, aux, n2;   // objective, greedy state (d^2 for the DPP), squared norm
  int col;              // pool column
  long long id;         // -1: no eligible candidate
};

struct DivPlan {
  int cluster, m_loc, warps, rows, d4, cpitch;
  int64_t smem;
};

// Per-CTA shared memory: rows * (m_loc candidates + the chosen buffers + the per-warp bests).
static int64_t div_smem(int rows, int m_loc, int d4, int cpitch, int k, int warps) {
  const int64_t slots = (int64_t)rows * m_loc;
  return round_up(slots * d4 * 4, 16) + round_up(slots * cpitch * 4, 16) + round_up((int64_t)rows * d4 * 4, 16) +
         round_up((int64_t)rows * k * 4, 16) + round_up(slots * 8, 16) + 3 * round_up(slots * 4, 16) +
         2 * (int64_t)rows * warps * (int64_t)sizeof(DivBest);
}

static DivPlan div_plan(int m, int dim, int k, bool dpp) {
  DivPlan p;
  p.d4 = (dim + 3) / 4 * 4;
  p.cpitch = dpp ? (k | 1) : 0;                   // odd: the 4 octets of a warp read c-vectors in different banks
  for (p.cluster = 1;; p.cluster *= 2) {
    p.m_loc = (m + p.cluster - 1) / p.cluster;
    p.warps = (p.m_loc + 3) / 4 < kDivMaxWarps ? (p.m_loc + 3) / 4 : kDivMaxWarps;
    p.rows = 1;
    p.smem = div_smem(1, p.m_loc, p.d4, p.cpitch, k, p.warps);
    if (p.smem <= kDivSmemCap || p.cluster == 8) break;
  }
  if (p.cluster == 1)
    while (p.rows * 2 * p.warps <= kDivMaxWarps &&
           div_smem(p.rows * 2, p.m_loc, p.d4, p.cpitch, k, p.warps) <= kDivSmemPacked) {
      p.rows *= 2;
      p.smem = div_smem(p.rows, p.m_loc, p.d4, p.cpitch, k, p.warps);
    }
  return p;
}

__device__ __forceinline__ bool div_better(const DivBest& a, const DivBest& b) {
  if (a.id < 0) return false;
  if (b.id < 0) return true;
  if (a.obj != b.obj) return a.obj > b.obj;
  if (a.id != b.id) return a.id < b.id;
  return a.col < b.col;
}

__device__ __forceinline__ DivBest div_shfl(const DivBest& b, int o) {
  DivBest r;
  r.obj = __shfl_xor_sync(0xffffffffu, b.obj, o);
  r.aux = __shfl_xor_sync(0xffffffffu, b.aux, o);
  r.n2 = __shfl_xor_sync(0xffffffffu, b.n2, o);
  r.col = __shfl_xor_sync(0xffffffffu, b.col, o);
  r.id = __shfl_xor_sync(0xffffffffu, b.id, o);
  return r;
}

__device__ __forceinline__ DivBest div_warp_best(DivBest b) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const DivBest c = div_shfl(b, o);
    if (div_better(c, b)) b = c;
  }
  return b;
}

// a . b over d4 floats by the octet of lane q (0..7); every lane of the octet returns the same bits.  All 32 lanes of
// the warp must call it; a lane with live == false contributes nothing to its octet.
__device__ __forceinline__ float octet_dot(const float* a, const float* b, int d4, int q, bool live) {
  float v = 0.f;
  if (live)
    for (int c = q * 4; c < d4; c += 32) {
      const float4 x = *reinterpret_cast<const float4*>(a + c), y = *reinterpret_cast<const float4*>(b + c);
      v = fmaf(x.x, y.x, v); v = fmaf(x.y, y.y, v); v = fmaf(x.z, y.z, v); v = fmaf(x.w, y.w, v);
    }
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

__device__ __forceinline__ float octet_cdot(const float* a, const float* b, int n, int q, bool live) {
  float v = 0.f;
  if (live)
    for (int u = q; u < n; u += 8) v = fmaf(a[u], b[u], v);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v;
}

// cosine similarity from a dot product and two squared norms, clipped to [-1, 1]; 0 with a zero vector.  The same
// quotient as slate.cu's cosine distance (sim = 1 - distance): for a == b it is exactly 1.
__device__ __forceinline__ float cosine_sim(float dot, float na, float nb) {
  if (na == 0.f || nb == 0.f) return 0.f;
  const float p = na * nb;
  const float c = (p >= FLT_MIN && p <= FLT_MAX) ? dot / sqrtf(p)
                                                 : (float)((double)dot / sqrt((double)na * (double)nb));
  return fminf(fmaxf(c, -1.f), 1.f);
}

// DPP: objective a2 * s + log d^2 (a2 = 2 alpha); MMR: wrel * s - wdiv * max sim, the penalty 0 before the first pick
template <bool DPP, bool VEC>
__global__ void __launch_bounds__(kDivThreads, 2)
diversify_kernel(const long long* __restrict__ ids, const float* __restrict__ scores, long long n_rows, int m, int k,
                 const float* __restrict__ table, long long n_items, int dim, int d4, int cpitch, int m_loc, int R,
                 int warps, float wrel, float wdiv, float a2, long long* __restrict__ ids_out,
                 long long* __restrict__ pos_out, float* __restrict__ gain_out, int* __restrict__ flag) {
  extern __shared__ __align__(16) unsigned char smem[];
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks(), crank = (int)cluster.block_rank();
  const int slots = R * m_loc;
  unsigned char* p = smem;
  auto carve = [&](int64_t bytes) { unsigned char* r = p; p += (bytes + 15) & ~(int64_t)15; return r; };
  float* s_x = reinterpret_cast<float*>(carve((int64_t)slots * d4 * 4));       // [slots, d4] staged rows
  float* s_c = reinterpret_cast<float*>(carve((int64_t)slots * cpitch * 4));   // [slots, cpitch] DPP c-vectors
  float* s_cx = reinterpret_cast<float*>(carve((int64_t)R * d4 * 4));          // [R, d4] the chosen row
  float* s_cc = reinterpret_cast<float*>(carve((int64_t)R * k * 4));           // [R, k] its c-vector
  long long* s_id = reinterpret_cast<long long*>(carve((int64_t)slots * 8));   // id, -1 once padding or selected
  float* s_s = reinterpret_cast<float*>(carve((int64_t)slots * 4));            // score
  float* s_n2 = reinterpret_cast<float*>(carve((int64_t)slots * 4));           // squared norm
  float* s_aux = reinterpret_cast<float*>(carve((int64_t)slots * 4));          // MMR: max sim; DPP: d^2
  DivBest* s_best = reinterpret_cast<DivBest*>(p);                             // [2, R, warps]

  const int tid = threadIdx.x, G = warps * 32;
  const int slot = tid / G, gt = tid - slot * G, wi = gt >> 5, lane = tid & 31, q = lane & 7, oct = lane >> 3;
  const long long row0 = (long long)(blockIdx.x / C) * R, row = row0 + slot;
  const int col0 = crank * m_loc;

  for (int e = tid; e < slots; e += blockDim.x) {
    const int r = e / m_loc, col = col0 + (e - r * m_loc);
    long long id = -1;
    float s = 0.f;
    if (row0 + r < n_rows && col < m) {
      id = ids[(row0 + r) * m + col];
      s = scores[(row0 + r) * m + col];
      if (id < -1 || id >= n_items) {
        atomicOr(flag, 1);
        id = -1;
      }
      if (id >= 0 && !isfinite(s)) atomicOr(flag, 2);
    }
    s_id[e] = id;
    s_s[e] = s;
  }
  __syncthreads();
  const int w4 = d4 >> 2;
  for (int e = tid; e < slots * w4; e += blockDim.x) {
    const int i = e / w4, c = (e - i * w4) * 4;
    const long long id = s_id[i];
    if (id < 0) continue;                                  // never read: a dead slot takes part in no dot product
    float* dst = s_x + (int64_t)i * d4 + c;
    const float* src = table + id * dim + c;
    if (VEC) {
      cp_async16(dst, src);
    } else {
      float4 v;
      v.x = c < dim ? __ldg(src) : 0.f;
      v.y = c + 1 < dim ? __ldg(src + 1) : 0.f;
      v.z = c + 2 < dim ? __ldg(src + 2) : 0.f;
      v.w = c + 3 < dim ? __ldg(src + 3) : 0.f;
      *reinterpret_cast<float4*>(dst) = v;
    }
  }
  if (VEC) asm volatile("cp.async.wait_all;\n" ::: "memory");
  __syncthreads();

  // squared norms and the initial greedy state
  const int passes = (m_loc + warps * 4 - 1) / (warps * 4);
  for (int ps = 0; ps < passes; ++ps) {
    const int i = (ps * warps + wi) * 4 + oct, e = slot * m_loc + i;
    const bool live = i < m_loc && s_id[e] >= 0;
    const float* x = s_x + (int64_t)e * d4;
    const float n2 = octet_dot(x, x, d4, q, live);
    if (live && q == 0) {
      s_n2[e] = n2;
      s_aux[e] = DPP ? 0.5f * (1.f + cosine_sim(n2, n2, n2)) : -INFINITY;   // S_ii: 1, or 1/2 for a zero vector
    }
  }
  __syncthreads();

  long long chosen = -1;       // the item picked at the previous step (-1: none yet)
  float cn2 = 0.f, cd = 0.f;   // its squared norm and, for the DPP, d = sqrt(d^2) at selection
  int filled = 0;
  bool done = row >= n_rows;
  for (int t = 0; t < k; ++t) {
    const int par = t & 1;
    if (!done) {
      DivBest best;
      best.id = -1;
      best.obj = best.aux = best.n2 = 0.f;
      best.col = 0;
      for (int ps = 0; ps < passes; ++ps) {
        const int i = (ps * warps + wi) * 4 + oct, e = slot * m_loc + i;
        long long id = i < m_loc ? s_id[e] : -1;
        const bool dies = id >= 0 && id == chosen;         // the chosen item, and every other slot of the same id
        if (dies) id = -1;
        const bool live = id >= 0, update = live && chosen >= 0;
        const float dot = octet_dot(s_x + (int64_t)e * d4, s_cx + (int64_t)slot * d4, d4, q, update);
        float aux = live ? s_aux[e] : 0.f;
        if (DPP) {
          const float cdot = octet_cdot(s_c + (int64_t)e * cpitch, s_cc + (int64_t)slot * k, t - 1, q, update);
          if (update) {
            const float ev = (0.5f * (1.f + cosine_sim(dot, s_n2[e], cn2)) - cdot) / cd;
            aux -= ev * ev;
            if (q == 0) s_c[(int64_t)e * cpitch + t - 1] = ev;
          }
        } else if (update) {
          aux = fmaxf(aux, cosine_sim(dot, s_n2[e], cn2));
        }
        __syncwarp();
        if (q == 0 && i < m_loc) {
          if (dies) s_id[e] = -1;
          if (update) s_aux[e] = aux;
        }
        if (live) {
          const float s = s_s[e];
          DivBest b;
          if (DPP) b.obj = a2 * s + (aux > 0.f ? logf(aux) : -INFINITY);
          else b.obj = aux == -INFINITY ? wrel * s : wrel * s - wdiv * aux;
          b.aux = aux;
          b.n2 = s_n2[e];
          b.col = col0 + i;
          b.id = id;
          if (div_better(b, best)) best = b;
        }
      }
      best = div_warp_best(best);
      if (lane == 0) s_best[(par * R + slot) * warps + wi] = best;
    }
    cluster.sync();                                        // every CTA's bests of this step are written
    if (!done) {
      DivBest win;
      win.id = -1;
      win.obj = win.aux = win.n2 = 0.f;
      win.col = 0;
      for (int e = lane; e < C * warps; e += 32) {
        const DivBest* src = cluster.map_shared_rank(s_best + (par * R + slot) * warps + e % warps, e / warps);
        const DivBest b = *src;
        if (div_better(b, win)) win = b;
      }
      win = div_warp_best(win);
      if (win.id < 0 || (DPP && win.aux < kDppEps)) {
        done = true;
      } else {
        if (crank == 0 && gt == 0) {
          ids_out[row * k + t] = win.id;
          pos_out[row * k + t] = win.col;
          gain_out[row * k + t] = win.obj;
        }
        ++filled;
        chosen = win.id;
        cn2 = win.n2;
        cd = sqrtf(win.aux);
        const int owner = win.col / m_loc, li = slot * m_loc + (win.col - owner * m_loc);
        const float* xr = cluster.map_shared_rank(s_x + (int64_t)li * d4, owner);
        for (int c = gt * 4; c < d4; c += G * 4)
          *reinterpret_cast<float4*>(s_cx + (int64_t)slot * d4 + c) = *reinterpret_cast<const float4*>(xr + c);
        if (DPP) {
          const float* cr = cluster.map_shared_rank(s_c + (int64_t)li * cpitch, owner);
          for (int u = gt; u < t; u += G) s_cc[slot * k + u] = cr[u];
        }
      }
    }
    // s_cx / s_cc complete; a cluster's CTAs agree on done, for they reduce the same bests
    if (__syncthreads_and(done)) break;
  }
  if (crank == 0 && row < n_rows)
    for (int t = filled + gt; t < k; t += G) {
      ids_out[row * k + t] = -1;
      pos_out[row * k + t] = -1;
      gain_out[row * k + t] = __int_as_float(0x7fffffff);
    }
  cluster.sync();                                          // no CTA leaves while another may read its shared memory
}

template <bool DPP, bool VEC>
static int launch_diversify(const DivPlan& pl, const int64_t* ids, const float* scores, int64_t n_rows, int m, int k,
                            const float* table, int64_t n_items, int dim, float wrel, float wdiv, float a2,
                            int64_t* ids_out, int64_t* pos_out, float* gain_out, int32_t* flag, cudaStream_t st) {
  auto kernel = diversify_kernel<DPP, VEC>;
  RECNN_CHECK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)pl.smem));
  const int64_t blocks = pl.cluster == 1 ? ceil_div(n_rows, pl.rows) : n_rows * pl.cluster;
  RECNN_REQUIRE(blocks < (1ll << 31), "n_rows");
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)blocks, 1, 1);
  cfg.blockDim = dim3((unsigned)(pl.rows * pl.warps * 32), 1, 1);
  cfg.dynamicSmemBytes = (size_t)pl.smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = (unsigned)pl.cluster;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  RECNN_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kernel, reinterpret_cast<const long long*>(ids), scores, (long long)n_rows,
                                      m, k, table, (long long)n_items, dim, pl.d4, pl.cpitch, pl.m_loc, pl.rows,
                                      pl.warps, wrel, wdiv, a2, reinterpret_cast<long long*>(ids_out),
                                      reinterpret_cast<long long*>(pos_out), gain_out, flag));
  RECNN_CHECK_LAUNCH("diversify_kernel");
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

extern "C" int recnn_slate_diversify(const int64_t* ids, const float* scores, int64_t n_rows, int32_t m, int32_t k,
                                     const float* table, int64_t n_items, int32_t dim, int32_t method, float weight,
                                     int64_t* ids_out, int64_t* pos_out, float* gain_out, int32_t* error_flag,
                                     void* stream) {
  RECNN_REQUIRE(table && error_flag, "null pointer");
  RECNN_REQUIRE(n_rows == 0 || (ids && scores && ids_out && pos_out && gain_out), "null pointer");
  RECNN_REQUIRE(n_rows >= 0 && n_items > 0, "sizes");
  RECNN_REQUIRE(m >= 1 && m <= kDivMaxPool, "1 <= m <= 256");
  RECNN_REQUIRE(dim >= 1 && dim <= kDivMaxDim, "1 <= dim <= 1024");
  RECNN_REQUIRE(k >= 1 && k <= kDivMaxK && k <= m, "1 <= k <= min(64, m)");
  RECNN_REQUIRE(method == RECNN_DIVERSIFY_MMR || method == RECNN_DIVERSIFY_DPP, "method");
  RECNN_REQUIRE(weight >= 0.f && weight <= 1.f, "0 <= weight <= 1");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  if (n_rows == 0) return RECNN_OK;
  // the DPP at weight 1 orders by score: it is MMR at weight 1 (objective and gain = the score, no stopping rule)
  const bool dpp = method == RECNN_DIVERSIFY_DPP && weight < 1.f;
  const double w = weight;
  const float wrel = dpp ? 0.f : weight, wdiv = dpp ? 0.f : (float)(1.0 - w), a2 = dpp ? (float)(w / (1.0 - w)) : 0.f;
  const DivPlan pl = div_plan(m, dim, k, dpp);
  const bool vec = dim % 4 == 0 && (reinterpret_cast<uintptr_t>(table) & 15) == 0;
  if (dpp)
    return vec ? launch_diversify<true, true>(pl, ids, scores, n_rows, m, k, table, n_items, dim, wrel, wdiv, a2,
                                              ids_out, pos_out, gain_out, error_flag, st)
               : launch_diversify<true, false>(pl, ids, scores, n_rows, m, k, table, n_items, dim, wrel, wdiv, a2,
                                               ids_out, pos_out, gain_out, error_flag, st);
  return vec ? launch_diversify<false, true>(pl, ids, scores, n_rows, m, k, table, n_items, dim, wrel, wdiv, a2,
                                             ids_out, pos_out, gain_out, error_flag, st)
             : launch_diversify<false, false>(pl, ids, scores, n_rows, m, k, table, n_items, dim, wrel, wdiv, a2,
                                              ids_out, pos_out, gain_out, error_flag, st);
}
