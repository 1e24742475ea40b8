// The slab producer of the retrieval metrics that are not inner products (RECNN_METRIC_L1 .. RECNN_METRIC_CORR, see
// recnn_b200.h for their arithmetic): out[q, j] = the distance of query q to item j, written where the GEMM of the
// L2 / IP / COS metrics writes its scores, so that the top-k, exclusion and rank kernels read it unchanged.
//
// One CTA computes a 128 x 128 tile of (query, item) pairs with 256 threads, each owning an 8 x 8 register micro-tile
// (rows ty*4 + {0..3} and 64 + ty*4 + {0..3}, columns likewise from tx), so that every pair is one thread summing d
// ascending.  d runs through shared memory in chunks of 16, stored d-major ([d][row]) and double buffered: the next
// chunk is loaded from global memory into registers while the current one is consumed, then stored to the other
// buffer, one barrier per chunk.  Staging goes through registers rather than cp.async because the rows may start at
// any 4-byte address and correlation centres each value as it is staged.  The inner loop reads four float4 per d
// (two of queries, two of items: broadcast within a warp's two ty rows, 256 contiguous bytes for its 16 tx), so it
// has no bank conflicts; padding d beyond dim is staged as 0, which leaves every metric's sum unchanged.
#pragma once

#include "common.cuh"

namespace recnn {

constexpr int kDistTile = 128;     // queries and items per CTA
constexpr int kDistChunk = 8;      // d per shared-memory stage
constexpr int kDistThreads = 256;

__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

// CORR: the mean of one row, x_0 for a constant row (whose centred values are then exactly 0).  The loads go out 16 at
// a time ahead of the ascending sum: one row per thread would otherwise wait on memory once per element.
__device__ __forceinline__ float corr_mean(const float* __restrict__ x, int dim) {
  const float x0 = __ldg(x);
  bool constant = true;
  float s = 0.f;
  for (int d0 = 0; d0 < dim; d0 += 16) {
    float v[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) v[i] = d0 + i < dim ? __ldg(x + d0 + i) : x0;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      if (d0 + i < dim) s += v[i];
      constant &= v[i] == x0;
    }
  }
  return constant ? x0 : s / (float)dim;
}

// CORR: the mean and centred norm of one row; a constant row has mean x_0 and norm 0
__device__ __forceinline__ void corr_stats(const float* __restrict__ x, int dim, float& mean, float& norm) {
  mean = corr_mean(x, dim);
  float n = 0.f;
  for (int d = 0; d < dim; ++d) {
    const float c = x[d] - mean;
    n = fmaf(c, c, n);
  }
  norm = sqrtf(n);
}

// one (query, item) pair of metric M: step() once per d, ascending, then finish()
template <int M>
struct PairDist {
  float a = 0.f, b = 0.f;
  __device__ __forceinline__ void step(float q, float t) {
    if (M == RECNN_METRIC_L1) {
      a += fabsf(q - t);
    } else if (M == RECNN_METRIC_LINF) {
      a = max_nan(a, fabsf(q - t));
    } else if (M == RECNN_METRIC_CANBERRA) {
      const float den = fabsf(q) + fabsf(t);
      a += den == 0.f ? 0.f : fabsf(q - t) / den;
    } else if (M == RECNN_METRIC_BRAYCURTIS) {
      a += fabsf(q - t);
      b += fabsf(q + t);
    } else {
      a = fmaf(q, t, a);                      // CORR: centred values
    }
  }
  // qn, tn: the centred norms (CORR only)
  __device__ __forceinline__ float finish(float qn, float tn) const {
    if (M == RECNN_METRIC_BRAYCURTIS) return a == 0.f ? 0.f : a / b;
    if (M == RECNN_METRIC_CORR) {
      const float den = qn * tn;
      float d = 1.f - (den == 0.f ? 0.f : a / den);
      d = d < 0.f ? 0.f : d;                  // comparisons, not fminf/fmaxf: a NaN stays NaN and ranks last
      return d > 2.f ? 2.f : d;
    }
    return a;
  }
};

// grid (ceil(n_items / 128), ceil(nq / 128)).  out[q, j] for q < nq, j < n_items (row pitch ldo, a multiple of 4, out
// 16-byte aligned; the pad columns of the last tile up to ldo may be written).  stats: recnn_item_norms for CORR.
template <int M>
__global__ void __launch_bounds__(kDistThreads, M == RECNN_METRIC_BRAYCURTIS ? 1 : 2)
distance_slab_kernel(const float* __restrict__ Q, int nq, const float* __restrict__ T, int n_items, int dim,
                     const float* __restrict__ stats, float* __restrict__ out, long long ldo) {
  __shared__ __align__(16) float sQ[2][kDistChunk][kDistTile];
  __shared__ __align__(16) float sT[2][kDistChunk][kDistTile];
  __shared__ float s_qmean[M == RECNN_METRIC_CORR ? kDistTile : 1], s_qnorm[M == RECNN_METRIC_CORR ? kDistTile : 1];
  __shared__ float s_tmean[M == RECNN_METRIC_CORR ? kDistTile : 1], s_tnorm[M == RECNN_METRIC_CORR ? kDistTile : 1];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int r0 = blockIdx.y * kDistTile;
  const long long j0 = (long long)blockIdx.x * kDistTile;
  // staging: thread stages row sr of both tiles, d sh * 4 .. sh * 4 + 3 of each chunk
  const int sr = tid & (kDistTile - 1), sh = tid >> 7;
  const bool q_ok = r0 + sr < nq, t_ok = j0 + sr < n_items;
  const float* qrow = Q + (long long)(q_ok ? r0 + sr : 0) * dim;
  const float* trow = T + (t_ok ? j0 + sr : 0) * dim;
  // CORR: the query means here; each query's centred norm is summed from the staged chunks by its staging thread
  float qmean = 0.f, tmean = 0.f, qn2 = 0.f;
  if (M == RECNN_METRIC_CORR) {
    if (sh == 0) {
      s_qmean[sr] = q_ok ? corr_mean(qrow, dim) : 0.f;
    } else {
      s_tmean[sr] = t_ok ? __ldg(stats + j0 + sr) : 0.f;
      s_tnorm[sr] = t_ok ? __ldg(stats + n_items + j0 + sr) : 0.f;
    }
    __syncthreads();
    qmean = s_qmean[sr];
    tmean = s_tmean[sr];
  }
  float rq[kDistChunk / 2], rt[kDistChunk / 2];
  auto load = [&](int d0) {
#pragma unroll
    for (int i = 0; i < kDistChunk / 2; ++i) {
      const int d = d0 + sh * (kDistChunk / 2) + i;
      rq[i] = q_ok && d < dim ? __ldg(qrow + d) - qmean : 0.f;
      rt[i] = t_ok && d < dim ? __ldg(trow + d) - tmean : 0.f;
    }
  };
  auto store = [&](int buf) {
#pragma unroll
    for (int i = 0; i < kDistChunk / 2; ++i) {
      sQ[buf][sh * (kDistChunk / 2) + i][sr] = rq[i];
      sT[buf][sh * (kDistChunk / 2) + i][sr] = rt[i];
    }
  };

  PairDist<M> acc[8][8];
  const int chunks = (dim + kDistChunk - 1) / kDistChunk;
  load(0);
  store(0);
  __syncthreads();
  for (int c = 0; c < chunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < chunks) load((c + 1) * kDistChunk);
    if (M == RECNN_METRIC_CORR && sh == 0) {
#pragma unroll
      for (int kk = 0; kk < kDistChunk; ++kk) qn2 = fmaf(sQ[buf][kk][sr], sQ[buf][kk][sr], qn2);   // d ascending
    }
#pragma unroll 2                          // fully unrolled, the next d's operands push L1 and LINF past 128 registers
    for (int kk = 0; kk < kDistChunk; ++kk) {
      const float4 q0 = *reinterpret_cast<const float4*>(&sQ[buf][kk][ty * 4]);
      const float4 q1 = *reinterpret_cast<const float4*>(&sQ[buf][kk][64 + ty * 4]);
      const float4 t0 = *reinterpret_cast<const float4*>(&sT[buf][kk][tx * 4]);
      const float4 t1 = *reinterpret_cast<const float4*>(&sT[buf][kk][64 + tx * 4]);
      const float qv[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
      const float tv[8] = {t0.x, t0.y, t0.z, t0.w, t1.x, t1.y, t1.z, t1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j].step(qv[i], tv[j]);
    }
    if (c + 1 < chunks) store(buf ^ 1);
    __syncthreads();
  }
  if (M == RECNN_METRIC_CORR) {
    if (sh == 0) s_qnorm[sr] = sqrtf(qn2);
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = (i < 4 ? 0 : 64) + ty * 4 + (i & 3);
    if (r0 + r >= nq) continue;
    const float qn = M == RECNN_METRIC_CORR ? s_qnorm[r] : 0.f;
    float* o = out + (long long)(r0 + r) * ldo + j0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int c = h * 64 + tx * 4;            // a multiple of 4: c < n_items - j0 keeps c + 3 inside the pitch
      if (j0 + c >= n_items) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j)
        v[j] = acc[i][h * 4 + j].finish(qn, M == RECNN_METRIC_CORR ? s_tnorm[c + j] : 0.f);
      *reinterpret_cast<float4*>(o + c) = make_float4(v[0], v[1], v[2], v[3]);
    }
  }
}

// per item: the mean, then (at out + n_items) the centred norm, one thread per row (CORR's recnn_item_norms)
__global__ void __launch_bounds__(256)
corr_stats_kernel(const float* __restrict__ table, long long n_items, int dim, float* __restrict__ out) {
  const long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n_items) return;
  float m, n;
  corr_stats(table + row * dim, dim, m, n);
  out[row] = m;
  out[n_items + row] = n;
}

// out [nq, ldo] <- the distances of queries Q [nq, dim] to every item of T [n_items, dim] under a metric >= L1
static inline int distance_slab(int metric, const float* Q, int64_t nq, const float* T, int64_t n_items, int dim,
                                const float* stats, float* out, int64_t ldo, cudaStream_t st) {
  const dim3 grid((unsigned)ceil_div(n_items, kDistTile), (unsigned)ceil_div(nq, kDistTile));
  auto kernel = metric == RECNN_METRIC_L1           ? distance_slab_kernel<RECNN_METRIC_L1>
                : metric == RECNN_METRIC_LINF       ? distance_slab_kernel<RECNN_METRIC_LINF>
                : metric == RECNN_METRIC_CANBERRA   ? distance_slab_kernel<RECNN_METRIC_CANBERRA>
                : metric == RECNN_METRIC_BRAYCURTIS ? distance_slab_kernel<RECNN_METRIC_BRAYCURTIS>
                                                    : distance_slab_kernel<RECNN_METRIC_CORR>;
  kernel<<<grid, kDistThreads, 0, st>>>(Q, (int)nq, T, (int)n_items, dim, stats, out, ldo);
  RECNN_CHECK_LAUNCH("distance_slab_kernel");
  return RECNN_OK;
}

}  // namespace recnn
