// Distances between the items of each served slate, read straight from the resident embedding table: the diversity
// view of the reference's demo (examples/streamlit_demo.py:355-445, recnn/utils/plot.py:9-35: scipy cdist "cosine" /
// "euclidean" over the recommended items' embeddings), reduced per row to a mean and a minimum.
//
// One CTA owns R rows (R * KP <= 64 slots, KP = k rounded up to 4).  The rows' item vectors are staged in shared memory
// one 128-dim slice at a time (cp.async when every row is 16-byte aligned; zeros for empty slots and the padding of a
// dim that is not a multiple of 4, which add exactly nothing to a sum of squares or a dot product).  Each thread owns a
// 4 x 4 register tile of pairs: slots {ti + T x} x {tj + T y}, T = KP / 4, ti <= tj, over the T (T + 1) / 2 tiles of a
// row.  The strided slots put the 16 lanes that read different tj on consecutive staged rows, which a 132-float pitch
// spreads over all 32 banks; the lanes that share ti read the same address (broadcast).  On a diagonal tile (ti == tj)
// only x < y is a pair, so every unordered pair is formed exactly once, by one thread, and the matrix gets the same bits
// on both sides.  Per-pair partials stay in registers across slices; per-slot squared norms (cosine) accumulate in the
// same fma order as the dot products, so a repeated id gives dot == |a|^2 bit for bit and a distance of exactly 0.
//
// Per row: each thread sums its valid pairs in fp64 in a fixed order, then one warp adds the tiles' partials in a fixed
// order (a strided loop and a fixed xor tree).  A row's outputs depend only on its own ids: no float atomics, no
// dependence on the other rows of the call.
#include <float.h>
#include <math.h>

#include "common.cuh"

namespace recnn {

constexpr int kSlateSlice = 128;               // dims staged per pass
constexpr int kSlatePitch = kSlateSlice + 4;   // floats between staged rows: row r + 1 starts 4 banks after row r
constexpr int kSlateSlots = 64;                // staged slots per CTA: R * KP <= 64
constexpr int kSlateThreads = 160;             // k = 64: 136 tiles

struct SlatePlan {
  int kp, t, tiles, rows, threads;
  int64_t smem;
};

static SlatePlan slate_plan(int k) {
  SlatePlan p;
  p.kp = (k + 3) / 4 * 4;
  p.t = p.kp / 4;
  p.tiles = p.t * (p.t + 1) / 2;
  p.rows = kSlateSlots / p.kp;
  const int work = p.rows * p.tiles;
  p.threads = work < 64 ? 64 : (int)round_up(work, 32);
  const int64_t slots = (int64_t)p.rows * p.kp, tiles = (int64_t)p.rows * p.tiles;
  p.smem = round_up(tiles * 8, 16) + round_up(slots * 8, 16) + slots * kSlatePitch * 4 + round_up(slots * 4, 16) +
           round_up(tiles * 4, 16);
  return p;
}

__device__ __forceinline__ float slate_nan() { return __int_as_float(0x7fffffff); }

// acc: the sum of squared differences (EUCLIDEAN) or the dot product (COSINE); na, nb the squared norms (COSINE)
template <int METRIC>
__device__ __forceinline__ float pair_distance(float acc, float na, float nb) {
  if (METRIC == RECNN_SLATE_EUCLIDEAN) return sqrtf(acc);
  if (na == 0.f || nb == 0.f) return 1.f;                 // a zero vector: 1 by convention (scipy gives NaN)
  // sqrt(fl(x * x)) == x in binary floating point, so for a == b the quotient is exactly 1; where the fp32 product
  // leaves the normal range it is formed in fp64, where it is exact
  const float p = na * nb;
  const float c = (p >= FLT_MIN && p <= FLT_MAX) ? acc / sqrtf(p)
                                                 : (float)((double)acc / sqrt((double)na * (double)nb));
  return fminf(fmaxf(1.f - c, 0.f), 2.f);                 // scipy's clip of the cosine distance to [0, 2]
}

template <int METRIC, bool VEC>
__global__ void __launch_bounds__(kSlateThreads, 4)
slate_distances_kernel(const long long* __restrict__ ids, long long n_rows, int k, const float* __restrict__ table,
                       long long n_items, int dim, int kp, int T, int tiles, int R, float* __restrict__ mean_out,
                       float* __restrict__ min_out, int* __restrict__ count_out, float* __restrict__ matrix_out,
                       int* __restrict__ flag) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int slots = R * kp, work = R * tiles;
  double* s_sum = reinterpret_cast<double*>(smem);                                      // [R * tiles]
  long long* s_src = reinterpret_cast<long long*>(smem + ((work * 8 + 15) & ~15));      // [slots] item id or -1
  float* s_x = reinterpret_cast<float*>(reinterpret_cast<unsigned char*>(s_src) + ((slots * 8 + 15) & ~15));
  float* s_n2 = s_x + slots * kSlatePitch;                                              // [slots]
  float* s_min = s_n2 + ((slots + 3) & ~3);                                             // [R * tiles]
  const int tid = threadIdx.x;
  const long long row0 = (long long)blockIdx.x * R;

  for (int q = tid; q < slots; q += blockDim.x) {
    const int r = q / kp, s = q - r * kp;
    long long id = -1;
    if (row0 + r < n_rows && s < k) {
      id = ids[(row0 + r) * k + s];
      if (id < -1 || id >= n_items) {
        atomicOr(flag, 1);
        id = -1;
      }
    }
    s_src[q] = id;
    s_n2[q] = 0.f;
  }

  // this thread's tile: row r of the CTA, slots {ti + T x} x {tj + T y}
  const bool active = tid < work;
  const int r = active ? tid / tiles : 0;
  int ti = 0, tl = active ? tid - r * tiles : 0;
  while (tl >= T - ti) { tl -= T - ti; ++ti; }
  const int tj = ti + tl;
  const float* xa = s_x + (r * kp + ti) * kSlatePitch;
  const float* xb = s_x + (r * kp + tj) * kSlatePitch;
  float acc[4][4];
#pragma unroll
  for (int x = 0; x < 4; ++x)
#pragma unroll
    for (int y = 0; y < 4; ++y) acc[x][y] = 0.f;

  for (int d0 = 0; d0 < dim; d0 += kSlateSlice) {
    const int w = dim - d0 < kSlateSlice ? dim - d0 : kSlateSlice, w4 = (w + 3) >> 2;
    __syncthreads();                                       // the previous slice is consumed (and s_src is written)
    for (int e = tid; e < slots * w4; e += blockDim.x) {
      const int q = e / w4, c = (e - q * w4) * 4;
      float* dst = s_x + q * kSlatePitch + c;
      const long long id = s_src[q];
      if (id < 0) {
        *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
      } else if (VEC) {
        cp_async16(dst, table + id * dim + d0 + c);
      } else {
        const float* src = table + id * dim + d0 + c;
        float4 v;
        v.x = __ldg(src);
        v.y = c + 1 < w ? __ldg(src + 1) : 0.f;
        v.z = c + 2 < w ? __ldg(src + 2) : 0.f;
        v.w = c + 3 < w ? __ldg(src + 3) : 0.f;
        *reinterpret_cast<float4*>(dst) = v;
      }
    }
    if (VEC) asm volatile("cp.async.wait_all;\n" ::: "memory");
    __syncthreads();
    if (METRIC == RECNN_SLATE_COSINE) {
      for (int q = tid; q < slots; q += blockDim.x) {
        float n = s_n2[q];
        const float* v = s_x + q * kSlatePitch;
        for (int c = 0; c < w4 * 4; c += 4) {
          const float4 a = *reinterpret_cast<const float4*>(v + c);
          n = fmaf(a.x, a.x, n); n = fmaf(a.y, a.y, n); n = fmaf(a.z, a.z, n); n = fmaf(a.w, a.w, n);
        }
        s_n2[q] = n;
      }
    }
    if (active) {
#pragma unroll 2
      for (int c = 0; c < w4 * 4; c += 4) {
        float4 a[4], b[4];
#pragma unroll
        for (int x = 0; x < 4; ++x) {
          a[x] = *reinterpret_cast<const float4*>(xa + x * T * kSlatePitch + c);
          b[x] = *reinterpret_cast<const float4*>(xb + x * T * kSlatePitch + c);
        }
#pragma unroll
        for (int x = 0; x < 4; ++x)
#pragma unroll
          for (int y = 0; y < 4; ++y) {
            float v = acc[x][y];
            if (METRIC == RECNN_SLATE_EUCLIDEAN) {
              float t;
              t = a[x].x - b[y].x; v = fmaf(t, t, v);
              t = a[x].y - b[y].y; v = fmaf(t, t, v);
              t = a[x].z - b[y].z; v = fmaf(t, t, v);
              t = a[x].w - b[y].w; v = fmaf(t, t, v);
            } else {
              v = fmaf(a[x].x, b[y].x, v); v = fmaf(a[x].y, b[y].y, v);
              v = fmaf(a[x].z, b[y].z, v); v = fmaf(a[x].w, b[y].w, v);
            }
            acc[x][y] = v;
          }
      }
    }
  }
  __syncthreads();                                         // s_n2 complete

  const bool mat = matrix_out != nullptr;
  if (active) {
    const long long row = row0 + r;
    float* M = mat ? matrix_out + row * k * k : nullptr;
    double sum = 0.0;
    float mn = INFINITY;
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
      for (int y = 0; y < 4; ++y) {
        if (ti == tj && x >= y) continue;                  // the diagonal tile holds each pair twice and i == i
        const int i = ti + T * x, j = tj + T * y;
        const bool ok = s_src[r * kp + i] >= 0 && s_src[r * kp + j] >= 0;
        const float d = pair_distance<METRIC>(acc[x][y], s_n2[r * kp + i], s_n2[r * kp + j]);
        if (ok) {
          sum += (double)d;
          mn = fminf(mn, d);
        }
        if (mat && row < n_rows && i < k && j < k) {
          const float v = ok ? d : slate_nan();
          M[(long long)i * k + j] = v;
          M[(long long)j * k + i] = v;
        }
      }
    s_sum[tid] = sum;
    s_min[tid] = mn;
  }
  if (mat) {
    for (int q = tid; q < slots; q += blockDim.x) {
      const int rr = q / kp, s = q - rr * kp;
      if (row0 + rr < n_rows && s < k) matrix_out[(row0 + rr) * k * k + (long long)s * k + s] = s_src[q] >= 0 ? 0.f : slate_nan();
    }
  }
  __syncthreads();

  const int lane = tid & 31;
  for (int rr = tid >> 5; rr < R; rr += blockDim.x >> 5) {
    double s = 0.0;
    float m = INFINITY;
    int c = 0;
    for (int t = lane; t < tiles; t += 32) {
      s += s_sum[rr * tiles + t];
      m = fminf(m, s_min[rr * tiles + t]);
    }
    for (int q = lane; q < kp; q += 32) c += s_src[rr * kp + q] >= 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      m = fminf(m, __shfl_xor_sync(0xffffffffu, m, o));
      c += __shfl_xor_sync(0xffffffffu, c, o);
    }
    const long long row = row0 + rr;
    if (lane == 0 && row < n_rows) {
      const bool two = c >= 2;
      mean_out[row] = two ? (float)(s / (double)((long long)c * (c - 1) / 2)) : slate_nan();
      min_out[row] = two ? m : slate_nan();
      count_out[row] = c;
    }
  }
}

}  // namespace recnn

using namespace recnn;

extern "C" int recnn_slate_distances(const int64_t* ids, int64_t n_rows, int32_t k, const float* table,
                                     int64_t n_items, int32_t dim, int32_t metric, float* mean_out, float* min_out,
                                     int32_t* count_out, float* matrix_out, int32_t* error_flag, void* stream) {
  RECNN_REQUIRE(table && error_flag, "null pointer");
  RECNN_REQUIRE(n_rows == 0 || (ids && mean_out && min_out && count_out), "null pointer");
  RECNN_REQUIRE(n_rows >= 0 && n_items > 0 && dim > 0, "sizes");
  RECNN_REQUIRE(k >= 1 && k <= 64, "1 <= k <= 64");
  RECNN_REQUIRE(metric == RECNN_SLATE_EUCLIDEAN || metric == RECNN_SLATE_COSINE, "metric");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  if (n_rows == 0) return RECNN_OK;
  const SlatePlan p = slate_plan(k);
  const int64_t blocks = ceil_div(n_rows, p.rows);
  RECNN_REQUIRE(blocks < (1ll << 31), "n_rows");
  const bool vec = dim % 4 == 0 && (reinterpret_cast<uintptr_t>(table) & 15) == 0;
  auto kernel = metric == RECNN_SLATE_EUCLIDEAN
                    ? (vec ? slate_distances_kernel<RECNN_SLATE_EUCLIDEAN, true>
                           : slate_distances_kernel<RECNN_SLATE_EUCLIDEAN, false>)
                    : (vec ? slate_distances_kernel<RECNN_SLATE_COSINE, true>
                           : slate_distances_kernel<RECNN_SLATE_COSINE, false>);
  kernel<<<(unsigned)blocks, p.threads, (size_t)p.smem, st>>>(
      reinterpret_cast<const long long*>(ids), n_rows, k, table, n_items, dim, p.kp, p.t, p.tiles, p.rows, mean_out,
      min_out, count_out, matrix_out, error_flag);
  RECNN_CHECK_LAUNCH("slate_distances_kernel");
  return RECNN_OK;
}
