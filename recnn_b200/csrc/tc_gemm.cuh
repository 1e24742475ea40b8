// Hopper (sm_90a) tensor-core GEMM with fp32-grade accuracy: error-compensated 3xTF32
// on warpgroup MMAs (wgmma), operands staged by TMA, chunked accumulation in registers.
//
//   C[m,n] = sum_k A(m,k) * B(n,k)            (+ fused epilogue)
//
// Why 3xTF32: the parity bar is the reference's fp32 CPU result to 1e-5
// (BASELINE.json north_star); one TF32 pass has a 10-bit mantissa (~1e-3).  Each
// fp32 operand x is split into  hi = rna_tf32(x)  and  lo = rna_tf32(x - hi)  (the
// subtraction is exact).  Three MMAs per 8-wide k-slice,  lo_a*hi_b + hi_a*lo_b + hi_a*hi_b;
// the dropped lo*lo term is < 2^-22 relative.
//
// Why chunked accumulation: the tensor core's fp32 accumulate truncates, so an unchunked
// all-positive sum drifts by ~1e-8 per accumulate.  So
//   * the big hi*hi products of only CH k-blocks (K = 64, 8 accumulates) are summed in a chunk
//     accumulator D_hi; after each chunk it is added to a register-resident running sum with
//     round-to-nearest FADDs;
//   * the two small cross terms go to a separate accumulator D_lo that lives for the whole tile
//     (its magnitude is 2^-11 of the result, so its truncation error is irrelevant) and is
//     added once at the end.
// hi is rounded to nearest (not truncated), so |lo| <= 2^-12 |x| is symmetric and the dropped
// lo*lo term is unbiased.
//
// One 128 x BN output tile per CTA (BN = 64 or 128), two warpgroups (256 threads):
//   thread 0      issues the TMA loads: raw fp32 tiles of A and B -> smem stage s, STAGES k-blocks ahead  (full[s])
//   all threads   together split the raw stage into hi / lo tiles in the canonical K-major
//                 128B-swizzled wgmma layout (one of two split buffers; MN-major operands are transposed on the
//                 way), then each warpgroup issues the wgmmas of its 64 rows.  Splitting
//                 k-block i overlaps the wgmmas of k-block i-1.  Epilogue: the accumulators are staged through
//                 shared memory so that each thread applies bias/relu/dropout/... to one contiguous row segment.
// No separate producer warp: ptxas budgets registers of a wgmma kernel per whole warpgroup, and a third one would cap
// every thread at 168 registers, while the 128-wide tile keeps 3 x 64 accumulators (running sum, D_hi, D_lo) per thread.
// tf32 wgmma reads both operands K-major from shared memory; writing the split tiles is where the layout is fixed.
// Programmatic dependent launch: the producer calls griddepcontrol.launch_dependents once its last load is issued,
// every kernel parks at griddepcontrol.wait after its prologue (barrier init, tensor-map prefetch), and is launched
// with programmatic stream serialization, so the next GEMM's prologue overlaps this one's tail.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "gemm_simt.cuh"   // Epilogue struct + EpiKind

namespace recnn {
namespace tc {

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a pipeline bug must not hang the GPU, so after ~2 s of polling the kernel
// traps and the launch surfaces as a CUDA error instead.  No printf here: a function call inside the
// k-loop makes ptxas serialise every wgmma (warning C7510), which would undo the split / MMA overlap.
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 4000000000ll) __trap();
  }
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void cta_sync() { asm volatile("bar.sync 0;" ::: "memory"); }
// Programmatic dependent launch: launch_dependents lets the next kernel of the stream
// be scheduled onto idle SMs while this one finishes; its threads park at griddep_wait() -- after their prologue,
// before any global-memory access -- until this grid has completed and its writes are visible.  Both are no-ops for
// a launch without the programmatic-serialization attribute.
__device__ __forceinline__ void griddep_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ float lds32(uint32_t addr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, const float4& v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

// ------------------------------------------------------------------ warpgroup MMA
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving reads / writes of accumulator registers across an asynchronous wgmma.
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, both operands K-major tf32 in shared memory; accumulate = 0 overwrites D.
__device__ __forceinline__ void wgmma_tf32(float (&d)[32], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(accumulate));
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}

// Round-to-nearest (ties away) to TF32 = add half a TF32 ulp to the magnitude bits, clear the low 13.
// Bit-identical to cvt.rna.tf32.f32 for finite inputs, but two full-rate integer ops instead of a conversion.
__device__ __forceinline__ float tf32_rna(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
// x = hi + lo (+ <= 2^-24 |x|): hi = rna_tf32(x), lo = rna_tf32(x - hi).  Both are exact tf32 values, so the
// result does not depend on how the tensor core treats the low 13 bits of an operand word.
__device__ __forceinline__ void tf32_split(float x, float& hi, float& lo) {
  hi = tf32_rna(x);
  lo = tf32_rna(x - hi);
}
__device__ __forceinline__ void tf32_split4(const float4& x, float4& hi, float4& lo) {
  tf32_split(x.x, hi.x, lo.x);
  tf32_split(x.y, hi.y, lo.y);
  tf32_split(x.z, hi.z, lo.z);
  tf32_split(x.w, hi.w, lo.w);
}

// ------------------------------------------------------------------ descriptors
// wgmma shared-memory matrix descriptor, K-major operand in the 128-byte swizzle: rows of 128 bytes (BK = 32
// fp32), 8-row groups 1024 bytes apart (SBO), LBO unused for swizzled K-major layouts (1).  Advancing the start
// address by 32 bytes selects the next 8-wide k-slice inside the swizzle atom.
__device__ __forceinline__ uint64_t gmma_desc_k128(uint32_t saddr) {
  return uint64_t((saddr & 0x3FFFF) >> 4) | (uint64_t(1) << 16) | (uint64_t(1024 >> 4) << 32) | (uint64_t(1) << 62);
}

struct Problem {
  int M, N, K0, K1;      // K = K0 (+ K1 from a second A tensor: virtual concat along K, K-major A only)
  int k_chunk;           // k extent per split (multiple of BK), split index = blockIdx.z
  int b_k1_offset;       // B's k coordinate where the K1 segment starts (== K0 for a dense weight)
  int n_out_offset;      // column offset added when storing (C window)
  int b_n_offset;        // B's n coordinate of output column 0 (window into a wider B, e.g. W1[:, S:S+A])
  int n_skip;            // the first n_skip output columns are computed but not stored (operand lead pads)
};

template <int BN_, int STAGES_, bool A_MN_, bool B_MN_>
struct Cfg {
  // BK = 32: one 128-byte row per operand row and k-block, the width of the 128-byte swizzle.
  static constexpr int BM = 128, BN = BN_, BK = 32, STAGES = STAGES_;
  static constexpr int CH = 64 / BK;                               // k-blocks per accumulation chunk (K = 64)
  static constexpr bool A_MN = A_MN_, B_MN = B_MN_;
  static constexpr int A_BYTES = BM * BK * 4, B_BYTES = BN * BK * 4;
  static constexpr int RAW_BYTES = A_BYTES + B_BYTES;              // one TMA stage: raw A | raw B
  static constexpr int SPLIT_BYTES = 2 * A_BYTES + 2 * B_BYTES;    // one split buffer: A hi | A lo | B hi | B lo
  static constexpr int SMEM_BYTES = STAGES * RAW_BYTES + 2 * SPLIT_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  static constexpr int THREADS = 256;                              // two warpgroups
  static constexpr int NR = BN / 2;                                // accumulator registers per thread (64 x BN / 128)
  static constexpr int EPI_LD = BN + 4;                            // row pitch (floats) of the staged output tile
  static constexpr int COLS_PER_THREAD = BN / 2;                   // epilogue: one row segment per thread
  static_assert(BN == 64 || BN == 128, "BN");
  static_assert(BM * EPI_LD * 4 <= 2 * SPLIT_BYTES, "the staged output tile reuses the split buffers");
  static_assert(SMEM_BYTES <= 227 * 1024, "smem");
};

// ------------------------------------------------------------------ epilogue on a register-resident row
// acc[j] is C[m, nb + j] for j < NC (NC = 16 or a multiple of 32), handled in blocks of W = min(NC, 32)
// columns.  Stores 16 bytes at a time when the destination allows it.
template <int EPI, int NC>
__device__ __forceinline__ void epilogue_row(const Epilogue& e, const Problem& p, int m, int nb, int z,
                                             float (&acc)[NC]) {
  constexpr int W = NC < 32 ? NC : 32;
  static_assert(NC % W == 0 && (W == 16 || W == 32), "epilogue block width");
  const int N = p.N;
  if (m >= p.M) return;
  float* out_row;
  if (EPI == EPI_PARTIAL) out_row = e.out + ((long long)z * p.M + m) * e.ldo + p.n_out_offset;
  else out_row = e.out + (long long)m * e.ldo + p.n_out_offset;
#pragma unroll
  for (int j0 = 0; j0 < NC; j0 += W) {
    if (nb + j0 < N) {
      uint32_t keep_bits = 0xFFFFFFFFu;
      if (EPI == EPI_HIDDEN && e.train) {
        if (e.mask) {
          keep_bits = 0;
          const uint8_t* mrow = e.mask + (long long)m * N + nb + j0;
#pragma unroll
          for (int j = 0; j < W; ++j)
            if (nb + j0 + j < N && mrow[j]) keep_bits |= 1u << j;
        } else {
          // same stream as the CUDA-core path: bit (idx & 31) of word idx >> 5, idx = m*N + n
          const unsigned long long idx = (unsigned long long)m * N + nb + j0;
          if ((idx & 31) + W <= 32) {          // the block's W bits sit in one 32-bit word
            keep_bits = philox_keep_bits32(e.seed, (unsigned long long)*e.rng_step, e.stream_id, idx >> 5) >> (idx & 31);
          } else {
            keep_bits = 0;
#pragma unroll 1
            for (int j = 0; j < W; ++j) {
              const unsigned long long ij = idx + j;
              const uint32_t w = philox_keep_bits32(e.seed, (unsigned long long)*e.rng_step, e.stream_id, ij >> 5);
              keep_bits |= ((w >> (ij & 31)) & 1u) << j;
            }
          }
        }
      }
#pragma unroll
      for (int j4 = 0; j4 < W; j4 += 4) {
        const int n = nb + j0 + j4;
        if (n < N) {
          float v[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            float x = acc[j0 + j4 + u];
            const int nn = n + u;
            if (nn < N) {
              if (EPI == EPI_HIDDEN) {
                x = x + __ldg(e.bias + nn);
                if (e.add) x += e.add[(long long)m * e.ldadd + nn];
                x = fmaxf(x, 0.f);
                if (e.train) x = ((keep_bits >> (j4 + u)) & 1u) ? x * 2.0f : 0.f;
              } else if (EPI == EPI_LINEAR) {
                x = x + __ldg(e.bias + nn);
                if (e.apply_tanh) x = tanhf(x);
                if (e.add_noise) {
                  float z0;
                  if (e.noise) z0 = e.noise[(long long)m * N + nn];
                  else {
                    const unsigned long long idx = (unsigned long long)m * N + nn;
                    Philox ph(e.seed);
                    const uint4 r = ph(idx, ((unsigned long long)*e.rng_step << 8) | e.stream_id);
                    const float u1 = (r.x + 1.0f) * 2.3283064365386963e-10f;
                    const float u2 = r.y * 2.3283064365386963e-10f;
                    z0 = sqrtf(-2.0f * __logf(u1)) * __cosf(6.283185307179586f * u2) * e.noise_std;
                  }
                  x += fminf(fmaxf(z0, -e.noise_clip), e.noise_clip);
                }
              } else if (EPI == EPI_GATE) {
                x = e.h[(long long)m * e.ldh + nn] > 0.f ? x * e.gate_scale : 0.f;
              } else if (EPI == EPI_ACCUM) {
                x = out_row[nn] + x;
                if (e.h) x = e.h[(long long)m * e.ldh + nn] > 0.f ? x * e.gate_scale : 0.f;
              }
            }
            v[u] = x;
          }
          float* dst = out_row + n;
          if (n + 3 < N && n >= p.n_skip && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int u = 0; u < 4; ++u)
              if (n + u < N && n + u >= p.n_skip) dst[u] = v[u];
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------ operand split
// Raw tile of ROWS operand rows x BK k (as TMA wrote it) -> hi / lo tiles in the K-major 128B-swizzled layout:
// element (r, k) at byte r*128 + ((k/4) ^ (r%8))*16 + (k%4)*4.  A K-major raw tile was written by TMA in exactly
// that layout, so the split keeps every offset.  An MN-major raw tile is ROWS/32 boxes of [BK k-rows x 32 elements]
// in the same 128-byte swizzle (16-byte unit index ^= k % 8); it is transposed here, one thread per (row, 4 k),
// which reads one conflict-free 128-byte row per warp and k.
template <bool MN, int ROWS, int BK>
__device__ __forceinline__ void split_tile(uint32_t raw, uint32_t hi, uint32_t lo, int t) {
  constexpr int QUADS = ROWS * BK / 4;
  static_assert(QUADS % 256 == 0, "a tile must split evenly over the 256 threads");
#pragma unroll
  for (int j = 0; j < QUADS / 256; ++j) {
    const uint32_t q = (uint32_t)t + 256u * j;
    float4 x;
    uint32_t off;
    if (!MN) {
      off = 16u * q;
      x = lds128(raw + off);
    } else {
      const uint32_t r = q % ROWS, kq = q / ROWS;
      off = r * 128u + ((kq ^ (r & 7u)) << 4);
      const uint32_t cb = raw + (r >> 5) * (BK * 128u) + (r & 3u) * 4u, unit = (r & 31u) >> 2;
      float v[4];
#pragma unroll
      for (uint32_t u = 0; u < 4; ++u) {
        const uint32_t k = 4u * kq + u;
        v[u] = lds32(cb + k * 128u + ((unit ^ (k & 7u)) << 4));
      }
      x = make_float4(v[0], v[1], v[2], v[3]);
    }
    float4 xh, xl;
    tf32_split4(x, xh, xl);
    sts128(hi + off, xh);
    sts128(lo + off, xl);
  }
}

// ------------------------------------------------------------------ the kernel
template <class C, int EPI>
__global__ void __launch_bounds__(C::THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap map_a0, const __grid_constant__ CUtensorMap map_a1,
               const __grid_constant__ CUtensorMap map_b, Problem p, Epilogue epi) {
  constexpr int BM = C::BM, BN = C::BN, BK = C::BK, STAGES = C::STAGES, CH = C::CH, NR = C::NR;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem = (smem_u32(smem_raw) + 1023u) & ~1023u;       // shared-window address, 1 KB aligned
  auto raw_a = [&](int s) { return smem + (uint32_t)s * C::RAW_BYTES; };
  auto raw_b = [&](int s) { return smem + (uint32_t)s * C::RAW_BYTES + C::A_BYTES; };
  const uint32_t split0 = smem + (uint32_t)STAGES * C::RAW_BYTES;
  auto a_hi = [&](int b) { return split0 + (uint32_t)b * C::SPLIT_BYTES; };
  auto a_lo = [&](int b) { return a_hi(b) + C::A_BYTES; };
  auto b_hi = [&](int b) { return a_hi(b) + 2 * C::A_BYTES; };
  auto b_lo = [&](int b) { return a_hi(b) + 2 * C::A_BYTES + C::B_BYTES; };
  const uint32_t bars = split0 + 2u * C::SPLIT_BYTES;
  auto full = [&](int s) { return bars + 8u * s; };                   // TMA -> all threads

  const int ct = threadIdx.x;                            // 0..255
  const int wg = ct >> 7;                                // rows 64*wg .. 64*wg + 63 of the tile
  const int lane = ct & 31;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM, z = blockIdx.z;
  // k-blocks: segment 0 then segment 1, each padded up to a multiple of BK (TMA zero-fills the tail)
  const int nkb0 = (p.K0 + BK - 1) / BK, nkb1 = (p.K1 + BK - 1) / BK;
  const int kb_per_split = p.k_chunk / BK;
  const int kb_begin = z * kb_per_split;
  const int kb_end = min(nkb0 + nkb1, kb_begin + kb_per_split);
  const int num_kb = max(kb_end - kb_begin, 0);

  // Thread 0 issues the TMA loads of k-block i into raw stage i % STAGES.  A stage is refilled right after the
  // barrier that follows its split, so no "empty" barrier is needed.
  auto load = [&](int i) {
    const int st = i % STAGES;
    const int kb = kb_begin + i;
    const bool seg1 = kb >= nkb0;
    const int ka = seg1 ? (kb - nkb0) * BK : kb * BK;                     // k coordinate inside A's segment
    const int kbcol = seg1 ? p.b_k1_offset + (kb - nkb0) * BK : kb * BK;  // k coordinate in B
    const CUtensorMap* ma = seg1 ? &map_a1 : &map_a0;
    mbar_expect_tx(full(st), C::RAW_BYTES);
    if (!C::A_MN) {
      tma_load_2d(raw_a(st), ma, full(st), ka, m0);                         // box {BK, 128}
    } else {
#pragma unroll
      for (int c = 0; c < BM / 32; ++c)                                     // box {32, BK} per 32-wide M chunk
        tma_load_2d(raw_a(st) + c * (BK * 128), ma, full(st), m0 + 32 * c, ka);
    }
    if (!C::B_MN) {
      tma_load_2d(raw_b(st), &map_b, full(st), kbcol, p.b_n_offset + n0);   // box {BK, BN}
    } else {
#pragma unroll
      for (int c = 0; c < BN / 32; ++c)
        tma_load_2d(raw_b(st) + c * (BK * 128), &map_b, full(st), p.b_n_offset + n0 + 32 * c, kbcol);
    }
    // After the last load the next kernel of the stream may be scheduled.  Its CTAs run their prologue and park at
    // griddepcontrol.wait holding an SM each, so releasing them here rather than at kernel entry keeps them off SMs
    // that concurrent GEMMs of the step's other chains could use.
    if (i == num_kb - 1) griddep_launch_dependents();
  };

  if (ct == 0) {
    tma_prefetch_desc(&map_a0);
    tma_prefetch_desc(&map_b);
    if (p.K1 > 0) tma_prefetch_desc(&map_a1);
    for (int s = 0; s < STAGES; ++s) mbar_init(full(s), 1);
    fence_barrier_init();
  }
  __syncthreads();
  griddep_wait();                                        // everything below may touch global memory
  if (ct == 0) {
    for (int i = 0; i < STAGES && i < num_kb; ++i) load(i);
    if (num_kb == 0) griddep_launch_dependents();
  }

  float acc[NR], dhi[NR], dlo[NR];
#pragma unroll
  for (int j = 0; j < NR; ++j) { acc[j] = 0.f; dhi[j] = 0.f; dlo[j] = 0.f; }

  uint32_t s = 0, ph = 0;
  int kin = 0;                                           // position of k-block i in its chunk
  for (int i = 0; i < num_kb; ++i) {
    const int b = i & 1;
    mbar_wait(full(s), ph);
    // split buffer b was last read by the wgmmas of k-block i-2: complete in this warpgroup after wait<1>, in both
    // after the barrier
    wgmma_wait<1>();
    cta_sync();
    split_tile<C::A_MN, BM, BK>(raw_a(s), a_hi(b), a_lo(b), ct);
    split_tile<C::B_MN, BN, BK>(raw_b(s), b_hi(b), b_lo(b), ct);
    fence_proxy_async();                                 // generic-proxy writes -> visible to the tensor core
    cta_sync();
    if (ct == 0 && i + STAGES < num_kb) load(i + STAGES);   // raw stage consumed by every thread: refill it
    __syncwarp();
    if (kin == 0 && i > 0) {                             // new chunk: fold the finished one into the running sum
      wgmma_wait<0>();
      fence_regs(dhi);
#pragma unroll
      for (int j = 0; j < NR; ++j) acc[j] = __fadd_rn(acc[j], dhi[j]);
    }
    const uint32_t da_hi = a_hi(b) + (uint32_t)wg * (64 * 128), da_lo = a_lo(b) + (uint32_t)wg * (64 * 128);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < BK / 8; ++k) {
      const uint64_t ah = gmma_desc_k128(da_hi + 32u * k), al = gmma_desc_k128(da_lo + 32u * k);
      const uint64_t bh = gmma_desc_k128(b_hi(b) + 32u * k), bl = gmma_desc_k128(b_lo(b) + 32u * k);
      wgmma_tf32(dlo, al, bh, (i == 0 && k == 0) ? 0u : 1u);
      wgmma_tf32(dlo, ah, bl, 1u);
      wgmma_tf32(dhi, ah, bh, (kin == 0 && k == 0) ? 0u : 1u);
    }
    wgmma_commit();
    if (++s == (uint32_t)STAGES) { s = 0; ph ^= 1u; }
    if (++kin == CH) kin = 0;
  }
  wgmma_wait<0>();
  fence_regs(dhi);
  fence_regs(dlo);
  if (num_kb > 0) {
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] = __fadd_rn(acc[j], dhi[j]);
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[j] = __fadd_rn(acc[j], dlo[j]);
  }

  // Stage the tile through shared memory (it reuses the split buffers: every wgmma has completed above, the barrier
  // makes that true for both warpgroups).  Accumulator fragment: warp w4 of a warpgroup holds rows 16*w4 + lane/4
  // (+8); register 4j + {0,1,2,3} is column 8j + 2*(lane%4) {+0, +1, +0, +1} of row {r, r, r+8, r+8}.
  cta_sync();
  float* tile = reinterpret_cast<float*>(smem_raw + (split0 - smem_u32(smem_raw)));
  {
    const int r0 = 64 * wg + 16 * ((ct >> 5) & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int j = 0; j < NR / 4; ++j) {
      *reinterpret_cast<float2*>(tile + r0 * C::EPI_LD + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(tile + (r0 + 8) * C::EPI_LD + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
  }
  cta_sync();
  constexpr int NC = C::COLS_PER_THREAD;
  const int row = ct & 127, g = ct >> 7;
  float out[NC];
#pragma unroll
  for (int j = 0; j < NC; j += 4) {
    const float4 v = *reinterpret_cast<const float4*>(tile + row * C::EPI_LD + g * NC + j);
    out[j] = v.x; out[j + 1] = v.y; out[j + 2] = v.z; out[j + 3] = v.w;
  }
  epilogue_row<EPI, NC>(epi, p, m0 + row, n0 + g * NC, z, out);
}

// ------------------------------------------------------------------ host side
// cuTensorMapEncodeTiled is fetched from the driver at run time (the library does not
// link libcuda, so it also loads on a box without a GPU).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn get_encode_fn();

// 2-D fp32 tensor [rows, cols] with row pitch ld (floats, multiple of 4); box = {box_cols, box_rows}.
// swizzle_bytes: 32 / 64 / 128 = the 16-byte-unit swizzles of that span.
int make_tmap(CUtensorMap* out, const float* base, int64_t rows, int64_t cols, int64_t ld, int box_cols,
              int box_rows, int swizzle_bytes);

// A global operand.  rows/cols describe the tensor as stored (only used for B; A's extents come
// from the Problem): K-major B is [N_total, K_total], MN-major B is [K_total, N_total].
struct Operand {
  const float* ptr;
  long long ld;
  long long rows, cols;
};

// k-blocks (of bk) per split and the effective split count for a requested split count.
int split_plan(int K_total_blocks, int splits_req, int* k_chunk, int bk = 16);

// Launch one GEMM.  Returns the effective number of k-splits (> 0) or a negative RECNN_E_* code.
template <bool A_MN, bool B_MN, int EPI>
int launch(const Operand& A0, const Operand& A1, const Operand& B, const Problem& p, int splits, int bn,
           const Epilogue& epi, cudaStream_t st);

}  // namespace tc
}  // namespace recnn
