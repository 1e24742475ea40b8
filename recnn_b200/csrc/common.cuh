// Shared device/host helpers for the recnn_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/recnn_b200.h"

namespace recnn {

// ---- error plumbing ---------------------------------------------------------
void set_error(const char* fmt, ...);
void count_launch();   // every kernel launch of this library bumps a process-wide counter

#define RECNN_CHECK_CUDA(expr)                                                        \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess) {                                                          \
      ::recnn::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),      \
                         __FILE__, __LINE__);                                         \
      return RECNN_E_CUDA;                                                            \
    }                                                                                 \
  } while (0)

#define RECNN_CHECK_LAUNCH(name)                                                      \
  do {                                                                                \
    cudaError_t _e = cudaGetLastError();                                              \
    if (_e != cudaSuccess) {                                                          \
      ::recnn::set_error("launch of %s failed: %s (%s:%d)", name,                     \
                         cudaGetErrorString(_e), __FILE__, __LINE__);                 \
      return RECNN_E_CUDA;                                                            \
    }                                                                                 \
    ::recnn::count_launch();                                                          \
  } while (0)

#define RECNN_REQUIRE(cond, msg)                                                      \
  do {                                                                                \
    if (!(cond)) {                                                                    \
      ::recnn::set_error("invalid argument: %s (%s)", msg, #cond);                    \
      return RECNN_E_INVALID;                                                         \
    }                                                                                 \
  } while (0)

#define RECNN_PROPAGATE(expr)                                                         \
  do {                                                                                \
    int _s = (expr);                                                                  \
    if (_s != RECNN_OK) return _s;                                                    \
  } while (0)

constexpr int kNumSMs = 132;   // H100 SXM: grid caps; kernels that need every CTA resident query the device

static inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }
static inline int64_t round_up(int64_t a, int64_t b) { return ceil_div(a, b) * b; }

// ---- caller-provided workspace / scratch ------------------------------------
// Every entry point lays out the memory it is given with ONE layout function over a Carve: run on a null base it only
// sizes (the *_workspace_bytes / *_scratch_floats queries), run on the caller's pointer it cuts the same slices, so
// the query and the call cannot disagree.  Every slice starts on a 256-byte boundary (TMA needs 16).  The base is
// aligned up first and the size counts that slack, so any caller address works.
constexpr int64_t kCarveAlign = 256;
struct Carve {
  char* base;        // aligned; null: sizing only
  int64_t off = 0;
  explicit Carve(void* p)
      : base(p ? reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + kCarveAlign - 1) &
                                         ~static_cast<uintptr_t>(kCarveAlign - 1))
               : nullptr) {}
  template <class T = float>
  T* take(int64_t count) {
    T* r = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += round_up(count * (int64_t)sizeof(T), kCarveAlign);
    return r;
  }
  int64_t bytes() const { return off + kCarveAlign; }     // + the slack of aligning an arbitrary base
  int64_t floats() const { return ceil_div(bytes(), 4); }
};

// RECNN_E_WORKSPACE (with both sizes in the message) unless the caller's `have` bytes hold a layout of `need` bytes
static inline int check_workspace(int64_t need, int64_t have) {
  if (need <= have) return RECNN_OK;
  set_error("workspace too small: need %lld bytes, got %lld", (long long)need, (long long)have);
  return RECNN_E_WORKSPACE;
}

// ---- arena layout of one MLP (nn.Module.parameters() order) -----------------
// Weight rows are padded to a multiple of 4 floats (16 bytes) so that every matrix in the arena is
// a legal TMA tensor: linear1.weight of the Actor is [H, 1290] with row pitch 1292, of the Critic
// [H, 1418] with pitch 1420.  The nn.Parameter objects on the Python side are strided views of the
// arena, so the padding is invisible to state_dict / optimizers; pad elements stay 0 forever
// (their gradient is never written, Adam/SGD/Polyak of 0 with 0 is 0).
struct NetLayout {
  int in_dim, hidden, out_dim;
  int ld1, ld2, ld3;                 // row pitches of w1 [H,in], w2 [H,H], w3 [out,H]
  int64_t w1, b1, w2, b2, w3, b3, count;
  __host__ __device__ NetLayout() {}
  __host__ __device__ NetLayout(int in_, int h, int out_) : in_dim(in_), hidden(h), out_dim(out_) {
    ld1 = (in_ + 3) / 4 * 4;
    ld2 = (h + 3) / 4 * 4;
    ld3 = (h + 3) / 4 * 4;
    const int64_t hb = (h + 3) / 4 * 4, ob = (out_ + 3) / 4 * 4;
    w1 = 0;
    b1 = w1 + (int64_t)h * ld1;
    w2 = b1 + hb;
    b2 = w2 + (int64_t)h * ld2;
    w3 = b2 + hb;
    b3 = w3 + (int64_t)out_ * ld3;
    count = b3 + ob;
  }
};
static inline NetLayout actor_layout(const recnn_dims& d) {
  return NetLayout(d.state_dim, d.hidden, d.action_dim);
}
static inline NetLayout critic_layout(const recnn_dims& d) {
  return NetLayout(d.state_dim + d.action_dim, d.hidden, 1);
}
static inline int pad4(int n) { return (n + 3) / 4 * 4; }

// ---- warp helpers -----------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum in a fixed order (deterministic). `red` needs >= 32 floats.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : 0.f;
  if (warp == 0) t = warp_sum(t);
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  t = red[0];
  return t;
}

// 16-byte global -> shared copy that bypasses the registers (cp.async; both addresses 16-byte aligned)
__device__ __forceinline__ void cp_async16(float* dst, const float* src) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(src) : "memory");
}

// ---- Philox4x32-10 (perf-mode dropout / TD3 noise) ---------------------------
struct Philox {
  uint32_t key0, key1;
  __device__ __forceinline__ Philox(uint64_t seed) : key0((uint32_t)seed), key1((uint32_t)(seed >> 32)) {}
  __device__ __forceinline__ uint4 operator()(uint64_t ctr_lo, uint64_t ctr_hi) const {
    uint32_t c0 = (uint32_t)ctr_lo, c1 = (uint32_t)(ctr_lo >> 32);
    uint32_t c2 = (uint32_t)ctr_hi, c3 = (uint32_t)(ctr_hi >> 32);
    uint32_t k0 = key0, k1 = key1;
#pragma unroll
    for (int r = 0; r < 10; ++r) {
      const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
      const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
      c0 = hi1 ^ c1 ^ k0;
      c1 = lo1;
      c2 = hi0 ^ c3 ^ k1;
      c3 = lo0;
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    return make_uint4(c0, c1, c2, c3);
  }
};

// Dropout keep-bit for element `idx` of mask stream `stream_id` at rng step `step`.
// One Philox call yields 128 bits = 128 consecutive elements' keep bits.
__device__ __forceinline__ uint32_t philox_keep_bits32(uint64_t seed, uint64_t step, uint32_t stream_id,
                                                       uint64_t word_idx /* idx/32 */) {
  Philox ph(seed);
  const uint4 r = ph(word_idx >> 2, (step << 8) | stream_id);
  const uint32_t w = (uint32_t)(word_idx & 3);
  return w == 0 ? r.x : (w == 1 ? r.y : (w == 2 ? r.z : r.w));
}

}  // namespace recnn
