// Non-GEMM kernels of the update step: critic head (256 -> 1) forward with the TD
// target / losses fused in, its backward, split-K partial reduction, the L1
// "clip" quirk, the fused optimizers and the Polyak update.  All of them touch
// a few MB that sit in L2; they exist to keep the launch count and the number
// of passes low, and to make every reduction order-deterministic.
#include "pointwise.cuh"

namespace recnn {

// Every block calls this after writing its partial result; returns true in the
// block that arrives last.  The ticket wraps to 0 so it never needs a reset.
__device__ __forceinline__ bool last_block_done(unsigned* ticket) {
  __shared__ bool is_last;
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned t = atomicInc(ticket, gridDim.x - 1);
    is_last = (t == gridDim.x - 1);
  }
  __syncthreads();
  return is_last;
}

// ---------------------------------------------------------------- critic head
__global__ void __launch_bounds__(256) critic_head_kernel(HeadArgs a) {
  __shared__ float red[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const float b3 = a.b3[0];
  const float inv_n = 1.0f / (float)a.n_rows_global;
  float warp_acc = 0.f;
  for (long long n = (long long)blockIdx.x * wpb + warp; n < a.n_rows; n += (long long)gridDim.x * wpb) {
    const float* row = a.h2 + n * a.hidden;
    float s = 0.f;
    for (int c = lane; c < a.hidden; c += 32) s = fmaf(row[c], __ldg(a.w3 + c), s);
    s = warp_sum(s);
    const float q = s + b3;
    if (lane == 0) {
      if (a.out) a.out[n] = q;
      switch (a.mode) {
        case HEAD_TARGET_DDPG: {
          // reward + (1.0 - done) * gamma * target, then clamp   (misc.py:6-7, :33-35)
          const float t = __fadd_rn(a.reward[n], __fmul_rn(__fmul_rn(__fsub_rn(1.0f, a.done[n]), a.gamma), q));
          a.y[n] = fminf(fmaxf(t, a.min_value), a.max_value);
        } break;
        case HEAD_TARGET_TD3_A: a.tmp[n] = q; break;
        case HEAD_TARGET_TD3_B: {
          const float qm = fminf(a.tmp[n], q);
          a.y[n] = __fadd_rn(a.reward[n], __fmul_rn(__fmul_rn(__fsub_rn(1.0f, a.done[n]), a.gamma), qm));
        } break;
        case HEAD_VALUE: {
          const float diff = __fsub_rn(q, a.y[n]);
          a.dq[n] = __fmul_rn(__fmul_rn(2.0f, diff), inv_n);
          warp_acc = __fadd_rn(warp_acc, __fmul_rn(diff, diff));
        } break;
        case HEAD_POLICY: warp_acc = __fsub_rn(warp_acc, q); break;
        default: break;
      }
    }
  }
  if (a.mode != HEAD_VALUE && a.mode != HEAD_POLICY) return;
  // deterministic two-level sum: warps in order, then blocks in order
  if (lane == 0) red[warp] = warp_acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < wpb; ++w) t += red[w];
    a.block_partials[blockIdx.x] = t;
  }
  if (last_block_done(a.ticket)) {
    float t = 0.f;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) t += a.block_partials[b];
    t = block_sum(t, red);
    if (threadIdx.x == 0) *a.loss = t / (float)a.n_rows_global;
  }
}

int launch_critic_head(const HeadArgs& a, cudaStream_t st) {
  if (a.n_rows <= 0) return RECNN_OK;
  const int64_t blocks = ceil_div(a.n_rows, 8);
  const int grid = (int)(blocks < 2 * kNumSMs ? blocks : 2 * kNumSMs);
  critic_head_kernel<<<grid, 256, 0, st>>>(a);
  RECNN_CHECK_LAUNCH("critic_head_kernel");
  return RECNN_OK;
}

// ---------------------------------------------------------------- fused critic head (value step)
template <int HC>   // hidden = 32 * HC
__global__ void __launch_bounds__(256) value_head_fused_kernel(ValueHeadArgs a) {
  constexpr int H = 32 * HC;
  __shared__ float red[8][H + 2];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float w3r[HC], tw3r[HC], gw[HC];
#pragma unroll
  for (int j = 0; j < HC; ++j) {
    w3r[j] = __ldg(a.w3 + lane + 32 * j);
    tw3r[j] = a.th2 ? __ldg(a.tw3 + lane + 32 * j) : 0.f;
    gw[j] = 0.f;
  }
  const float b3 = a.b3[0], tb3 = a.th2 ? a.tb3[0] : 0.f;
  const float inv_n = 1.0f / (float)a.n_rows_global;
  float gb = 0.f, lacc = 0.f;
  for (long long n = (long long)blockIdx.x * 8 + warp; n < a.n_rows; n += (long long)gridDim.x * 8) {
    float h[HC];
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < HC; ++j) {
      h[j] = a.h2[n * H + lane + 32 * j];
      s = fmaf(h[j], w3r[j], s);
    }
    const float q = warp_sum(s) + b3;
    float y;
    if (a.th2) {
      float t = 0.f;
#pragma unroll
      for (int j = 0; j < HC; ++j) t = fmaf(a.th2[n * H + lane + 32 * j], tw3r[j], t);
      const float tq = warp_sum(t) + tb3;
      // reward + (1.0 - done) * gamma * target, then clamp   (misc.py:6-7, :33-35)
      const float e = __fadd_rn(a.reward[n], __fmul_rn(__fmul_rn(__fsub_rn(1.0f, a.done[n]), a.gamma), tq));
      y = fminf(fmaxf(e, a.min_value), a.max_value);
      if (lane == 0) a.y[n] = y;
    } else {
      y = a.y[n];
    }
    const float diff = __fsub_rn(q, y);
    const float dq = __fmul_rn(__fmul_rn(2.0f, diff), inv_n);
    lacc = __fadd_rn(lacc, __fmul_rn(diff, diff));
    if (a.learn) {
#pragma unroll
      for (int j = 0; j < HC; ++j) {
        a.dz2[n * H + lane + 32 * j] = h[j] > 0.f ? __fmul_rn(__fmul_rn(dq, w3r[j]), a.gate_scale) : 0.f;
        gw[j] = fmaf(dq, h[j], gw[j]);
      }
      gb += dq;
    }
  }
  // warps in order, then blocks in order: deterministic
#pragma unroll
  for (int j = 0; j < HC; ++j) red[warp][lane + 32 * j] = gw[j];
  if (lane == 0) {
    red[warp][H] = gb;
    red[warp][H + 1] = lacc;
  }
  __syncthreads();
  for (int c = threadIdx.x; c < H + 2; c += blockDim.x) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += red[w][c];
    a.block_partials[(long long)blockIdx.x * (H + 2) + c] = t;
  }
  if (last_block_done(a.ticket)) {
    for (int c = threadIdx.x; c < H + 2; c += blockDim.x) {
      float t = 0.f;
      for (unsigned b = 0; b < gridDim.x; ++b) t += a.block_partials[(long long)b * (H + 2) + c];
      if (c < H) {
        if (a.learn) a.gw3[c] = t;
      } else if (c == H) {
        if (a.learn) a.gb3[0] = t;
      } else {
        *a.loss = t / (float)a.n_rows_global;
      }
    }
  }
}

bool value_head_fusable(int hidden) { return hidden % 32 == 0 && hidden >= 32 && hidden <= 256; }

int launch_value_head_fused(const ValueHeadArgs& a, cudaStream_t st) {
  if (a.n_rows <= 0) return RECNN_OK;
  RECNN_REQUIRE(value_head_fusable(a.hidden), "fused value head needs hidden = 32..256, multiple of 32");
  const int64_t blocks = ceil_div(a.n_rows, 8);
  const int grid = (int)(blocks < kNumSMs ? blocks : kNumSMs);
  switch (a.hidden / 32) {
#define RECNN_VH_CASE(HC) case HC: value_head_fused_kernel<HC><<<grid, 256, 0, st>>>(a); break;
    RECNN_VH_CASE(1) RECNN_VH_CASE(2) RECNN_VH_CASE(3) RECNN_VH_CASE(4)
    RECNN_VH_CASE(5) RECNN_VH_CASE(6) RECNN_VH_CASE(7) RECNN_VH_CASE(8)
#undef RECNN_VH_CASE
    default: break;
  }
  RECNN_CHECK_LAUNCH("value_head_fused_kernel");
  return RECNN_OK;
}

__global__ void __launch_bounds__(256)
critic_head_bwd_kernel(const float* __restrict__ dq, float dq_const, const float* __restrict__ w3,
                       const float* __restrict__ h2, float gate_scale, float* __restrict__ dz2,
                       long long total, int hidden) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / hidden;
    const int c = (int)(i - n * hidden);
    const float g = dq ? dq[n] : dq_const;
    dz2[i] = h2[i] > 0.f ? __fmul_rn(__fmul_rn(g, __ldg(w3 + c)), gate_scale) : 0.f;
  }
}

int launch_critic_head_bwd(const float* dq, float dq_const, const float* w3, const float* h2,
                           float gate_scale, float* dz2, int64_t n_rows, int hidden, cudaStream_t st) {
  const int64_t total = n_rows * hidden;
  if (total <= 0) return RECNN_OK;
  const int64_t blocks = ceil_div(total, 256);
  const int grid = (int)(blocks < 8 * kNumSMs ? blocks : 8 * kNumSMs);
  critic_head_bwd_kernel<<<grid, 256, 0, st>>>(dq, dq_const, w3, h2, gate_scale, dz2, total, hidden);
  RECNN_CHECK_LAUNCH("critic_head_bwd_kernel");
  return RECNN_OK;
}

// ---------------------------------------------------------------- split-K reduce
__global__ void __launch_bounds__(256)
reduce_partials_kernel(const float* __restrict__ part, int splits, int C, int K1,
                       float* __restrict__ w_dst, long long ldw, float* __restrict__ b_dst) {
  const long long total = (long long)C * K1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
       i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < splits; ++z) s += part[(long long)z * total + i];     // fixed order: deterministic
    const int c = (int)(i / K1), k = (int)(i - (long long)c * K1);
    if (k < K1 - 1) w_dst[(long long)c * ldw + k] = s;
    else b_dst[c] = s;
  }
}

int launch_reduce_partials(const float* part, int splits, int C, int K1, float* w_dst, long long ldw,
                           float* b_dst, cudaStream_t st) {
  const int64_t total = (int64_t)C * K1;
  const int64_t blocks = ceil_div(total, 256);
  const int grid = (int)(blocks < 8 * kNumSMs ? blocks : 8 * kNumSMs);
  reduce_partials_kernel<<<grid, 256, 0, st>>>(part, splits, C, K1, w_dst, ldw, b_dst);
  RECNN_CHECK_LAUNCH("reduce_partials_kernel");
  return RECNN_OK;
}

// Column sums of dZ [n_rows, C] per row-split, written into column K1-1 of the split-K partial
// buffer part[z][c][K1] (the bias-gradient column next to a tensor-core weight gradient).
__global__ void __launch_bounds__(256)
colsum_partials_kernel(const float* __restrict__ dz, long long n_rows, int C, long long rows_per_split,
                       float* __restrict__ part, int K1) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx, z = blockIdx.y;
  const long long r0 = (long long)z * rows_per_split;
  const long long r1 = min(n_rows, r0 + rows_per_split);
  float s = 0.f;
  if (c < C)
    for (long long r = r0 + ry; r < r1; r += 8) s += dz[r * C + c];
  red[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][cx];
    part[((long long)z * C + c) * K1 + (K1 - 1)] = t;
  }
}

// Critic head weight gradient (the 256 -> 1 layer): part[z][0][c] = sum_r dq[r] * h2[r, c] over the
// rows of split z, part[z][0][H] = sum_r dq[r]   (dW3 = dq^T h2, db3 = sum dq; misc.py:43 backward).
__global__ void __launch_bounds__(256)
head_grad_partials_kernel(const float* __restrict__ dq, const float* __restrict__ h2, long long n_rows, int H,
                          long long rows_per_split, float* __restrict__ part) {
  __shared__ float red[8][33];
  const int cx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + cx, z = blockIdx.y;
  const long long r0 = (long long)z * rows_per_split;
  const long long r1 = min(n_rows, r0 + rows_per_split);
  float s = 0.f;
  if (c < H) {
    for (long long r = r0 + ry; r < r1; r += 8) s = fmaf(dq[r], h2[r * H + c], s);
  } else if (c == H) {
    for (long long r = r0 + ry; r < r1; r += 8) s += dq[r];
  }
  red[ry][cx] = s;
  __syncthreads();
  if (ry == 0 && c <= H) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += red[i][cx];
    part[(long long)z * (H + 1) + c] = t;
  }
}

int launch_head_grad_partials(const float* dq, const float* h2, int64_t n_rows, int H, int64_t rows_per_split,
                              int splits, float* part, cudaStream_t st) {
  dim3 grid((unsigned)ceil_div(H + 1, 32), (unsigned)splits);
  head_grad_partials_kernel<<<grid, 256, 0, st>>>(dq, h2, n_rows, H, rows_per_split, part);
  RECNN_CHECK_LAUNCH("head_grad_partials_kernel");
  return RECNN_OK;
}

int launch_colsum_partials(const float* dz, int64_t n_rows, int C, int64_t rows_per_split, int splits,
                           float* part, int K1, cudaStream_t st) {
  dim3 grid((unsigned)ceil_div(C, 32), (unsigned)splits);
  colsum_partials_kernel<<<grid, 256, 0, st>>>(dz, n_rows, C, rows_per_split, part, K1);
  RECNN_CHECK_LAUNCH("colsum_partials_kernel");
  return RECNN_OK;
}

// ---------------------------------------------------------------- pad columns of the action images
__global__ void __launch_bounds__(256)
zero_pad_columns_kernel(float* b0, float* b1, float* b2, long long n_rows, int ld, int lead, int cols) {
  const int pads = ld - cols;                         // lead + trailing pad columns per row
  float* const bufs[3] = {b0, b1, b2};
  float* const buf = bufs[blockIdx.y];
  if (!buf) return;
  const long long total = n_rows * pads;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / pads;
    const int k = (int)(i - r * pads);
    const int col = k < lead ? k : lead + cols + (k - lead);     // lead pads, then the pads behind the data
    buf[r * ld + col] = 0.f;
  }
}

int launch_zero_pad_columns(float* b0, float* b1, float* b2, int64_t n_rows, int ld, int lead, int cols, cudaStream_t st) {
  RECNN_REQUIRE(ld >= lead + cols && lead >= 0 && cols > 0, "pad geometry");
  if (ld == lead + cols && lead == 0) return RECNN_OK;
  if (n_rows <= 0) return RECNN_OK;
  const int64_t total = n_rows * (ld - cols);
  const int64_t blocks = ceil_div(total, 256);
  dim3 grid((unsigned)(blocks < kNumSMs ? blocks : kNumSMs), 3);
  zero_pad_columns_kernel<<<grid, 256, 0, st>>>(b0, b1, b2, n_rows, ld, lead, cols);
  RECNN_CHECK_LAUNCH("zero_pad_columns_kernel");
  return RECNN_OK;
}

// ---------------------------------------------------------------- L1 clip quirk
__global__ void __launch_bounds__(256)
l1_clip_coef_kernel(const float* __restrict__ g, long long count, float max_norm, float* coef, float* l1_out,
                    float* block_partials, unsigned* ticket) {
  __shared__ float red[32];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x)
    s += fabsf(g[i]);
  s = block_sum(s, red);
  if (threadIdx.x == 0) block_partials[blockIdx.x] = s;
  if (last_block_done(ticket)) {
    float t = 0.f;
    for (unsigned b = threadIdx.x; b < gridDim.x; b += blockDim.x) t += block_partials[b];
    t = block_sum(t, red);
    if (threadIdx.x == 0) {
      // clip_coef = max_norm / (total_norm + 1e-6), clamped from above at 1.0
      const float c = max_norm / (t + 1e-6f);
      *coef = fminf(c, 1.0f);
      if (l1_out) *l1_out = t;
    }
  }
}

int launch_l1_clip_coef(const float* grads, int64_t count, float max_norm, float* coef, float* l1_out,
                        float* block_partials, unsigned* ticket, cudaStream_t st) {
  const int64_t blocks = ceil_div(count, 256 * 8);
  const int grid = (int)(blocks < 2 * kNumSMs ? (blocks > 0 ? blocks : 1) : 2 * kNumSMs);
  l1_clip_coef_kernel<<<grid, 256, 0, st>>>(grads, count, max_norm, coef, l1_out, block_partials, ticket);
  RECNN_CHECK_LAUNCH("l1_clip_coef_kernel");
  return RECNN_OK;
}

__global__ void scale_inplace_kernel(float* x, long long count, const float* scale) {
  const float s = *scale;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x)
    x[i] = __fmul_rn(x[i], s);
}

int launch_scale_inplace(float* x, int64_t count, const float* scale, cudaStream_t st) {
  const int64_t blocks = ceil_div(count, 256);
  const int grid = (int)(blocks < 4 * kNumSMs ? (blocks > 0 ? blocks : 1) : 4 * kNumSMs);
  scale_inplace_kernel<<<grid, 256, 0, st>>>(x, count, scale);
  RECNN_CHECK_LAUNCH("scale_inplace_kernel");
  return RECNN_OK;
}

// ---------------------------------------------------------------- optimizers
// torch.optim.Adam / SGD (single-tensor CPU path of torch 2.11), one flat arena.  The per-element math lives in
// pointwise.cuh (opt_apply) so that the all-reduce kernel of the data-parallel step can apply the very same update.
__global__ void __launch_bounds__(256)
optimizer_kernel(int kind, OptConsts k, double beta1, double beta2, double lr, double wd, double n_sma_threshold,
                 int k_look, float* __restrict__ p, float* __restrict__ g, float* __restrict__ m,
                 float* __restrict__ v, float* __restrict__ slow, int* __restrict__ t_ptr,
                 const float* __restrict__ grad_scale, long long count, unsigned* ticket, GradSource src) {
  __shared__ OptStep s_st;
  const int t = *t_ptr + 1;
  if (threadIdx.x == 0) s_st = opt_step_scalars(kind, beta1, beta2, lr, wd, n_sma_threshold, k_look, t);
  __syncthreads();
  const OptStep st = s_st;
  const float gs = grad_scale ? *grad_scale : 1.0f;
  if (src.n_layers) {
    // gradient still in split-K partials (arena: count % 4 == 0, 16-byte aligned): four elements per thread
    for (long long i4 = (long long)blockIdx.x * blockDim.x + threadIdx.x; i4 < (count >> 2);
         i4 += (long long)gridDim.x * blockDim.x) {
      float4 gv = grad4_at(src, g, (unsigned)(4 * i4));
      if (grad_scale) {
        gv.x = __fmul_rn(gv.x, gs); gv.y = __fmul_rn(gv.y, gs); gv.z = __fmul_rn(gv.z, gs); gv.w = __fmul_rn(gv.w, gs);
      }
      *reinterpret_cast<float4*>(g + 4 * i4) = gv;       // .grad holds what the optimizer consumed
      opt_apply(kind, k, st, t, p, m, v, slow, 4 * i4 + 0, gv.x);
      opt_apply(kind, k, st, t, p, m, v, slow, 4 * i4 + 1, gv.y);
      opt_apply(kind, k, st, t, p, m, v, slow, 4 * i4 + 2, gv.z);
      opt_apply(kind, k, st, t, p, m, v, slow, 4 * i4 + 3, gv.w);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
         i += (long long)gridDim.x * blockDim.x) {
      float grad = g[i];
      if (grad_scale) {
        grad = __fmul_rn(grad, gs);
        g[i] = grad;                      // the reference leaves the scaled grad in .grad
      }
      opt_apply(kind, k, st, t, p, m, v, slow, i, grad);
    }
  }
  // ++t by the block that finishes last (every block has read t by then); without a ticket the
  // launcher appends a one-thread kernel instead
  if (ticket) {
    if (last_block_done(ticket) && threadIdx.x == 0) *t_ptr = t;
  }
}

__global__ void bump_counter_kernel(int* t) { *t += 1; }
__global__ void bump_counter64_kernel(long long* t) { *t += 1; }

// end of a step: ++*rng_step (if any) and the step's error words -> one int in the caller's loss block
__global__ void finish_kernel(long long* rng_step, const unsigned* oob, const unsigned* dp_mismatch, float* flags_out) {
  if (rng_step) *rng_step += 1;
  const int bits = (*oob ? 1 : 0) | (*dp_mismatch ? 2 : 0);
  *reinterpret_cast<int*>(flags_out) = bits;
}
int launch_finish(long long* rng_step, const unsigned* oob, const unsigned* dp_mismatch, float* flags_out,
                  cudaStream_t st) {
  finish_kernel<<<1, 1, 0, st>>>(rng_step, oob, dp_mismatch, flags_out);
  RECNN_CHECK_LAUNCH("finish_kernel");
  return RECNN_OK;
}

int launch_bump64(long long* t, cudaStream_t st) {
  bump_counter64_kernel<<<1, 1, 0, st>>>(t);
  RECNN_CHECK_LAUNCH("bump_counter64_kernel");
  return RECNN_OK;
}

int launch_optimizer(const recnn_optim& o, const recnn_net& net, int64_t count, const float* grad_scale,
                     cudaStream_t st, unsigned* ticket, const GradSource* src) {
  RECNN_REQUIRE(o.kind == RECNN_OPT_SGD || o.kind == RECNN_OPT_ADAM || o.kind == RECNN_OPT_RANGER,
                "built-in optimizer kind must be SGD, ADAM or RANGER");
  RECNN_REQUIRE(net.params && net.grads && net.opt_t, "optimizer needs params, grads and the step counter");
  if (o.kind == RECNN_OPT_ADAM) RECNN_REQUIRE(net.opt_m && net.opt_v, "Adam needs exp_avg / exp_avg_sq arenas");
  if (o.kind == RECNN_OPT_RANGER) RECNN_REQUIRE(net.opt_m && net.opt_v && net.opt_slow, "Ranger needs exp_avg / exp_avg_sq / slow arenas");
  if (o.kind == RECNN_OPT_SGD && o.momentum != 0.f) RECNN_REQUIRE(net.opt_m, "SGD momentum needs a buffer arena");
  const OptConsts k = opt_consts(o);
  GradSource gs;
  memset(&gs, 0, sizeof(gs));
  if (src) {
    RECNN_REQUIRE(count % 4 == 0 && (reinterpret_cast<uintptr_t>(net.grads) & 15) == 0, "partial-sourced gradients need a 16-byte aligned arena");
    gs = *src;
  }
  const int64_t blocks = ceil_div(count, 256 * 4);
  const int grid = (int)(blocks < 4 * kNumSMs ? (blocks > 0 ? blocks : 1) : 4 * kNumSMs);
  optimizer_kernel<<<grid, 256, 0, st>>>(o.kind, k, o.beta1, o.beta2, o.lr, o.weight_decay, o.n_sma_threshold, o.k,
                                         net.params, net.grads, net.opt_m, net.opt_v, net.opt_slow, net.opt_t,
                                         grad_scale, count, ticket, gs);
  RECNN_CHECK_LAUNCH("optimizer_kernel");
  if (!ticket) {
    bump_counter_kernel<<<1, 1, 0, st>>>(net.opt_t);
    RECNN_CHECK_LAUNCH("bump_counter_kernel");
  }
  return RECNN_OK;
}

// ---------------------------------------------------------------- Polyak
__global__ void __launch_bounds__(256)
polyak_kernel(float* __restrict__ target, const float* __restrict__ net, long long count, float one_minus_tau,
              float tau) {
  // target.data * (1.0 - soft_tau) + param.data * soft_tau   (recnn/utils/misc.py:3-5)
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < count;
       i += (long long)gridDim.x * blockDim.x)
    target[i] = __fadd_rn(__fmul_rn(target[i], one_minus_tau), __fmul_rn(net[i], tau));
}

int launch_polyak(float* target, const float* net, int64_t count, double tau, cudaStream_t st) {
  const int64_t blocks = ceil_div(count, 256 * 4);
  const int grid = (int)(blocks < 4 * kNumSMs ? (blocks > 0 ? blocks : 1) : 4 * kNumSMs);
  polyak_kernel<<<grid, 256, 0, st>>>(target, net, count, (float)(1.0 - tau), (float)tau);
  RECNN_CHECK_LAUNCH("polyak_kernel");
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

extern "C" int recnn_polyak_update(float* target, const float* net, int64_t count, double tau, void* stream) {
  RECNN_REQUIRE(target && net && count >= 0, "target/net must be non-null");
  if (count == 0) return RECNN_OK;
  return launch_polyak(target, net, count, tau, static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_optimizer_step(const recnn_optim* o, const recnn_net* net, int64_t count,
                                    const float* grad_scale, void* stream) {
  RECNN_REQUIRE(o && net && count > 0, "optimizer/net must be non-null");
  return launch_optimizer(*o, *net, count, grad_scale, static_cast<cudaStream_t>(stream));
}
