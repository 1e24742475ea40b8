// The behaviour policy beta of REINFORCE with Top-K correction: class Beta of the reference's Top-K notebook
// (examples/2. REINFORCE TopK Off Policy Correction/3. TopK Reinforce Off Policy Correction.ipynb, cell 3), one
// training step per forward call.  Included at the end of step.cu after reinforce.cuh and critic_ids.cuh: it reuses
// linear_out / weight_grad on row-offset weight pointers, the online max / sum fold (logit_stats_kernel), the ordered
// row sum and the chunk rule.
//
// For rows s_n with target ids a_n:  z = W s + b,  p = softmax(z) (dim 1),  L = mean_n(-log_softmax(p_n)[a_n]).
// CrossEntropyLoss is applied to the probabilities -- a softmax of a softmax, as the notebook does.  With
// T = sum_j e^{p_j} and U = sum_j p_j e^{p_j}:
//   dL/dz_nj = (p_nj / N) ((e^{p_nj} - U_n) / T_n + p_{n,a_n} - [j == a_n]),   dW = dZ^T S,  db = colsum dZ.
// Every p is about 1/num_items, so e^p ~ 1, T ~ num_items and the signal of e^{p_j} - U is of order p: summed as
// e^p in fp32 it is lost.  Hence the expm1 form, with sum_j p_j = 1:
//   T = num_items + sum expm1(p),   e^{p_j} - U = expm1(p_j) - sum_k p_k expm1(p_k),   L_n = log T_n - p_{n,a_n}.
//
// Passes: (1) per item chunk, the logits go straight into the caller's probs_out [N, num_items] (the notebook's
// return value) and are folded into a running max / sum; (2) one CTA per row turns them into p in place and forms
// the row's T, sum p expm1(p), p_a and loss term; (3) per chunk in a fixed order, dZ [N, w] from probs_out, the
// chunk's dW rows (split-K partials reduced into the gradient arena) and db slice; (4) the built-in optimizer over the
// arena, skipped on the device when an id was out of range.  No float atomics: repeats are bit-identical.
#pragma once

namespace recnn {

struct BetaLayout {
  int ldw;                   // row pitch of the weight [num_items, S]: pad4(S), so every chunk starts 16-byte aligned
  int64_t w, b, count;
};
static inline BetaLayout beta_layout(const recnn_beta_dims& d) {
  BetaLayout l;
  l.ldw = pad4(d.state_dim);
  l.w = 0;
  l.b = (int64_t)d.num_items * l.ldw;
  l.count = l.b + pad4(d.num_items);
  return l;
}

struct BetaWorkspace {
  float* img;                                          // [n, pad4(S)] state image (when the state is not TMA-legal)
  float* dz;                                           // [n, chunk] one chunk of dL/dz
  float *run_max, *run_sum, *za, *T, *pe, *pa, *row_loss;   // [n]
  float* partial;                                      // split-K partials of one chunk's dW
  unsigned* flags;                                     // [0] error bit, [1] optimizer ticket
  int64_t bytes;
};

static BetaWorkspace beta_carve(const recnn_beta_dims& d, int64_t n, int chunk, void* base) {
  BetaWorkspace w;
  char* p = static_cast<char*>(base);
  int64_t off = 0;
  auto take = [&](int64_t floats) {
    float* r = base ? reinterpret_cast<float*>(p + off) : nullptr;
    off += round_up(floats * 4, 256);
    return r;
  };
  w.img = take(n * pad4(d.state_dim));
  w.dz = take(n * (int64_t)chunk);
  float** rows[7] = {&w.run_max, &w.run_sum, &w.za, &w.T, &w.pe, &w.pa, &w.row_loss};
  for (auto r : rows) *r = take(n);
  w.partial = take(chunked_partial_floats(chunk, d.num_items, d.state_dim, n));
  w.flags = reinterpret_cast<unsigned*>(take(8));
  w.bytes = off;
  return w;
}

static bool beta_dims_ok(const recnn_beta_dims* d) { return d && d->state_dim > 0 && d->num_items > 0; }

// Logits -> p in place (the row's max / sum of exp from pass 1), then the row's T, sum p expm1(p), p_a and loss term.
// An id outside [0, items) flags *err; its row adds no loss (and, in beta_dz_kernel, no gradient).  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
beta_rows_kernel(float* __restrict__ P, long long ld, long long n, int items, const long long* __restrict__ action,
                 const float* __restrict__ run_max, const float* __restrict__ run_sum, const float* __restrict__ za,
                 float* __restrict__ T_out, float* __restrict__ pe_out, float* __restrict__ pa_out,
                 float* __restrict__ row_loss, unsigned* err) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float* row = P + r * ld;
    const float M = run_max[r], S = run_sum[r];
    float s1 = 0.f, s2 = 0.f;
    for (int j = threadIdx.x; j < items; j += blockDim.x) {
      const float p = expf(row[j] - M) / S;            // softmax_rows_kernel's normalisation
      row[j] = p;
      const float e = expm1f(p);
      s1 += e;
      s2 += p * e;
    }
    s1 = block_sum(s1, red);
    s2 = block_sum(s2, red);
    if (threadIdx.x == 0) {
      const long long a = action[r];
      const bool ok = a >= 0 && a < items;
      const float pa = ok ? expf(za[r] - M) / S : 0.f;   // == row[a]
      const float T = (float)items + s1;
      T_out[r] = T;
      pe_out[r] = s2;
      pa_out[r] = pa;
      row_loss[r] = ok ? logf(T) - pa : 0.f;
      if (!ok) *err = 1u;
    }
    __syncthreads();
  }
}

// dz[r, j] = (p / n) ((expm1(p) - pe_r) / T_r + pa_r - [c0 + j == a_r]) over the chunk's w items of probs (pitch ld);
// zero for a row whose id is out of range.  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
beta_dz_kernel(const float* __restrict__ P, long long ld, long long n, int w, int c0, int items,
               const long long* __restrict__ action, const float* __restrict__ T, const float* __restrict__ pe,
               const float* __restrict__ pa, float inv_n, float* __restrict__ dz) {
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float* row = P + r * ld + c0;
    float* out = dz + r * w;
    const long long a = action[r];
    if (a < 0 || a >= items) {
      for (int j = threadIdx.x; j < w; j += blockDim.x) out[j] = 0.f;
      continue;
    }
    const long long al = a - c0;                       // outside [0, w) when the target is in another chunk
    const float t = T[r], e = pe[r], q = pa[r];
    for (int j = threadIdx.x; j < w; j += blockDim.x) {
      const float p = row[j];
      const float g = (expm1f(p) - e) / t + q - (j == al ? 1.f : 0.f);
      out[j] = p * inv_n * g;
    }
  }
}

}  // namespace recnn

using namespace recnn;

extern "C" int recnn_beta_layout(const recnn_beta_dims* d, int64_t* out) {
  RECNN_REQUIRE(beta_dims_ok(d) && out, "dims / out");
  const BetaLayout l = beta_layout(*d);
  out[0] = l.w; out[1] = l.b; out[2] = l.ldw; out[3] = l.count;
  return RECNN_OK;
}

extern "C" int64_t recnn_beta_workspace_bytes(const recnn_beta_dims* d, int64_t n_rows, int32_t chunk_items) {
  if (!beta_dims_ok(d) || n_rows <= 0 || !critic_chunk_ok(d->num_items, chunk_items)) return 0;
  return beta_carve(*d, n_rows, chunk_items, nullptr).bytes;
}

extern "C" int64_t recnn_sizeof_beta_args(void) { return (int64_t)sizeof(recnn_beta_args); }
extern "C" int64_t recnn_offsetof_beta_args(int field) {
  switch (field) {
    case 0: return offsetof(recnn_beta_args, dims);
    case 1: return offsetof(recnn_beta_args, n_rows);
    case 2: return offsetof(recnn_beta_args, net);
    case 3: return offsetof(recnn_beta_args, optim);
    case 4: return offsetof(recnn_beta_args, state);
    case 5: return offsetof(recnn_beta_args, action);
    case 6: return offsetof(recnn_beta_args, probs_out);
    case 7: return offsetof(recnn_beta_args, loss);
    case 8: return offsetof(recnn_beta_args, error);
    case 9: return offsetof(recnn_beta_args, workspace_bytes);
    default: return -1;
  }
}

// Beta.forward(state, action) of the notebook's cell 3: forward, CrossEntropyLoss on the probabilities, zero_grad +
// backward, optim.step(); probs_out holds the pre-step probabilities.
extern "C" int recnn_beta_step(const recnn_beta_args* a, void* stream) {
  RECNN_REQUIRE(a != nullptr, "args");
  RECNN_REQUIRE(beta_dims_ok(&a->dims), "dims");
  RECNN_REQUIRE(a->n_rows > 0, "n_rows");
  const int S = a->dims.state_dim, I = a->dims.num_items, W = a->chunk_items;
  RECNN_REQUIRE(critic_chunk_ok(I, W), "chunk_items must be num_items or a positive multiple of 128 below it");
  const int64_t widest = pad4(S) > W ? pad4(S) : W;
  RECNN_REQUIRE(a->n_rows < (1ll << 31) / (widest + 1), "n_rows too large for int32 tile indexing");
  RECNN_REQUIRE(a->state && a->state_ld >= S && a->action, "state / state_ld / action");
  RECNN_REQUIRE(a->probs_out && a->loss && a->error && a->workspace, "probs_out / loss / error / workspace");
  RECNN_REQUIRE(a->net.params && a->net.grads, "net needs params and grads");
  const int64_t n = a->n_rows;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const BetaWorkspace w = beta_carve(a->dims, n, W, a->workspace);
  if (w.bytes > a->workspace_bytes) {
    set_error("workspace too small: need %lld bytes, got %lld", (long long)w.bytes, (long long)a->workspace_bytes);
    return RECNN_E_WORKSPACE;
  }
  const BetaLayout l = beta_layout(a->dims);
  const float* P = a->net.params;
  float* G = a->net.grads;
  float* probs = a->probs_out;
  const long long* act = reinterpret_cast<const long long*>(a->action);
  const int n_chunks = (int)ceil_div(I, W);
  RECNN_CHECK_CUDA(cudaMemsetAsync(w.flags, 0, 8 * sizeof(unsigned), st));
  recnn_dims dd;
  memset(&dd, 0, sizeof(dd));
  dd.state_dim = S;
  Seg xs;
  RECNN_PROPAGATE(repitch_state(dd, a->state, n, w.img, &xs, st, a->state_ld));
  // pass 1: logits of each chunk into probs_out, folded into the row's running max / sum of exp; the target's logit
  for (int c = 0; c < n_chunks; ++c) {
    const int c0 = c * W, wc = I - c0 < W ? I - c0 : W;
    RECNN_PROPAGATE(linear_out(xs, P + l.w + (int64_t)c0 * l.ldw, l.ldw, P + l.b + c0, wc, n, 0, nullptr, probs + c0, I,
                               st));
    logit_stats_kernel<<<row_grid(n), kRowThreads, 0, st>>>(probs + c0, I, n, wc, c0, act, w.run_max, w.run_sum, w.za);
    RECNN_CHECK_LAUNCH("logit_stats_kernel");
  }
  beta_rows_kernel<<<row_grid(n), kRowThreads, 0, st>>>(probs, I, n, I, act, w.run_max, w.run_sum, w.za, w.T, w.pe,
                                                        w.pa, w.row_loss, w.flags);
  RECNN_CHECK_LAUNCH("beta_rows_kernel");
  sum_rows_kernel<<<1, 1024, 0, st>>>(w.row_loss, n, (float)(1.0 / (double)n), a->loss);
  RECNN_CHECK_LAUNCH("sum_rows_kernel");
  // pass 2: dZ of each chunk, its dW rows and db slice (overwriting the arena: zero_grad + backward)
  for (int c = 0; c < n_chunks; ++c) {
    const int c0 = c * W, wc = I - c0 < W ? I - c0 : W;
    beta_dz_kernel<<<row_grid(n), kRowThreads, 0, st>>>(probs, I, n, wc, c0, I, act, w.T, w.pe, w.pa,
                                                        (float)(1.0 / (double)n), w.dz);
    RECNN_CHECK_LAUNCH("beta_dz_kernel");
    RECNN_PROPAGATE(weight_grad(w.dz, wc, xs, kNoSeg, n, G + l.w + (int64_t)c0 * l.ldw, l.ldw, G + l.b + c0, w.partial,
                                st));
  }
  if (a->optim.kind != RECNN_OPT_EXTERNAL)
    RECNN_PROPAGATE(launch_optimizer(a->optim, a->net, l.count, nullptr, st, w.flags + 1, nullptr, w.flags));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(a->error, w.flags, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return RECNN_OK;
}
