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
//
// Sharded over the item vocabulary (recnn_beta_shard_*), rank r holds rows [lo, hi) of W and b, and the step needs no
// all-reduce: only two all-gathers of per-row statistics.  begin is pass 1 over the local block, writing a record of
// the policy's format (reinforce.cuh: local max m_r, local sum s_r, the target's logit from its owner); rows merges the
// records in rank order (shard_merge_row), turns the block into p and writes a second record with the block's partial
// sums of expm1(p) and p expm1(p); end sums those in rank order into T and U and runs passes (3) and (4) over the
// local block.  Every input of T, U, p_a and the loss is identical on every rank after the exchanges, so those are the
// same bits everywhere; at W = 1 every phase computes exactly what recnn_beta_step does.
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
  Carve c(base);
  w.img = c.take(n * pad4(d.state_dim));
  w.dz = c.take(n * (int64_t)chunk);
  float** rows[7] = {&w.run_max, &w.run_sum, &w.za, &w.T, &w.pe, &w.pa, &w.row_loss};
  for (auto r : rows) *r = c.take(n);
  w.partial = c.take(chunked_partial_floats(chunk, d.num_items, d.state_dim, n));
  w.flags = c.take<unsigned>(8);
  w.bytes = c.bytes();
  return w;
}

static bool beta_dims_ok(const recnn_beta_dims* d) { return d && d->state_dim > 0 && d->num_items > 0; }

// p = exp(z - M) / S in place over the w items of one row (softmax_rows_kernel's normalisation); *s1, *s2 <- the
// CTA's sums of expm1(p) and p expm1(p) over them, valid in every thread.
__device__ __forceinline__ void beta_normalise_row(float* __restrict__ row, int w, float M, float S, float* red,
                                                   float* s1, float* s2) {
  float a = 0.f, b = 0.f;
  for (int j = threadIdx.x; j < w; j += blockDim.x) {
    const float p = expf(row[j] - M) / S;
    row[j] = p;
    const float e = expm1f(p);
    a += e;
    b += p * e;
  }
  *s1 = block_sum(a, red);
  *s2 = block_sum(b, red);
}

// Row r's T = items + sum expm1(p), sum p expm1(p), p_a = exp(z_a - M) / S and loss term log T - p_a, from the sums
// over the whole vocabulary.  An id outside [0, items) sets bit 1 of *err; its row adds no loss.
__device__ __forceinline__ void beta_row_terms(long long r, long long a, int items, float M, float S, float za, float s1,
                                               float s2, float* __restrict__ T_out, float* __restrict__ pe_out,
                                               float* __restrict__ pa_out, float* __restrict__ row_loss,
                                               unsigned* err) {
  const bool ok = a >= 0 && a < items;
  const float pa = ok ? expf(za - M) / S : 0.f;        // == p[a]
  const float T = (float)items + s1;
  T_out[r] = T;
  pe_out[r] = s2;
  pa_out[r] = pa;
  row_loss[r] = ok ? logf(T) - pa : 0.f;
  if (!ok) atomicOr(err, 1u);
}

// Logits -> p in place (the row's max / sum of exp from pass 1), then the row's T, sum p expm1(p), p_a and loss term.
// An id outside [0, items) flags *err; its row adds no loss (and, in beta_dz_kernel, no gradient).  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
beta_rows_kernel(float* __restrict__ P, long long ld, long long n, int items, const long long* __restrict__ action,
                 const float* __restrict__ run_max, const float* __restrict__ run_sum, const float* __restrict__ za,
                 float* __restrict__ T_out, float* __restrict__ pe_out, float* __restrict__ pa_out,
                 float* __restrict__ row_loss, unsigned* err) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float M = run_max[r], S = run_sum[r];
    float s1, s2;
    beta_normalise_row(P + r * ld, items, M, S, red, &s1, &s2);
    if (threadIdx.x == 0)
      beta_row_terms(r, action[r], items, M, S, za[r], s1, s2, T_out, pe_out, pa_out, row_loss, err);
    __syncthreads();
  }
}

// dz[r, j] = (p / n) ((expm1(p) - pe_r) / T_r + pa_r - [lo + c0 + j == a_r]) over the chunk's w items of probs (pitch
// ld: the arena's width), lo the global id of the arena's first item (0 unsharded); zero for a row whose id is outside
// [0, items).  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
beta_dz_kernel(const float* __restrict__ P, long long ld, long long n, int w, int c0, int lo, int items,
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
    const long long al = a - lo - c0;                  // outside [0, w) when the target is in another chunk or rank
    const float t = T[r], e = pe[r], q = pa[r];
    for (int j = threadIdx.x; j < w; j += blockDim.x) {
      const float p = row[j];
      const float g = (expm1f(p) - e) / t + q - (j == al ? 1.f : 0.f);
      out[j] = p * inv_n * g;
    }
  }
}

// Sharded, after exchange 1: the rank-order merge of the gathered records (M, S, z_a into the workspace for the end
// phase), p in place over the rank's block [n, w], and its partial sums s1 = sum expm1(p), s2 = sum p expm1(p) into
// part (the first two planes of the exchange-2 record).  Bit 2 of *err when the headers do not tile the vocabulary.
// At W = 1, M = m_0 and S = s_0: beta_rows_kernel's p.  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
beta_shard_rows_kernel(float* __restrict__ P, long long n, int w, const float* __restrict__ g, ShardPlan p,
                       float* __restrict__ run_max, float* __restrict__ run_sum, float* __restrict__ za,
                       float* __restrict__ part, unsigned* err) {
  __shared__ float red[32];
  if (blockIdx.x == 0 && threadIdx.x == 0 && shard_plan_bad(g, shard_record_floats(n), p, n)) atomicOr(err, 2u);
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float M, S, z, s1, s2;
    shard_merge_row(g, p.world, n, r, M, S, z);
    beta_normalise_row(P + r * w, w, M, S, red, &s1, &s2);
    if (threadIdx.x == 0) {
      run_max[r] = M;
      run_sum[r] = S;
      za[r] = z;
      part[r] = s1;
      part[n + r] = s2;
    }
    __syncthreads();
  }
}

// Sharded, after exchange 2: the vocabulary sums in rank order (at W = 1, 0 + s1_0 = s1_0: the unsharded bits), then
// beta_row_terms.  Bit 2 of *err when the headers do not tile the vocabulary.  One thread per row.
__global__ void beta_shard_terms_kernel(const float* __restrict__ g, long long n, ShardPlan p,
                                        const long long* __restrict__ action, const float* __restrict__ run_max,
                                        const float* __restrict__ run_sum, const float* __restrict__ za,
                                        float* __restrict__ T_out, float* __restrict__ pe_out,
                                        float* __restrict__ pa_out, float* __restrict__ row_loss, unsigned* err) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = shard_record_floats(n);
  if (r == 0 && shard_plan_bad(g, stride, p, n)) atomicOr(err, 2u);
  if (r >= n) return;
  float s1 = 0.f, s2 = 0.f;
  for (int q = 0; q < p.world; ++q) {
    s1 += shard_plane(g, n, 0, q, stride)[r];
    s2 += shard_plane(g, n, 1, q, stride)[r];
  }
  beta_row_terms(r, action[r], p.items, run_max[r], run_sum[r], za[r], s1, s2, T_out, pe_out, pa_out, row_loss, err);
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
  if (!beta_dims_ok(d) || n_rows <= 0 || !chunk_ok(d->num_items, chunk_items)) return 0;
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
    case 10: return offsetof(recnn_beta_args, n_rows_global);
    default: return -1;
  }
}

// The argument checks of the step and of its sharded phases (dims are the arena's: local ones on a shard); *w <- the
// carved workspace.
static int beta_check(const recnn_beta_args* a, BetaWorkspace* w) {
  RECNN_REQUIRE(a != nullptr, "args");
  RECNN_REQUIRE(beta_dims_ok(&a->dims), "dims");
  RECNN_REQUIRE(a->n_rows > 0, "n_rows");
  RECNN_REQUIRE(a->n_rows_global == 0 || a->n_rows_global >= a->n_rows, "n_rows_global is 0 or at least n_rows");
  const int S = a->dims.state_dim, I = a->dims.num_items, W = a->chunk_items;
  RECNN_REQUIRE(chunk_ok(I, W), "chunk_items must be num_items or a positive multiple of 128 below it");
  const int64_t widest = pad4(S) > W ? pad4(S) : W;
  RECNN_REQUIRE(a->n_rows < (1ll << 31) / (widest + 1), "n_rows too large for int32 tile indexing");
  RECNN_REQUIRE(a->state && a->state_ld >= S && a->action, "state / state_ld / action");
  RECNN_REQUIRE(a->probs_out && a->loss && a->error && a->workspace, "probs_out / loss / error / workspace");
  RECNN_REQUIRE(a->net.params && a->net.grads, "net needs params and grads");
  *w = beta_carve(a->dims, a->n_rows, W, a->workspace);
  return check_workspace(w->bytes, a->workspace_bytes);
}

// Pass 1: the state re-pitched into img (when it is not TMA-legal), then the logits of each chunk of W items into z,
// folded into the row's running max / sum of exp (run_max, run_sum) and the target's logit (za; lo: the global id of
// the arena's first item).  z has row pitch ldz: with ldz == num_items it is the step's probs_out and each chunk lands
// in its own columns; otherwise it is a [n, W] scratch that every chunk overwrites (the inference-only log-prob).
static int beta_logits_pass(const recnn_beta_dims& d, const float* P, const float* state, int64_t state_ld,
                            const long long* act, int64_t n, int W, float* img, float* z, int64_t ldz, int lo,
                            float* run_max, float* run_sum, float* za, cudaStream_t st) {
  const int S = d.state_dim, I = d.num_items;
  const BetaLayout l = beta_layout(d);
  Seg xs;
  RECNN_PROPAGATE(repitch_state(S, state, n, img, &xs, st, state_ld));
  for (int c0 = 0; c0 < I; c0 += W) {
    const int wc = I - c0 < W ? I - c0 : W;
    float* zc = ldz == I ? z + c0 : z;
    RECNN_PROPAGATE(linear_out(xs, P + l.w + (int64_t)c0 * l.ldw, l.ldw, P + l.b + c0, wc, n, 0, nullptr, zc, ldz,
                               st));
    logit_stats_kernel<<<row_grid(n), kRowThreads, 0, st>>>(zc, ldz, n, wc, c0, act, lo, run_max, run_sum, za);
    RECNN_CHECK_LAUNCH("logit_stats_kernel");
  }
  return RECNN_OK;
}

// Pass 1 of the step and of its sharded begin: the flags zeroed, then beta_logits_pass into probs_out.
static int beta_step_logits(const recnn_beta_args* a, const BetaWorkspace& w, int lo, float* run_max, float* run_sum,
                            float* za, cudaStream_t st) {
  RECNN_CHECK_CUDA(cudaMemsetAsync(w.flags, 0, 8 * sizeof(unsigned), st));
  return beta_logits_pass(a->dims, a->net.params, a->state, a->state_ld, reinterpret_cast<const long long*>(a->action),
                          a->n_rows, a->chunk_items, w.img, a->probs_out, a->dims.num_items, lo, run_max, run_sum, za,
                          st);
}

// After the row terms: the mean loss, pass 2 (dZ of each chunk, its dW rows and db slice, overwriting the arena:
// zero_grad + backward), the built-in optimizer (skipped on the device when an error bit is set) and the error word.
static int beta_grad_pass(const recnn_beta_args* a, const BetaWorkspace& w, int lo, int items, cudaStream_t st) {
  const int S = a->dims.state_dim, I = a->dims.num_items, W = a->chunk_items;
  const int64_t n = a->n_rows;
  const BetaLayout l = beta_layout(a->dims);
  float* G = a->net.grads;
  const long long* act = reinterpret_cast<const long long*>(a->action);
  const Seg xs = state_seg(S, a->state, a->state_ld, w.img);     // what pass 1 left
  const double n_mean = a->n_rows_global > 0 ? (double)a->n_rows_global : (double)n;   // the cross-entropy's mean
  sum_rows_kernel<<<1, 1024, 0, st>>>(w.row_loss, n, (float)(1.0 / n_mean), a->loss);
  RECNN_CHECK_LAUNCH("sum_rows_kernel");
  for (int c0 = 0; c0 < I; c0 += W) {
    const int wc = I - c0 < W ? I - c0 : W;
    beta_dz_kernel<<<row_grid(n), kRowThreads, 0, st>>>(a->probs_out, I, n, wc, c0, lo, items, act, w.T, w.pe, w.pa,
                                                        (float)(1.0 / n_mean), w.dz);
    RECNN_CHECK_LAUNCH("beta_dz_kernel");
    RECNN_PROPAGATE(weight_grad(w.dz, wc, xs, kNoSeg, n, G + l.w + (int64_t)c0 * l.ldw, l.ldw, G + l.b + c0, w.partial,
                                st));
  }
  if (a->optim.kind != RECNN_OPT_EXTERNAL)
    RECNN_PROPAGATE(launch_optimizer(a->optim, a->net, l.count, nullptr, st, w.flags + 1, nullptr, w.flags));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(a->error, w.flags, sizeof(int32_t), cudaMemcpyDeviceToDevice, st));
  return RECNN_OK;
}

// Beta.forward(state, action) of the notebook's cell 3: forward, CrossEntropyLoss on the probabilities, zero_grad +
// backward, optim.step(); probs_out holds the pre-step probabilities.
extern "C" int recnn_beta_step(const recnn_beta_args* a, void* stream) {
  BetaWorkspace w;
  RECNN_PROPAGATE(beta_check(a, &w));
  const int I = a->dims.num_items;
  const int64_t n = a->n_rows;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_PROPAGATE(beta_step_logits(a, w, 0, w.run_max, w.run_sum, w.za, st));
  beta_rows_kernel<<<row_grid(n), kRowThreads, 0, st>>>(a->probs_out, I, n, I, reinterpret_cast<const long long*>(
                                                            a->action), w.run_max, w.run_sum, w.za, w.T, w.pe, w.pa,
                                                        w.row_loss, w.flags);
  RECNN_CHECK_LAUNCH("beta_rows_kernel");
  return beta_grad_pass(a, w, 0, I, st);
}

// ---- beta sharded over the item vocabulary: the three phases around the two all-gathers (see the header) ----------
static int beta_shard_check(const recnn_beta_args* a, const recnn_vocab_shard* v, BetaWorkspace* w, ShardPlan* p) {
  RECNN_PROPAGATE(beta_check(a, w));
  return shard_plan(a->dims.num_items, v, p);
}

extern "C" int recnn_beta_shard_begin(const recnn_beta_args* a, const recnn_vocab_shard* v, float* record,
                                      void* stream) {
  BetaWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(beta_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(record != nullptr, "record");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = a->n_rows;
  RECNN_PROPAGATE(shard_record_init(p, record, n, st));
  return beta_step_logits(a, w, p.lo, shard_plane(record, n, 0), shard_plane(record, n, 1), shard_plane(record, n, 2),
                          st);
}

extern "C" int recnn_beta_shard_rows(const recnn_beta_args* a, const recnn_vocab_shard* v, const float* gathered,
                                     float* record, void* stream) {
  BetaWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(beta_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(gathered && record, "gathered / record");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = a->n_rows;
  RECNN_PROPAGATE(shard_record_init(p, record, n, st));
  beta_shard_rows_kernel<<<row_grid(n), kRowThreads, 0, st>>>(a->probs_out, n, a->dims.num_items, gathered, p,
                                                              w.run_max, w.run_sum, w.za, shard_plane(record, n, 0),
                                                              w.flags);
  RECNN_CHECK_LAUNCH("beta_shard_rows_kernel");
  return RECNN_OK;
}

extern "C" int recnn_beta_shard_end(const recnn_beta_args* a, const recnn_vocab_shard* v, const float* gathered,
                                    void* stream) {
  BetaWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(beta_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(gathered != nullptr, "gathered");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = a->n_rows;
  beta_shard_terms_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(
      gathered, n, p, reinterpret_cast<const long long*>(a->action), w.run_max, w.run_sum, w.za, w.T, w.pe, w.pa,
      w.row_loss, w.flags);
  RECNN_CHECK_LAUNCH("beta_shard_terms_kernel");
  return beta_grad_pass(a, w, p.lo, p.items, st);
}

// ---- log beta(a | s) of given items, inference only: pass 1 into a [n, chunk] scratch, then target_log_prob.  No
// gradient arena, optimizer state or probs_out is read or written.
struct BetaLogProbWorkspace {
  float *img, *z, *run_max, *run_sum, *za;       // [n, pad4(S)], [n, chunk], three [n]
  int64_t bytes;
};
static BetaLogProbWorkspace beta_log_prob_carve(const recnn_beta_dims& d, int64_t n, int chunk, void* base) {
  BetaLogProbWorkspace w;
  Carve c(base);
  w.img = c.take(n * pad4(d.state_dim));
  w.z = c.take(n * (int64_t)chunk);
  w.run_max = c.take(n);
  w.run_sum = c.take(n);
  w.za = c.take(n);
  w.bytes = c.bytes();
  return w;
}

extern "C" int64_t recnn_beta_log_prob_workspace_bytes(const recnn_beta_dims* d, int64_t n_rows, int32_t chunk_items) {
  if (!beta_dims_ok(d) || n_rows <= 0 || !chunk_ok(d->num_items, chunk_items)) return 0;
  return beta_log_prob_carve(*d, n_rows, chunk_items, nullptr).bytes;
}

// the checks of both log-prob entry points (d: the arena's dims, local on a shard); *w <- the carved workspace
static int beta_log_prob_check(const recnn_beta_dims* d, const float* params, const float* state, int64_t state_ld,
                               const int64_t* action, int64_t n_rows, int32_t chunk_items, void* workspace,
                               int64_t workspace_bytes, BetaLogProbWorkspace* w) {
  RECNN_REQUIRE(beta_dims_ok(d) && params && state && action && workspace, "null pointer / dims");
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(state_ld >= d->state_dim, "state_ld");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  const int64_t widest = pad4(d->state_dim) > chunk_items ? pad4(d->state_dim) : chunk_items;
  RECNN_REQUIRE(n_rows < (1ll << 31) / (widest + 1), "n_rows too large for int32 tile indexing");
  *w = beta_log_prob_carve(*d, n_rows, chunk_items, workspace);
  return check_workspace(w->bytes, workspace_bytes);
}

extern "C" int recnn_beta_log_prob(const recnn_beta_dims* d, const float* params, const float* state, int64_t state_ld,
                                   const int64_t* action, int64_t n_rows, int32_t chunk_items, float* log_prob_out,
                                   int32_t* error_flag, void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(log_prob_out && error_flag, "null pointer");
  BetaLogProbWorkspace w;
  RECNN_PROPAGATE(beta_log_prob_check(d, params, state, state_ld, action, n_rows, chunk_items, workspace,
                                      workspace_bytes, &w));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* act = reinterpret_cast<const long long*>(action);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(rank_target_check(act, n_rows, d->num_items, error_flag, st));
  RECNN_PROPAGATE(beta_logits_pass(*d, params, state, state_ld, act, n_rows, chunk_items, w.img, w.z, chunk_items, 0,
                                   w.run_max, w.run_sum, w.za, st));
  log_prob_finish_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(w.za, w.run_max, w.run_sum, act, n_rows,
                                                                          d->num_items, log_prob_out);
  RECNN_CHECK_LAUNCH("log_prob_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_beta_shard_log_prob_stats(const recnn_beta_dims* d, const recnn_vocab_shard* v,
                                               const float* params, const float* state, int64_t state_ld,
                                               const int64_t* action, int64_t n_rows, int32_t chunk_items,
                                               float* record, void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(record, "null pointer");
  BetaLogProbWorkspace w;
  RECNN_PROPAGATE(beta_log_prob_check(d, params, state, state_ld, action, n_rows, chunk_items, workspace,
                                      workspace_bytes, &w));
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_PROPAGATE(shard_record_init(p, record, n_rows, st));
  return beta_logits_pass(*d, params, state, state_ld, reinterpret_cast<const long long*>(action), n_rows, chunk_items,
                          w.img, w.z, chunk_items, p.lo, shard_plane(record, n_rows, 0),
                          shard_plane(record, n_rows, 1), shard_plane(record, n_rows, 2), st);
}
