// REINFORCE with (Top-K) off-policy correction: the policy side (SURVEY 8f-2).
//
// Restates, for one GPU, recnn/nn/models.py:76-184 (DiscreteActor: forward, Categorical sampling, log-probs, importance
// correction, lambda_K) and recnn/nn/update/reinforce.py:10-65 (ChooseREINFORCE: the three policy losses and their
// backward).  Included at the end of step.cu: it is built from the same four contraction helpers as the DDPG / TD3 step
// (hidden_layer, linear_out, backprop_hidden, weight_grad -> wgmma 3xTF32 GEMMs) plus a few row kernels.
//
// What is different from the reference's formulation:
//   * the reference keeps one autograd graph per env step (saved_log_probs, models.py:110,156,183) and back-propagates
//     through all of them at the policy update.  The policy's weights do not change between two policy updates, so the
//     sum of those backward passes is ONE backward pass over the concatenation of the saved batches: the caller keeps
//     (state, sampled action, beta log-prob, step index) per row -- 5 KB/row instead of the [N, num_items] probability
//     matrices -- and recnn_reinforce_policy_grad_chunked recomputes the forward on the R = T*N saved rows.
//   * d loss / d logits has a closed form (softmax + log + the scalar weight of the row), so it needs only per-row
//     statistics of the logits: max, sum of exp and the drawn action's logit.  The [R, num_items] logits are never
//     stored whole: the items are visited in chunks, twice (FlashAttention-style recomputation) -- pass 1 folds each
//     chunk's logits into the row statistics, pass 2 recomputes them, turns them into d logits in place and feeds the
//     dW2 rows of the chunk and an accumulating dh GEMM.  Scratch holds one [R, chunk] block; with one chunk the
//     logits are computed once.
//   * the per-row statistics are "exchange 1" of the vocabulary-sharded formulation
//     (oracle/reinforce_oracle.py: sharded_policy_grad).
//   * the normalised discounted returns (reinforce.py:44-52) are T scalars: host arithmetic in the caller.
//
// Per saved row n with sampled action a, p = clamp(pi[a], eps, 1-eps), lp = log p, R = return of the row's step:
//   basic   (reinforce.py:16-22)   L = -lp R                                 dL/dlp = -R
//   corr    (reinforce.py:24-33)   L = (p/b)(-lp) R     b = exp(beta lp)     dL/dlp = -R (p/b)(lp + 1)
//   top-K   (reinforce.py:35-44)   L = lam (p/b)(-lp) R, lam = K(1-p)^(K-1)  dL/dlp = -R/b [lam p (lp+1) - K(K-1)(1-p)^(K-2) p^2 lp]
// and d lp / d logits[j] = [j == a] - pi[j]   (corr and lam are NOT detached in the reference: models.py:150,168-171).
#pragma once

namespace recnn {

struct DiscreteLayout {
  int ld1, ld2;                      // row pitches of w1 [H, S] and w2 [num_items, H]
  int64_t w1, b1, w2, b2, count;
};
static inline DiscreteLayout discrete_layout(const recnn_discrete_dims& d) {
  DiscreteLayout l;
  l.ld1 = pad4(d.state_dim);
  l.ld2 = pad4(d.hidden);
  l.w1 = 0;
  l.b1 = l.w1 + (int64_t)d.hidden * l.ld1;
  l.w2 = l.b1 + pad4(d.hidden);
  l.b2 = l.w2 + (int64_t)d.num_items * l.ld2;
  l.count = l.b2 + pad4(d.num_items);
  return l;
}

constexpr int kRowThreads = 256;
constexpr float kProbEps = 1.1920928955078125e-07f;     // torch.finfo(float32).eps: Categorical clamps probs to [eps, 1-eps]

__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float t = (threadIdx.x < nw) ? red[threadIdx.x] : -INFINITY;
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
  }
  if (threadIdx.x == 0) red[0] = t;
  __syncthreads();
  t = red[0];
  return t;
}

// z[r, :] <- softmax(z[r, :])      (models.py:99; F.softmax without dim on a 2-d input is dim=1)
// one CTA per row; the row is read twice (online max / sum, then the normalised write)
__global__ void __launch_bounds__(kRowThreads) softmax_rows_kernel(float* __restrict__ z, long long ld, long long n, int items) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float* row = z + r * ld;
    float m = -INFINITY, s = 0.f;
    for (int j = threadIdx.x; j < items; j += blockDim.x) {
      const float x = row[j];
      if (x > m) {
        s = s * __expf(m - x) + 1.f;      // m == -inf: s == 0, exp(-inf) == 0
        m = x;
      } else {
        s += __expf(x - m);
      }
    }
    const float M = block_max(m, red);
    s = (m == -INFINITY) ? 0.f : s * __expf(m - M);
    const float S = block_sum(s, red);
    for (int j = threadIdx.x; j < items; j += blockDim.x) row[j] = expf(row[j] - M) / S;
    __syncthreads();
  }
}

__device__ __forceinline__ float clamped_log_prob(float p) {
  return logf(fminf(fmaxf(p, kProbEps), 1.f - kProbEps));
}

// Categorical(probs).sample() and .log_prob(sample)   (models.py:107-110, 127-143).  torch normalises the probabilities
// by their row sum and clamps them to [eps, 1-eps] before the log (torch/distributions/categorical.py, utils.py).
// Sampling is by inverse CDF: the first j with cumsum(probs)[j] > u * sum(probs); u from `uniforms` (replayable) or from
// Philox keyed by (seed, draw, row).  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
categorical_sample_kernel(const float* __restrict__ probs, long long ld, long long n, int items,
                          const float* __restrict__ uniforms, unsigned long long seed, long long draw,
                          long long* __restrict__ action, float* __restrict__ logp) {
  __shared__ float red[32];
  __shared__ float warp_tot[kRowThreads / 32];
  __shared__ int found;
  __shared__ float run;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float* row = probs + r * ld;
    float t = 0.f;
    for (int j = threadIdx.x; j < items; j += blockDim.x) t += row[j];
    const float total = block_sum(t, red);
    float u;
    if (uniforms) {
      u = uniforms[r];
    } else {
      Philox ph(seed);
      const uint4 q = ph((unsigned long long)r, ((unsigned long long)draw << 8) | 0x5au);
      u = (float)(q.x >> 8) * (1.0f / 16777216.0f);          // [0, 1)
    }
    const float target = u * total;
    if (threadIdx.x == 0) {
      found = items;
      run = 0.f;
    }
    __syncthreads();
    for (int base = 0; base < items; base += blockDim.x) {
      const int j = base + threadIdx.x;
      const float p = j < items ? row[j] : 0.f;
      float incl = p;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
      }
      if (lane == 31) warp_tot[warp] = incl;
      __syncthreads();
      float before = run;
      for (int w = 0; w < warp; ++w) before += warp_tot[w];
      const float c = before + incl;
      if (j < items && p > 0.f && c > target) atomicMin(&found, j);
      __syncthreads();
      if (found < items) break;
      if (threadIdx.x == blockDim.x - 1) run = c;
      __syncthreads();
    }
    if (threadIdx.x == 0) {
      int a = found;
      if (a >= items) {                 // u * total rounded past the last partial sum: the last possible outcome
        a = items - 1;
        while (a > 0 && !(row[a] > 0.f)) --a;
      }
      action[r] = a;
      logp[r] = clamped_log_prob(row[a] / total);
    }
    __syncthreads();
  }
}

// .log_prob(action) of given actions (models.py:142-143 with action_source {pi: beta}: the policy's log-prob of the
// behaviour policy's sample).  One warp per row.
__global__ void categorical_log_prob_kernel(const float* __restrict__ probs, long long ld, long long n, int items,
                                            const long long* __restrict__ action, float* __restrict__ logp, int* oob) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= n) return;
  const int lane = threadIdx.x & 31;
  const float* row = probs + r * ld;
  float t = 0.f;
  for (int j = lane; j < items; j += 32) t += row[j];
  t = warp_sum(t);
  if (lane == 0) {
    const long long a = action[r];
    if (a < 0 || a >= items) {
      if (oob) *oob = 1;
      logp[r] = 0.f;
    } else {
      logp[r] = clamped_log_prob(row[a] / t);
    }
  }
}

// The policy gradient walks the items in chunks [c0, c0 + w) of a [rows, w] logits buffer (row pitch w): the full
// [rows, num_items] matrix is never stored.  Pass 1 folds each chunk into per-row running statistics; pass 2 recomputes
// each chunk's logits and turns them into d loss / d logits.  With one chunk this is the plain softmax backward.

// Pass 1: (run_max, run_sum) <- the online max / sum of exp over the logits seen so far (chunk c0 == 0 starts them);
// za[r] <- z[r, a_r] when the row's action lies in this chunk.  z: the chunk's [n, w] logits with row pitch ld.
// One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
logit_stats_kernel(const float* __restrict__ z, long long ld, long long n, int w, int c0,
                   const long long* __restrict__ action, float* __restrict__ run_max, float* __restrict__ run_sum,
                   float* __restrict__ za) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float* row = z + r * ld;
    float m = -INFINITY, s = 0.f;
    for (int j = threadIdx.x; j < w; j += blockDim.x) {     // the same reduction as softmax_rows_kernel
      const float x = row[j];
      if (x > m) {
        s = s * __expf(m - x) + 1.f;
        m = x;
      } else {
        s += __expf(x - m);
      }
    }
    const float M = block_max(m, red);
    s = (m == -INFINITY) ? 0.f : s * __expf(m - M);
    const float S = block_sum(s, red);
    if (threadIdx.x == 0) {
      if (c0 == 0) {
        run_max[r] = M;
        run_sum[r] = S;
      } else {
        const float M0 = run_max[r], Mn = fmaxf(M0, M);
        run_sum[r] = run_sum[r] * expf(M0 - Mn) + S * expf(M - Mn);
        run_max[r] = Mn;
      }
      const long long a = action[r];
      if (a >= c0 && a < (long long)c0 + w) za[r] = row[a - c0];
    }
    __syncthreads();
  }
}

// The row's loss term L and g = dL / d log pi(a), from pa = pi(a) (see the table at the top of this file).
__device__ __forceinline__ float reinforce_row_weight(float pa, float R, float beta_lp, int method, int K, float* loss) {
  const float p = fminf(fmaxf(pa, kProbEps), 1.f - kProbEps);
  const bool inside = pa > kProbEps && pa < 1.f - kProbEps;       // the clamp has zero slope outside
  const float lp = logf(p);
  float g, L;
  if (method == RECNN_REINFORCE_BASIC) {
    L = -lp * R;
    g = -R;
  } else {
    const float c = p / expf(beta_lp);
    if (method == RECNN_REINFORCE_CORRECTED) {
      L = c * -lp * R;
      g = -R * c * (lp + 1.f);
    } else {
      const float q = 1.f - p, Kf = (float)K;
      const float lam = Kf * powf(q, Kf - 1.f);
      const float dlam = K > 1 ? -Kf * (Kf - 1.f) * powf(q, Kf - 2.f) * p : 0.f;      // d lam / d lp
      L = lam * c * -lp * R;
      g = -R * c * (dlam * lp + lam * (lp + 1.f));
    }
  }
  *loss = L;
  return inside ? g : 0.f;
}

// After pass 1: g[r] and row_loss[r] from pi(a) = exp(z[a] - M) / S.  An action id outside [0, items) is flagged and
// contributes nothing (g = 0, L = 0).  One thread per row.
__global__ void reinforce_row_weights_kernel(long long n, int items, const long long* __restrict__ action,
                                             const float* __restrict__ run_max, const float* __restrict__ run_sum,
                                             const float* __restrict__ za, const float* __restrict__ beta_logp,
                                             const float* __restrict__ ret, int method, int K, float* __restrict__ g,
                                             float* __restrict__ row_loss, int* oob) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const long long a = action[r];
  float gr = 0.f, L = 0.f;
  if (a < 0 || a >= items) {
    if (oob) *oob = 1;
  } else {
    const float pa = expf(za[r] - run_max[r]) / run_sum[r];
    gr = reinforce_row_weight(pa, ret[r], beta_logp ? beta_logp[r] : 0.f, method, K, &L);
  }
  g[r] = gr;
  row_loss[r] = L;
}

// Pass 2: logits chunk -> d loss / d logits in place: dz[r, j] = g_r ([c0 + j == a_r] - exp(z - M_r) / S_r).
__global__ void __launch_bounds__(kRowThreads)
reinforce_dlogits_kernel(float* __restrict__ z, long long n, int w, int c0, const long long* __restrict__ action,
                         const float* __restrict__ run_max, const float* __restrict__ run_sum, const float* __restrict__ g) {
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float* row = z + r * w;
    const long long a = action[r] - c0;               // outside [0, w) when the action is in another chunk
    const float M = run_max[r], S = run_sum[r], gr = g[r];
    for (int j = threadIdx.x; j < w; j += blockDim.x) row[j] = gr * ((j == a ? 1.f : 0.f) - expf(row[j] - M) / S);
  }
}

// out[0] = scale * (sum of v[0..n) in a fixed order)  (one CTA)
__global__ void __launch_bounds__(1024) sum_rows_kernel(const float* __restrict__ v, long long n, float scale,
                                                        float* __restrict__ out) {
  __shared__ float red[32];
  float t = 0.f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) t += v[i];
  t = block_sum(t, red);
  if (threadIdx.x == 0) out[0] = t * scale;
}

static int row_grid(int64_t n) { return (int)(n < (int64_t)kNumSMs * 8 ? n : (int64_t)kNumSMs * 8); }

static bool chunk_ok(const recnn_discrete_dims& d, int64_t chunk) {
  return chunk == d.num_items || (chunk > 0 && chunk % 128 == 0 && chunk < d.num_items);
}

// split-K partial space of a weight gradient dW[C, K] over `rows` (either back end); *one_split: both use one split
static int64_t dw_partial_floats(int C, int K, int64_t rows, bool* one_split) {
  int64_t best = 0;
  bool one = true;
  for (int tcp = 0; tcp < 2; ++tcp) {
    const int s = dw_splits(C, K, rows, tcp != 0);
    const int64_t f = (int64_t)s * C * (K + 1);
    if (f > best) best = f;
    one = one && s == 1;
  }
  if (one_split) *one_split = one;
  return best;
}

// ... of a weight gradient [num_items, K] computed in row blocks of `chunk` items, the last one possibly narrower.
// dw_splits sees a block's width only through ceil(width / 128) and the partials grow with the width at a fixed split
// count, so the widest width of every 128-band bounds that band; once both back ends use one split, the partials only
// grow with the width.  Independent of num_items when chunk < num_items.
static int64_t chunked_partial_floats(int chunk, int num_items, int K, int64_t rows) {
  int64_t best = 0;
  if (chunk != num_items) {
    bool one = false;
    for (int64_t c = 128; c < chunk && !one; c += 128) {
      const int64_t f = dw_partial_floats((int)c, K, rows, &one);
      if (f > best) best = f;
    }
  }
  const int64_t f = dw_partial_floats(chunk, K, rows, nullptr);
  return f > best ? f : best;
}

// the two weight gradients of the policy, dW2 in row blocks of `chunk` items
static int64_t reinforce_partial_floats(const recnn_discrete_dims& d, int64_t rows, int chunk) {
  const int64_t f1 = dw_partial_floats(d.hidden, d.state_dim, rows, nullptr);
  const int64_t f2 = chunked_partial_floats(chunk, d.num_items, d.hidden, rows);
  return f1 > f2 ? f1 : f2;
}

struct DiscreteScratch {
  float *img, *h, *z, *dh, *row_loss, *run_max, *run_sum, *za, *g, *partial;
  int* flags;
  int64_t floats;
};
// chunk == 0: the forward only.  Otherwise the policy gradient over item chunks of `chunk` (z is [n, chunk]).
static DiscreteScratch discrete_carve(const recnn_discrete_dims& d, int64_t n, int chunk, float* base) {
  DiscreteScratch s;
  int64_t off = 0;
  auto take = [&](int64_t floats) {
    float* r = base ? base + off : nullptr;
    off += round_up(floats, 64);
    return r;
  };
  s.img = take(n * pad4(d.state_dim));
  s.h = take(n * d.hidden);
  s.flags = reinterpret_cast<int*>(take(4));
  s.z = s.dh = s.row_loss = s.run_max = s.run_sum = s.za = s.g = s.partial = nullptr;
  if (chunk > 0) {
    s.z = take(n * (int64_t)chunk);
    s.dh = take(n * d.hidden);
    s.row_loss = take(n);
    s.run_max = take(n);
    s.run_sum = take(n);
    s.za = take(n);
    s.g = take(n);
    s.partial = take(reinforce_partial_floats(d, n, chunk));
  }
  s.floats = off + 64;
  return s;
}
static float* align_floats(float* p) {      // 256-byte aligned start inside the caller's scratch
  return reinterpret_cast<float*>(round_up(reinterpret_cast<int64_t>(p), 256));
}

// h = relu(W1 s + b1) into s.h, kept for the backward; *xs_out = the re-pitched state
static int discrete_hidden(const recnn_discrete_dims& d, const float* params, const float* state, int64_t n,
                           const DiscreteScratch& s, cudaStream_t st, Seg* xs_out) {
  const DiscreteLayout l = discrete_layout(d);
  recnn_dims dd;
  memset(&dd, 0, sizeof(dd));
  dd.state_dim = d.state_dim; dd.hidden = d.hidden; dd.action_dim = d.num_items;
  Seg xs;
  RECNN_PROPAGATE(repitch_state(dd, state, n, s.img, &xs, st));
  if (xs_out) *xs_out = xs;
  Rng rng = {nullptr, 0, nullptr};
  return hidden_layer(xs, kNoSeg, params + l.w1, l.ld1, params + l.b1, d.hidden, n, false, nullptr, rng, 0, s.h, st);
}

// logits of items [c0, c0 + w) = W2[c0:c0+w] h + b2[c0:c0+w] into z (row pitch w).  W2's row pitch is pad4(H), so every
// chunk of W2 starts on a 16-byte boundary.
static int discrete_logits(const recnn_discrete_dims& d, const float* params, int64_t n, const DiscreteScratch& s,
                           int c0, int w, float* z, cudaStream_t st) {
  const DiscreteLayout l = discrete_layout(d);
  const Seg sh = {s.h, d.hidden, d.hidden, 0};
  return linear_out(sh, params + l.w2 + (int64_t)c0 * l.ld2, l.ld2, params + l.b2 + c0, w, n, 0, nullptr, z, w, st);
}

}  // namespace recnn

using namespace recnn;

static bool discrete_dims_ok(const recnn_discrete_dims* d) {
  return d && d->state_dim > 0 && d->hidden > 0 && d->num_items > 0;
}

extern "C" int recnn_discrete_layout(const recnn_discrete_dims* d, int64_t* out) {
  RECNN_REQUIRE(discrete_dims_ok(d) && out, "dims / out");
  const DiscreteLayout l = discrete_layout(*d);
  out[0] = l.w1; out[1] = l.b1; out[2] = l.w2; out[3] = l.b2; out[4] = l.ld1; out[5] = l.ld2; out[6] = l.count;
  return RECNN_OK;
}

extern "C" int64_t recnn_discrete_scratch_floats(const recnn_discrete_dims* d, int64_t n_rows, int32_t backward) {
  if (!discrete_dims_ok(d) || n_rows <= 0) return 0;
  return discrete_carve(*d, n_rows, backward != 0 ? d->num_items : 0, nullptr).floats;
}

extern "C" int64_t recnn_reinforce_scratch_floats(const recnn_discrete_dims* d, int64_t n_rows, int32_t chunk_items) {
  if (!discrete_dims_ok(d) || n_rows <= 0 || !chunk_ok(*d, chunk_items)) return 0;
  return discrete_carve(*d, n_rows, chunk_items, nullptr).floats;
}

extern "C" int recnn_discrete_forward(const recnn_discrete_dims* d, const float* params, const float* state,
                                      int64_t n_rows, float* probs_out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && probs_out && scratch, "null pointer / dims");
  if (n_rows <= 0) return RECNN_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const DiscreteScratch s = discrete_carve(*d, n_rows, 0, align_floats(scratch));
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, s, st, nullptr));
  RECNN_PROPAGATE(discrete_logits(*d, params, n_rows, s, 0, d->num_items, probs_out, st));
  softmax_rows_kernel<<<row_grid(n_rows), kRowThreads, 0, st>>>(probs_out, d->num_items, n_rows, d->num_items);
  RECNN_CHECK_LAUNCH("softmax_rows_kernel");
  return RECNN_OK;
}

extern "C" int recnn_categorical_sample(const float* probs, int64_t n_rows, int32_t num_items, int64_t ld,
                                        const float* uniforms, uint64_t seed, int64_t draw, int64_t* action_out,
                                        float* log_prob_out, void* stream) {
  RECNN_REQUIRE(probs && action_out && log_prob_out, "null pointer");
  RECNN_REQUIRE(num_items > 0 && ld >= num_items, "num_items / ld");
  if (n_rows <= 0) return RECNN_OK;
  categorical_sample_kernel<<<row_grid(n_rows), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, ld, n_rows, num_items, uniforms, seed, draw, reinterpret_cast<long long*>(action_out), log_prob_out);
  RECNN_CHECK_LAUNCH("categorical_sample_kernel");
  return RECNN_OK;
}

extern "C" int recnn_categorical_log_prob(const float* probs, int64_t n_rows, int32_t num_items, int64_t ld,
                                          const int64_t* action, float* log_prob_out, int32_t* oob_flag, void* stream) {
  RECNN_REQUIRE(probs && action && log_prob_out, "null pointer");
  RECNN_REQUIRE(num_items > 0 && ld >= num_items, "num_items / ld");
  if (n_rows <= 0) return RECNN_OK;
  const int warps = 8;
  categorical_log_prob_kernel<<<(unsigned)ceil_div(n_rows, warps), warps * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, ld, n_rows, num_items, reinterpret_cast<const long long*>(action), log_prob_out, oob_flag);
  RECNN_CHECK_LAUNCH("categorical_log_prob_kernel");
  return RECNN_OK;
}

// out[0] = policy loss, out[1] = 1.0 if an action id was outside [0, num_items) (that row contributes nothing)
extern "C" int recnn_reinforce_policy_grad_chunked(const recnn_discrete_dims* d, const float* params, float* grads,
                                                   const float* state, const int64_t* action, const float* beta_log_prob,
                                                   const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                                   int32_t chunk_items, float* out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && grads && state && action && returns && out && scratch,
                "null pointer / dims");
  RECNN_REQUIRE(method == RECNN_REINFORCE_BASIC || method == RECNN_REINFORCE_CORRECTED || method == RECNN_REINFORCE_TOPK,
                "unknown REINFORCE method");
  RECNN_REQUIRE(method == RECNN_REINFORCE_BASIC || beta_log_prob, "the corrected losses need the behaviour policy's log-probs");
  RECNN_REQUIRE(method != RECNN_REINFORCE_TOPK || top_k >= 1, "K >= 1");
  RECNN_REQUIRE(n_rows > 0, "no saved rows: select_action was never called since the last update");
  RECNN_REQUIRE(chunk_ok(*d, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const DiscreteLayout l = discrete_layout(*d);
  const int H = d->hidden, I = d->num_items, W = chunk_items;
  const int n_chunks = (int)ceil_div(I, W);
  const long long* act = reinterpret_cast<const long long*>(action);
  const DiscreteScratch s = discrete_carve(*d, n_rows, W, align_floats(scratch));
  RECNN_CHECK_CUDA(cudaMemsetAsync(s.flags, 0, 4 * sizeof(int), st));
  Seg xs;
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, s, st, &xs));
  // pass 1: per-row max / sum of exp over all logits, and the drawn action's logit
  for (int c = 0; c < n_chunks; ++c) {
    const int c0 = c * W, w = I - c0 < W ? I - c0 : W;
    RECNN_PROPAGATE(discrete_logits(*d, params, n_rows, s, c0, w, s.z, st));
    logit_stats_kernel<<<row_grid(n_rows), kRowThreads, 0, st>>>(s.z, w, n_rows, w, c0, act, s.run_max, s.run_sum,
                                                                  s.za);
    RECNN_CHECK_LAUNCH("logit_stats_kernel");
  }
  reinforce_row_weights_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(
      n_rows, I, act, s.run_max, s.run_sum, s.za, beta_log_prob, returns, method, top_k, s.g, s.row_loss, s.flags);
  RECNN_CHECK_LAUNCH("reinforce_row_weights_kernel");
  sum_rows_kernel<<<1, 1024, 0, st>>>(s.row_loss, n_rows, 1.f, out);
  RECNN_CHECK_LAUNCH("sum_rows_kernel");
  // pass 2, last chunk first (its logits are still in the buffer): dz = d loss / d logits of the chunk;
  // dW2[c0:c0+w] = dz^T h, db2[c0:c0+w] = colsum dz; dh (+)= dz W2[c0:c0+w], gated by [h > 0] after the last term
  const Seg sh = {s.h, H, H, 0};
  for (int c = n_chunks - 1; c >= 0; --c) {
    const int c0 = c * W, w = I - c0 < W ? I - c0 : W;
    if (c != n_chunks - 1) RECNN_PROPAGATE(discrete_logits(*d, params, n_rows, s, c0, w, s.z, st));
    reinforce_dlogits_kernel<<<row_grid(n_rows), kRowThreads, 0, st>>>(s.z, n_rows, w, c0, act, s.run_max, s.run_sum, s.g);
    RECNN_CHECK_LAUNCH("reinforce_dlogits_kernel");
    const int64_t w2 = l.w2 + (int64_t)c0 * l.ld2;
    RECNN_PROPAGATE(weight_grad(s.z, w, sh, kNoSeg, n_rows, grads + w2, l.ld2, grads + l.b2 + c0, s.partial, st));
    RECNN_PROPAGATE(backprop_hidden(s.z, w, params + w2, l.ld2, H, 0, H, n_rows, c == 0 ? s.h : nullptr, 1.f, s.dh, st,
                                    c != n_chunks - 1));
  }
  // dW1 = dh^T s, db1 = colsum dh
  RECNN_PROPAGATE(weight_grad(s.dh, H, xs, kNoSeg, n_rows, grads + l.w1, l.ld1, grads + l.b1, s.partial, st));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(out + 1, s.flags, sizeof(int), cudaMemcpyDeviceToDevice, st));
  return RECNN_OK;
}

extern "C" int recnn_reinforce_policy_grad(const recnn_discrete_dims* d, const float* params, float* grads,
                                           const float* state, const int64_t* action, const float* beta_log_prob,
                                           const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                           float* out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d), "null pointer / dims");
  return recnn_reinforce_policy_grad_chunked(d, params, grads, state, action, beta_log_prob, returns, n_rows, method,
                                             top_k, d->num_items, out, scratch, stream);
}
