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
      } else if (x != -INFINITY) {        // a -inf logit adds exp(-inf) = 0, and NaN = exp(-inf - -inf) while m is -inf
        s += __expf(x - m);
      }
    }
    const float M = block_max(m, red);
    s = (m == -INFINITY) ? s : s * __expf(m - M);   // no finite logit: s is 0, or NaN after a NaN logit (kept)
    const float S = block_sum(s, red);
    for (int j = threadIdx.x; j < items; j += blockDim.x) row[j] = expf(row[j] - M) / S;
    __syncthreads();
  }
}

__device__ __forceinline__ float clamped_log_prob(float p) {
  return logf(fminf(fmaxf(p, kProbEps), 1.f - kProbEps));
}

// The uniform of row r's draw: uniforms[r] (replayable) or Philox keyed by (seed, draw, row), in [0, 1).
__device__ __forceinline__ float draw_uniform(const float* uniforms, unsigned long long seed, long long draw, long long r) {
  if (uniforms) return uniforms[r];
  Philox ph(seed);
  const uint4 q = ph((unsigned long long)r, ((unsigned long long)draw << 8) | 0x5au);
  return (float)(q.x >> 8) * (1.0f / 16777216.0f);
}

struct CdfShared {
  float warp_tot[kRowThreads / 32];
  int found;
  float run;
};
// Inverse CDF inside one row, by the whole CTA: the first j with cumsum(row)[j] > target and row[j] > 0; when target
// rounded past the last partial sum, the last positive entry.  The result is valid in thread 0.
__device__ int inverse_cdf_row(const float* row, int items, float target, CdfShared& sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    sh.found = items;
    sh.run = 0.f;
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
    if (lane == 31) sh.warp_tot[warp] = incl;
    __syncthreads();
    float before = sh.run;
    for (int w = 0; w < warp; ++w) before += sh.warp_tot[w];
    const float c = before + incl;
    if (j < items && p > 0.f && c > target) atomicMin(&sh.found, j);
    __syncthreads();
    if (sh.found < items) break;
    if (threadIdx.x == blockDim.x - 1) sh.run = c;
    __syncthreads();
  }
  int a = sh.found;
  if (threadIdx.x == 0 && a >= items) {
    a = items - 1;
    while (a > 0 && !(row[a] > 0.f)) --a;
  }
  return a;
}

// Categorical(probs).sample() and .log_prob(sample)   (models.py:107-110, 127-143).  torch normalises the probabilities
// by their row sum and clamps them to [eps, 1-eps] before the log (torch/distributions/categorical.py, utils.py).
// Sampling is by inverse CDF: the first j with cumsum(probs)[j] > u * sum(probs); u from draw_uniform.  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
categorical_sample_kernel(const float* __restrict__ probs, long long ld, long long n, int items,
                          const float* __restrict__ uniforms, unsigned long long seed, long long draw,
                          long long* __restrict__ action, float* __restrict__ logp, long long row_offset = 0) {
  __shared__ float red[32];
  __shared__ CdfShared sh;
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float* row = probs + r * ld;
    float t = 0.f;
    for (int j = threadIdx.x; j < items; j += blockDim.x) t += row[j];
    const float total = block_sum(t, red);
    const float u = uniforms ? uniforms[r] : draw_uniform(nullptr, seed, draw, row_offset + r);
    const int a = inverse_cdf_row(row, items, u * total, sh);
    if (threadIdx.x == 0) {
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
// za[r] <- z[r, a_r - a_off] when that column lies in this chunk (a_off: the first item id of the arena's linear2 rows,
// 0 unless the vocabulary is sharded; action may be NULL).  z: the chunk's [n, w] logits with row pitch ld.
// One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
logit_stats_kernel(const float* __restrict__ z, long long ld, long long n, int w, int c0,
                   const long long* __restrict__ action, long long a_off, float* __restrict__ run_max,
                   float* __restrict__ run_sum, float* __restrict__ za) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    const float* row = z + r * ld;
    float m = -INFINITY, s = 0.f;
    for (int j = threadIdx.x; j < w; j += blockDim.x) {     // the same reduction as softmax_rows_kernel
      const float x = row[j];
      if (x > m) {
        s = s * __expf(m - x) + 1.f;
        m = x;
      } else if (x != -INFINITY) {
        s += __expf(x - m);
      }
    }
    const float M = block_max(m, red);
    s = (m == -INFINITY) ? s : s * __expf(m - M);
    const float S = block_sum(s, red);
    if (threadIdx.x == 0) {
      if (c0 == 0) {
        run_max[r] = M;
        run_sum[r] = S;
      } else {
        const float M0 = run_max[r], Mn = fmaxf(M0, M);
        // no finite logit yet (M0 == M == -inf): both sums are 0, and exp(-inf - -inf) would make them NaN
        run_sum[r] = Mn == -INFINITY ? 0.f : run_sum[r] * expf(M0 - Mn) + S * expf(M - Mn);
        run_max[r] = Mn;
      }
      if (action) {
        const long long a = action[r] - a_off;
        if (a >= c0 && a < (long long)c0 + w) za[r] = row[a - c0];
      }
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

// ---- Vocabulary-sharded policy: rank q of W holds the linear2 rows of items [lo_q, hi_q), linear1 is replicated.
// A rank's record of one forward, exchanged by all-gather: a header of kShardHeader int32 words {lo, hi, num_items,
// n_rows}, then three planes of n_rows floats -- the local max m_q, the local sum s_q = sum exp(z - m_q) and the logit
// of the row's action (from its owner; 0 on every other rank).  Every rank merges the W records in rank order, so all
// of them get the same bits; at W = 1 the merge is exact (M = m_0, S = s_0 exp(0) = s_0), so the sharded path computes
// what the unsharded one does.
constexpr int kShardHeader = 4;
__host__ __device__ __forceinline__ int64_t shard_record_floats(int64_t n) { return kShardHeader + 3 * n; }

// This rank's place in the plan: rank `rank` of `world` holds items [lo, hi) of the `items`-item vocabulary.
struct ShardPlan {
  int world, rank, lo, hi, items;
};

// The plan of an arena holding `local_items` items on shard v; RECNN_E_INVALID when v does not describe one.
static int shard_plan(int local_items, const recnn_vocab_shard* v, ShardPlan* p) {
  RECNN_REQUIRE(v && v->world >= 1 && v->rank >= 0 && v->rank < v->world && v->item_offset >= 0 &&
                    (int64_t)v->item_offset + local_items <= (int64_t)v->num_items,
                "shard: rank / world / item_offset + num_items outside the vocabulary");
  *p = ShardPlan{v->world, v->rank, v->item_offset, v->item_offset + local_items, v->num_items};
  return RECNN_OK;
}

// Plane j (of n floats) of a record; in gathered records of `stride` floats, of rank q's record.
template <typename T>
__host__ __device__ __forceinline__ T* shard_plane(T* rec, long long n, long long j, int q = 0, long long stride = 0) {
  return rec + q * stride + kShardHeader + j * n;
}

__device__ __forceinline__ void shard_header_write(float* rec, const ShardPlan& p, long long n) {
  int* h = reinterpret_cast<int*>(rec);
  h[0] = p.lo; h[1] = p.hi; h[2] = p.items; h[3] = (int)n;
}

// true unless the p.world headers (records of `stride` floats) tile [0, p.items) in rank order, every rank saw n rows
// and this rank's entry is [p.lo, p.hi)
__device__ bool shard_plan_bad(const float* __restrict__ g, long long stride, const ShardPlan& p, long long n) {
  int expect = 0;
  bool bad = false;
  for (int q = 0; q < p.world; ++q) {
    const int* h = reinterpret_cast<const int*>(g + q * stride);
    bad = bad || h[0] != expect || h[1] <= h[0] || h[2] != p.items || h[3] != (int)n;
    expect = h[1];
    if (q == p.rank) bad = bad || h[0] != p.lo || h[1] != p.hi;
  }
  return bad || expect != p.items;
}

// header, and a zero action-logit plane (the owners overwrite their rows in pass 1)
__global__ void shard_record_init_kernel(float* __restrict__ rec, long long n, ShardPlan p) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) shard_plane(rec, n, 2)[i] = 0.f;
  if (i == 0) shard_header_write(rec, p, n);
}

// the rank-order merge of row r's statistics from W records of `stride` floats that start with the header and the
// m and s planes: M = max m_q, S = sum s_q exp(m_q - M)
__device__ __forceinline__ void shard_merge_stats(const float* __restrict__ g, long long stride, int W, long long n,
                                                  long long r, float& M, float& S) {
  M = -INFINITY;
  for (int q = 0; q < W; ++q) M = fmaxf(M, shard_plane(g, n, 0, q, stride)[r]);
  S = 0.f;
  for (int q = 0; q < W; ++q) S += shard_plane(g, n, 1, q, stride)[r] * expf(shard_plane(g, n, 0, q, stride)[r] - M);
}

// the rank-order merge of row r: M and S as above, za = sum za_q
__device__ __forceinline__ void shard_merge_row(const float* __restrict__ g, int W, long long n, long long r, float& M,
                                                float& S, float& za) {
  const long long stride = shard_record_floats(n);
  shard_merge_stats(g, stride, W, n, r, M, S);
  za = 0.f;
  for (int q = 0; q < W; ++q) za += shard_plane(g, n, 2, q, stride)[r];
}

// gathered records -> the merged statistics of every row (into the scratch the unsharded path uses); *plan_bad
__global__ void shard_merge_kernel(const float* __restrict__ g, long long n, ShardPlan p, float* __restrict__ run_max,
                                   float* __restrict__ run_sum, float* __restrict__ za, int* plan_bad) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0 && shard_plan_bad(g, shard_record_floats(n), p, n)) *plan_bad = 1;
  if (r >= n) return;
  float M, S, z;
  shard_merge_row(g, p.world, n, r, M, S, z);
  run_max[r] = M;
  run_sum[r] = S;
  za[r] = z;
}

// the rank's logits block [n, w] -> its block of the softmax, exp(z - M) / S (the last loop of softmax_rows_kernel)
__global__ void __launch_bounds__(kRowThreads)
shard_softmax_finish_kernel(float* __restrict__ z, long long n, int w, const float* __restrict__ g, ShardPlan p,
                            int* plan_bad) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && shard_plan_bad(g, shard_record_floats(n), p, n)) *plan_bad = 1;
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float M, S, za;
    shard_merge_row(g, p.world, n, r, M, S, za);
    float* row = z + r * w;
    for (int j = threadIdx.x; j < w; j += blockDim.x) row[j] = expf(row[j] - M) / S;
  }
}

// A draw's record: two planes of n -- the global item id (int32 bits; -1 on every rank but the owner) and its log-prob.

// One draw per row over the whole vocabulary from the rank's block of the softmax.  Every rank finds the owner of u
// from the shard masses P_q = s_q exp(m_q - M) / S (the first rank whose cumulative mass exceeds u); the owner draws
// inside its block at u' = (u - C_{owner-1}) / P_owner with the inverse CDF of categorical_sample_kernel.  At W = 1,
// P_0 = 1 and u' = u exactly.  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
shard_sample_kernel(const float* __restrict__ probs, long long n, int w, const float* __restrict__ g, ShardPlan p,
                    const float* __restrict__ uniforms, unsigned long long seed, long long draw,
                    float* __restrict__ draw_rec) {
  __shared__ float red[32];
  __shared__ CdfShared sh;
  const long long stride = shard_record_floats(n);
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float M, S, za;
    shard_merge_row(g, p.world, n, r, M, S, za);
    const float u = draw_uniform(uniforms, seed, draw, r);
    int owner = -1, last = -1;
    float C = 0.f, before = 0.f, P = 0.f, last_before = 0.f, last_P = 0.f;
    for (int q = 0; q < p.world; ++q) {
      const float Pq = shard_plane(g, n, 1, q, stride)[r] * expf(shard_plane(g, n, 0, q, stride)[r] - M) / S;
      if (Pq > 0.f) {
        if (owner < 0 && C + Pq > u) {
          owner = q; before = C; P = Pq;
        }
        last = q; last_before = C; last_P = Pq;
      }
      C += Pq;
    }
    if (owner < 0) {                   // u rounded past the last cumulative mass: the last rank with mass
      owner = last; before = last_before; P = last_P;
    }
    if (owner != p.rank) {             // the same decision in every thread
      if (threadIdx.x == 0) {
        draw_rec[r] = __int_as_float(-1);
        draw_rec[n + r] = 0.f;
      }
      continue;
    }
    const float* row = probs + r * w;
    float t = 0.f;
    for (int j = threadIdx.x; j < w; j += blockDim.x) t += row[j];
    const float total = block_sum(t, red);
    const float u2 = fminf((u - before) / P, 0x1.fffffep-1f);
    const int a = inverse_cdf_row(row, w, u2 * total, sh);
    if (threadIdx.x == 0) {
      draw_rec[r] = __int_as_float(p.lo + a);
      draw_rec[n + r] = clamped_log_prob(row[a] / total * P);
    }
    __syncthreads();
  }
}

// the log-prob of given global ids, from their owner's block of the softmax; *oob when an id is outside [0, items)
__global__ void shard_log_prob_kernel(const float* __restrict__ probs, long long n, int w, int lo, int items,
                                      const long long* __restrict__ action, float* __restrict__ draw_rec, int* oob) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const long long a = action[r];
  if (a < 0 || a >= items) *oob = 1;
  const bool mine = a >= lo && a < (long long)lo + w;
  draw_rec[r] = __int_as_float(mine ? (int)a : -1);
  draw_rec[n + r] = mine ? clamped_log_prob(probs[r * w + (a - lo)]) : 0.f;
}

// gathered draw records [W][2][n] -> (id, log-prob) of every row; *disagree unless exactly one rank claimed the row
__global__ void shard_pick_kernel(const float* __restrict__ g, int W, long long n, long long* __restrict__ action,
                                  float* __restrict__ logp, int* disagree) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  int claims = 0, id = -1;
  float lp = 0.f;
  for (int q = 0; q < W; ++q) {
    const float* d = g + (long long)q * 2 * n;
    const int v = __float_as_int(d[r]);
    if (v >= 0) {
      if (claims == 0) {
        id = v;
        lp = d[n + r];
      }
      ++claims;
    }
  }
  if (claims != 1) *disagree = 1;
  action[r] = id;
  logp[r] = lp;
}

static int row_grid(int64_t n) { return (int)(n < (int64_t)kNumSMs * 8 ? n : (int64_t)kNumSMs * 8); }

static bool chunk_ok(int num_items, int64_t chunk) {
  return chunk == num_items || (chunk > 0 && chunk % 128 == 0 && chunk < num_items);
}

// split-K partial floats of a weight gradient [num_items, K] computed in row blocks of `chunk` items, the last one
// possibly narrower.  dw_splits sees a block's width only through ceil(width / 128) and the partials grow with the width
// at a fixed split count, so the widest width of every 128-band bounds that band; once both back ends use one split
// (the partials are exactly [c, K + 1]), they only grow with the width.  Independent of num_items when chunk < num_items.
static int64_t chunked_partial_floats(int chunk, int num_items, int K, int64_t rows) {
  int64_t best = dw_partial_floats(chunk, K, rows);
  if (chunk != num_items) {
    for (int64_t c = 128; c < chunk; c += 128) {
      const int64_t f = dw_partial_floats((int)c, K, rows);
      best = std::max(best, f);
      if (f == c * (K + 1)) break;
    }
  }
  return best;
}

struct DiscreteScratch {
  float *img, *h, *z, *dh, *row_loss, *run_max, *run_sum, *za, *g, *partial;
  int* flags;
  int64_t floats;
};
// chunk == 0: the forward only.  Otherwise the policy gradient over item chunks of `chunk` (z is [n, chunk]) and its
// two weight gradients, dW2 in row blocks of `chunk` items.
static DiscreteScratch discrete_carve(const recnn_discrete_dims& d, int64_t n, int chunk, void* base) {
  DiscreteScratch s;
  Carve c(base);
  s.img = c.take(n * pad4(d.state_dim));
  s.h = c.take(n * d.hidden);
  s.flags = c.take<int>(4);
  s.z = s.dh = s.row_loss = s.run_max = s.run_sum = s.za = s.g = s.partial = nullptr;
  if (chunk > 0) {
    s.z = c.take(n * (int64_t)chunk);
    s.dh = c.take(n * d.hidden);
    s.row_loss = c.take(n);
    s.run_max = c.take(n);
    s.run_sum = c.take(n);
    s.za = c.take(n);
    s.g = c.take(n);
    s.partial = c.take(std::max(dw_partial_floats(d.hidden, d.state_dim, n),
                                chunked_partial_floats(chunk, d.num_items, d.hidden, n)));
  }
  s.floats = c.floats();
  return s;
}

// h = relu(W1 s + b1) into s.h, kept for the backward; *xs_out = the re-pitched state
static int discrete_hidden(const recnn_discrete_dims& d, const float* params, const float* state, int64_t n,
                           const DiscreteScratch& s, cudaStream_t st, Seg* xs_out) {
  const DiscreteLayout l = discrete_layout(d);
  Seg xs;
  RECNN_PROPAGATE(repitch_state(d.state_dim, state, n, s.img, &xs, st));
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

// Pass 1 of the policy gradient over the arena's items in chunks of `chunk`: per-row max / sum of exp of every logit,
// and the logit of item a_r (a_off: the item id of the arena's first linear2 row).  The last chunk's logits stay in s.z.
static int reinforce_stats_pass(const recnn_discrete_dims& d, const float* params, int64_t n, const DiscreteScratch& s,
                                int chunk, const long long* act, long long a_off, float* run_max, float* run_sum,
                                float* za, cudaStream_t st) {
  const int I = d.num_items;
  for (int c0 = 0; c0 < I; c0 += chunk) {
    const int w = I - c0 < chunk ? I - c0 : chunk;
    RECNN_PROPAGATE(discrete_logits(d, params, n, s, c0, w, s.z, st));
    logit_stats_kernel<<<row_grid(n), kRowThreads, 0, st>>>(s.z, w, n, w, c0, act, a_off, run_max, run_sum, za);
    RECNN_CHECK_LAUNCH("logit_stats_kernel");
  }
  return RECNN_OK;
}

// Pass 2, last chunk first (its logits are still in s.z): dz = d loss / d logits of the chunk from s.run_max, s.run_sum
// and s.g; dW2[c0:c0+w] = dz^T h, db2[c0:c0+w] = colsum dz; dh (+)= dz W2[c0:c0+w], gated by [h > 0] after the last
// term; then dW1 = dh^T s, db1 = colsum dh.
static int reinforce_grad_pass(const recnn_discrete_dims& d, const float* params, float* grads, int64_t n,
                               const DiscreteScratch& s, int chunk, const long long* act, long long a_off, const Seg& xs,
                               cudaStream_t st) {
  const DiscreteLayout l = discrete_layout(d);
  const int H = d.hidden, I = d.num_items;
  const int n_chunks = (int)ceil_div(I, chunk);
  const Seg sh = {s.h, H, H, 0};
  for (int c = n_chunks - 1; c >= 0; --c) {
    const int c0 = c * chunk, w = I - c0 < chunk ? I - c0 : chunk;
    if (c != n_chunks - 1) RECNN_PROPAGATE(discrete_logits(d, params, n, s, c0, w, s.z, st));
    reinforce_dlogits_kernel<<<row_grid(n), kRowThreads, 0, st>>>(s.z, n, w, (int)(a_off + c0), act, s.run_max,
                                                                    s.run_sum, s.g);
    RECNN_CHECK_LAUNCH("reinforce_dlogits_kernel");
    const int64_t w2 = l.w2 + (int64_t)c0 * l.ld2;
    RECNN_PROPAGATE(weight_grad(s.z, w, sh, kNoSeg, n, grads + w2, l.ld2, grads + l.b2 + c0, s.partial, st));
    RECNN_PROPAGATE(backprop_hidden(s.z, w, params + w2, l.ld2, H, 0, H, n, c == 0 ? s.h : nullptr, 1.f, s.dh, st,
                                    c != n_chunks - 1));
  }
  return weight_grad(s.dh, H, xs, kNoSeg, n, grads + l.w1, l.ld1, grads + l.b1, s.partial, st);
}


// ---- The policy's top-k (serving): the k best items of every row by logit, with pi of each, never forming the
// [n, num_items] probabilities.  The items are visited in chunks as in pass 1 of the policy gradient: each chunk's
// logits fold into (run_max, run_sum) through logit_stats_kernel, and its best k candidates merge into a running list
// of k (key = -logit, global id) per row, sorted best first (ties: smaller id).  Finish: pi = exp(z - M) / S, the
// expression of softmax_rows_kernel.
constexpr int kMaxExclude = 256;     // E of the dense [n, E] form
constexpr int kTopkSplitCap = 31;     // the running list takes lane 0 of the merge warp

// -logit, with NaN and -inf logits ranked after every finite one (and still before an empty slot, by id)
__device__ __forceinline__ float logit_key(float z) { return finite_key(-z); }

__global__ void cand_fill_kernel(Cand* __restrict__ c, long long count) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) c[i] = Cand{FLT_MAX, kNoId};
}

// ---- The key a select pass ranks items by (smaller first).  LogitKey: -z, the top-k.  GumbelKey: -(z + G) with G a
// standard Gumbel variate per (row, item); the best k of z + G are k draws without replacement from softmax(z), in
// draw order (Gumbel-top-k, a Plackett-Luce draw), so sampling is the top-k pass with this key.
struct LogitKey {
  static constexpr bool kPruned = false;
  __device__ __forceinline__ float operator()(float z, long long, int) const { return logit_key(z); }
};

// G = -log(-log u) with u from Philox(seed) at counter (item id, global row << 8 | kGumbelTag); the tag is used by no
// other draw of the library (dropout / TD3 noise: streams 0..15, Categorical draws: 0x5a), and a row below 2^55 keeps
// the row bits clear of the tag.  u = (2 m + 1) 2^-24 with m the top 23 bits of word x: exact in fp32 and strictly
// inside (0, 1) -- the 24-bit (x >> 8) + 0.5 would round to 1 in fp32 at its largest value.
constexpr unsigned kGumbelTag = 0x67u;
constexpr long long kMaxSampleRow = 1LL << 55;
__device__ __forceinline__ float gumbel_noise(unsigned long long seed, long long row, int id) {
  const uint4 q = Philox(seed)((unsigned long long)id, ((unsigned long long)row << 8) | kGumbelTag);
  const float u = (float)(2u * (q.x >> 9) + 1u) * 5.9604644775390625e-08f;
  return -logf(-logf(u));
}

// The bound that lets the select pass skip the Philox call and the two logs.  u <= 1 - 2^-24, so -log u >=
// 2^-24 (1 + 2^-25) and G <= -log(2^-24) = 24 ln 2 = 16.6355 in exact arithmetic; logf is within 2 ulp, which moves
// -log u by a relative 2.4e-7 and G by as much absolutely, so 16.75 bounds every fp32 G.  With G <= kGumbelMax,
// z + G <= z + kGumbelMax, and fp32 rounding is monotone, so key(z) >= bound(z) for the same id: an item whose bound
// does not beat the thread's k-th and the row's running k-th cannot enter with its real key either, and skipping it
// changes no result.
constexpr float kGumbelMax = 16.75f;
struct GumbelKey {
  static constexpr bool kPruned = true;
  unsigned long long seed;
  long long row0;               // the global row of the call's row 0
  __device__ __forceinline__ float bound(float z) const { return fminf(-(z + kGumbelMax), FLT_MAX); }
  __device__ __forceinline__ float operator()(float z, long long r, int id) const {
    return fminf(-(z + gumbel_noise(seed, row0 + r, id)), FLT_MAX);     // NaN and -inf logits last, as logit_key
  }
};

// grid (splits, rows): the best k of columns [lo, hi) of one row of a chunk's logits z [n, w] (ids id0 + j) that beat
// the row's running k-th best, ascending, into part [n, splits, k] (empty slots: {FLT_MAX, kNoId}).  A candidate is
// tested against the row's excluded set (global ids, topk.cuh) only once it beats its thread's list and the running k-th
// (SETS; without, nothing is staged).  Key: the ranking key of a logit (LogitKey, GumbelKey); it is the last parameter,
// so the top-k's instantiations keep their parameter offsets.
template <int KMAX, bool SETS, class Key>
__global__ void __launch_bounds__(kTopkThreads)
policy_topk_select_kernel(const float* __restrict__ z, long long n, int w, int id0, int k, ItemSets ex, int stage_cap,
                          const Cand* __restrict__ run, Cand* __restrict__ part, Key key_of) {
  extern __shared__ int s_set[];
  const int sp = blockIdx.x, splits = gridDim.x;
  const int per = (w + splits - 1) / splits;
  const int lo = sp * per, hi = min(w, lo + per);
  for (long long r = blockIdx.y; r < n; r += gridDim.y) {
    SetView set = {nullptr, 0, true};
    if (SETS) {
      set = set_stage(ex, r, s_set, stage_cap);
      __syncthreads();
    }
    const Cand bar = run[r * k + k - 1];
    float keys[KMAX];
    int ids[KMAX];
    list_clear(keys, ids);
    const float* row = z + r * w;
    for (int j = lo + threadIdx.x; j < hi; j += blockDim.x) {
      const int id = id0 + j;
      if constexpr (Key::kPruned) {
        const float best = key_of.bound(row[j]);
        if (!better(best, id, keys[KMAX - 1], ids[KMAX - 1]) || !better(best, id, bar.key, bar.id)) continue;
      }
      const float key = key_of(row[j], r, id);
      if (better(key, id, keys[KMAX - 1], ids[KMAX - 1]) && better(key, id, bar.key, bar.id) &&
          (!SETS || set.n == 0 || !set_has(set, s_set, id)))
        list_insert(keys, ids, key, id);
    }
    block_merge(keys, ids, k, part + (r * splits + sp) * k);
    __syncthreads();                                        // s_set is refilled for the next row
  }
}

// one warp per row: run_out = the best k of run_in and the row's `splits` partial lists (all sorted)
__global__ void __launch_bounds__(128)
policy_topk_merge_kernel(const Cand* __restrict__ run_in, const Cand* __restrict__ part, int splits, int k, long long n,
                         Cand* __restrict__ run_out) {
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const Cand* mine = lane == 0 ? run_in + r * k : part + (r * splits + lane - 1) * k;
  const bool has = lane <= splits;
  warp_merge<1>(k, [&](int, int pos) { return has && pos < k ? mine[pos] : Cand{FLT_MAX, kNoId}; },
                [&](int i, float key, int id, int) {
                  if (lane == 0) run_out[r * k + i] = Cand{key, id};
                });
}

// ids (-1 for an empty slot) and pi = exp(z - M) / S of the final lists
__global__ void policy_topk_finish_kernel(const Cand* __restrict__ run, long long n, int k,
                                          const float* __restrict__ run_max, const float* __restrict__ run_sum,
                                          float* __restrict__ values, long long* __restrict__ ids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * k) return;
  const long long r = i / k;
  const Cand c = run[i];
  const bool none = c.id == kNoId;
  ids[i] = none ? -1 : c.id;
  values[i] = none ? 0.f : expf(-c.key - run_max[r]) / run_sum[r];
}

// *flag |= 1 when an excluded id is >= items (negative ids are padding)
__global__ void exclude_check_kernel(const long long* __restrict__ exclude, long long count, long long items,
                                     int* flag) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count && exclude[i] >= items) atomicOr(flag, 1);
}

// A rank's top-k record: the header {lo, hi, num_items, n_rows}, the m and s planes (written by the passes), then k
// logit planes and k id planes (int32 bits; an empty slot is logit -FLT_MAX, id -1), plane j holding every row's j-th.
__host__ __device__ __forceinline__ int64_t topk_record_floats(int64_t n, int k) {
  return kShardHeader + (2 + 2 * (int64_t)k) * n;
}

__global__ void policy_topk_record_kernel(const Cand* __restrict__ run, long long n, int k, ShardPlan p,
                                          float* __restrict__ rec) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) shard_header_write(rec, p, n);
  if (i >= n * k) return;
  const long long r = i / k, j = i % k;
  const Cand c = run[i];
  float* planes = shard_plane(rec, n, 2);
  planes[j * n + r] = -c.key;
  planes[(k + j) * n + r] = __int_as_float(c.id == kNoId ? -1 : c.id);
}

// gathered top-k records -> every rank's (values, ids): M and S merged in rank order (shard_merge_stats), then a k-way
// merge of the W sorted lists.  One warp per row, lane q reads rank q's list (W <= 32).  *flag |= 2 when the headers do
// not tile the vocabulary with this rank's block.
__global__ void __launch_bounds__(128)
policy_topk_shard_finish_kernel(const float* __restrict__ g, long long n, int k, ShardPlan p,
                                float* __restrict__ values, long long* __restrict__ ids, int* flag) {
  const long long stride = topk_record_floats(n, k);
  if (blockIdx.x == 0 && threadIdx.x == 0 && shard_plan_bad(g, stride, p, n)) atomicOr(flag, 2);
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int W = p.world;
  float M, S;
  shard_merge_stats(g, stride, W, n, r, M, S);
  const float* planes = shard_plane(g, n, 2, lane < W ? lane : 0, stride);
  warp_merge<1>(k, [&](int, int pos) {
    Cand c = {FLT_MAX, kNoId};
    if (lane < W && pos < k) {
      const int v = __float_as_int(planes[(k + pos) * n + r]);
      if (v >= 0) c = Cand{-planes[pos * n + r], v};
    }
    return c;
  }, [&](int i, float key, int id, int) {
    if (lane == 0) {
      const bool none = id == kNoId;
      ids[r * k + i] = none ? -1 : id;
      values[r * k + i] = none ? 0.f : expf(-key - M) / S;
    }
  });
}

// ---- Sampled slates (serving): the select pass with GumbelKey.  Its lists hold perturbed keys, so a winner's value
// needs its logit again: one warp per (row, slot) recomputes z = W2[id] . h + b2[id] from the hidden layer the pass left
// in the workspace (k dot products of length H per row, in a fixed lane order).  It is fp32 like the GEMM's logit but
// summed in another order, so a value differs from forward()'s by that reordering only.
__device__ __forceinline__ float item_logit(const float* __restrict__ h, const float* __restrict__ w2, int ld2,
                                            const float* __restrict__ b2, int H, int local) {
  const float* wr = w2 + (long long)local * ld2;
  float acc = 0.f;
  for (int c = threadIdx.x & 31; c < H; c += 32) acc = fmaf(h[c], wr[c], acc);
  return warp_sum(acc) + b2[local];
}

// ids (-1 for an empty slot) and pi = exp(z - M) / S of the final lists of an unsharded call
__global__ void __launch_bounds__(128)
policy_sample_finish_kernel(const Cand* __restrict__ run, long long n, int k, const float* __restrict__ h, int H,
                            const float* __restrict__ w2, int ld2, const float* __restrict__ b2,
                            const float* __restrict__ run_max, const float* __restrict__ run_sum,
                            float* __restrict__ values, long long* __restrict__ ids) {
  const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (i >= n * k) return;
  const long long r = i / k;
  const Cand c = run[i];
  if (c.id == kNoId) {
    if ((threadIdx.x & 31) == 0) { ids[i] = -1; values[i] = 0.f; }
    return;
  }
  const float zc = item_logit(h + r * H, w2, ld2, b2, H, c.id);
  if ((threadIdx.x & 31) == 0) {
    ids[i] = c.id;
    values[i] = expf(zc - run_max[r]) / run_sum[r];
  }
}

// A rank's sample record: the header {lo, hi, num_items, n_rows}, the m and s planes (written by the passes), k key
// planes (the perturbed keys -(z + G), an empty slot FLT_MAX), k logit planes, k id planes (int32 bits, empty -1), then
// the seed as two int32 words (low, high), so that the finish can refuse ranks that drew different noise.
__host__ __device__ __forceinline__ int64_t sample_record_floats(int64_t n, int k) {
  return kShardHeader + (2 + 3 * (int64_t)k) * n + 2;
}

__global__ void __launch_bounds__(128)
policy_sample_record_kernel(const Cand* __restrict__ run, long long n, int k, const float* __restrict__ h, int H,
                            const float* __restrict__ w2, int ld2, const float* __restrict__ b2, ShardPlan p,
                            unsigned long long seed, float* __restrict__ rec) {
  const long long i = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i == 0 && lane == 0) {
    shard_header_write(rec, p, n);
    int* s = reinterpret_cast<int*>(rec + sample_record_floats(n, k) - 2);
    s[0] = (int)(unsigned)seed;
    s[1] = (int)(unsigned)(seed >> 32);
  }
  if (i >= n * k) return;
  const long long r = i / k, j = i % k;
  const Cand c = run[i];
  float* planes = shard_plane(rec, n, 2);
  const float zc = c.id == kNoId ? 0.f : item_logit(h + r * H, w2, ld2, b2, H, c.id - p.lo);
  if (lane == 0) {
    planes[j * n + r] = c.key;
    planes[(k + j) * n + r] = zc;
    planes[(2 * k + j) * n + r] = __int_as_float(c.id == kNoId ? -1 : c.id);
  }
}

// gathered sample records -> every rank's (values, ids): M and S merged in rank order (shard_merge_stats), a k-way merge
// of the W sorted key lists, the value from the winner's logit.  One warp per row, lane q reads rank q's list (W <= 32).
// *flag |= 2 when the headers do not tile the vocabulary with this rank's block or a record's seed is not `seed`.
__global__ void __launch_bounds__(128)
policy_sample_shard_finish_kernel(const float* __restrict__ g, long long n, int k, ShardPlan p,
                                  unsigned long long seed, float* __restrict__ values, long long* __restrict__ ids,
                                  int* flag) {
  const long long stride = sample_record_floats(n, k);
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    bool bad = shard_plan_bad(g, stride, p, n);
    for (int q = 0; q < p.world; ++q) {
      const int* s = reinterpret_cast<const int*>(g + q * stride + stride - 2);
      bad = bad || (unsigned)s[0] != (unsigned)seed || (unsigned)s[1] != (unsigned)(seed >> 32);
    }
    if (bad) atomicOr(flag, 2);
  }
  const long long r = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int W = p.world;
  float M, S;
  shard_merge_stats(g, stride, W, n, r, M, S);
  const float* planes = shard_plane(g, n, 2, lane < W ? lane : 0, stride);
  float zc;                                                 // the logit of this lane's head, read with its key
  warp_merge<1>(k, [&](int, int pos) {
    Cand c = {FLT_MAX, kNoId};
    zc = 0.f;
    if (lane < W && pos < k) {
      const int v = __float_as_int(planes[(2 * k + pos) * n + r]);
      if (v >= 0) {
        c = Cand{planes[pos * n + r], v};
        zc = planes[(k + pos) * n + r];
      }
    }
    return c;
  }, [&](int i, float key, int id, int owner) {
    const float z = __shfl_sync(0xffffffffu, zc, owner);
    if (lane == 0) {
      const bool none = id == kNoId;
      ids[r * k + i] = none ? -1 : id;
      values[r * k + i] = none ? 0.f : expf(z - M) / S;
    }
  });
}

struct TopkWorkspace {
  DiscreteScratch s;           // img, h and z ([n, chunk]) for discrete_hidden / discrete_logits
  float *run_max, *run_sum;
  Cand *list[2], *part;        // two running lists [n, k] (ping-pong), the chunk's partial lists [n, splits, k]
  long long* sorted;           // the dense form's [n, E <= kMaxExclude] ids, each row ascending
  int64_t bytes;
};
static TopkWorkspace topk_carve(const recnn_discrete_dims& d, int64_t n, int k, int chunk, void* base) {
  TopkWorkspace w;
  Carve c(base);
  memset(&w.s, 0, sizeof(w.s));
  w.s.img = c.take(n * pad4(d.state_dim));
  w.s.h = c.take(n * d.hidden);
  w.s.z = c.take(n * (int64_t)chunk);
  w.run_max = c.take(n);
  w.run_sum = c.take(n);
  w.list[0] = c.take<Cand>(n * k);
  w.list[1] = c.take<Cand>(n * k);
  w.part = c.take<Cand>(n * topk_splits(n, chunk, kTopkSplitCap) * k);     // the widest chunk has the most splits
  w.sorted = c.take<long long>(n * kMaxExclude);
  w.bytes = c.bytes();
  return w;
}

// The hidden layer, then every chunk: logits, row statistics into (run_max, run_sum), selection by key_of's key and
// merge.  Candidate ids are id0 + the local item.  Returns the final lists; the hidden layer stays in w.s.h.
template <class Key>
static int policy_topk_pass(const recnn_discrete_dims& d, const float* params, const float* state, int64_t n, int k,
                            const ItemSets& ex, int chunk, int id0, const TopkWorkspace& w, float* run_max,
                            float* run_sum, const Cand** lists, cudaStream_t st, Key key_of = Key()) {
  const int I = d.num_items;
  // the dense form stages its E ids, a table up to kSetStage
  const int cap = !ex.ids ? 0 : (ex.offsets ? kSetStage : ex.stride), stage = cap * (int)sizeof(int);
  auto select = k <= 16 ? (cap ? policy_topk_select_kernel<16, true, Key> : policy_topk_select_kernel<16, false, Key>)
                        : (cap ? policy_topk_select_kernel<64, true, Key> : policy_topk_select_kernel<64, false, Key>);
  RECNN_PROPAGATE(discrete_hidden(d, params, state, n, w.s, st, nullptr));
  cand_fill_kernel<<<(unsigned)ceil_div(n * k, 256), 256, 0, st>>>(w.list[0], n * k);
  RECNN_CHECK_LAUNCH("cand_fill_kernel");
  int cur = 0;
  for (int c0 = 0; c0 < I; c0 += chunk) {
    const int cw = I - c0 < chunk ? I - c0 : chunk;
    RECNN_PROPAGATE(discrete_logits(d, params, n, w.s, c0, cw, w.s.z, st));
    logit_stats_kernel<<<row_grid(n), kRowThreads, 0, st>>>(w.s.z, cw, n, cw, c0, nullptr, 0, run_max, run_sum,
                                                            nullptr);
    RECNN_CHECK_LAUNCH("logit_stats_kernel");
    const int splits = topk_splits(n, cw, kTopkSplitCap);
    const dim3 grid((unsigned)splits, (unsigned)(n < 65535 ? n : 65535));
    select<<<grid, kTopkThreads, stage, st>>>(w.s.z, n, cw, id0 + c0, k, ex, cap, w.list[cur], w.part, key_of);
    RECNN_CHECK_LAUNCH("policy_topk_select_kernel");
    policy_topk_merge_kernel<<<(unsigned)ceil_div(n, 4), 128, 0, st>>>(w.list[cur], w.part, splits, k, n,
                                                                       w.list[cur ^ 1]);
    RECNN_CHECK_LAUNCH("policy_topk_merge_kernel");
    cur ^= 1;
  }
  *lists = w.list[cur];
  return RECNN_OK;
}

static int exclude_check(const long long* exclude, int64_t n, int n_ex, int64_t items, int* flag, cudaStream_t st) {
  if (n_ex == 0) return RECNN_OK;
  exclude_check_kernel<<<(unsigned)ceil_div(n * n_ex, 256), 256, 0, st>>>(exclude, n * n_ex, items, flag);
  RECNN_CHECK_LAUNCH("exclude_check_kernel");
  return RECNN_OK;
}

// The dense [n, n_ex] form as a table: each row sorted into the workspace, row r excluding segment r
static int dense_sets(const long long* exclude, int64_t n, int n_ex, const TopkWorkspace& w, ItemSets* out,
                      cudaStream_t st) {
  *out = ItemSets{nullptr, nullptr, nullptr, 0, 0, 0};
  if (n_ex == 0) return RECNN_OK;
  exclude_sort_kernel<<<(unsigned)n, pow2_threads(n_ex), 0, st>>>(exclude, n_ex, w.sorted);
  RECNN_CHECK_LAUNCH("exclude_sort_kernel");
  *out = ItemSets{w.sorted, nullptr, nullptr, n * n_ex, n, n_ex};
  return RECNN_OK;
}

// ---- The exact rank of each row's target item (offline evaluation): the number of eligible items j that the row's
// top-k would put before t, i.e. j != t, j not excluded and better(logit_key(z_j), j, logit_key(z_t), t).  Pass 1 is
// the policy gradient's stats pass with action = target (max, sum of exp and the target's logit za); pass 2 walks the
// chunks again, last chunk first (its logits are still in z), and counts the beating ids of each chunk with integer
// atomics (deterministic).  Both passes make the logits with the discrete_logits calls of topk's chunking, so the
// counts compare topk's own bits.

// grid (splits, rows): counts[r] += the ids id0 + j of columns [lo, hi) of z's row r that beat the target, minus the
// excluded ones (SETS).  za: the target's logit; a target outside [0, items) counts nothing.
template <bool SETS>
__global__ void __launch_bounds__(kTopkThreads)
policy_rank_count_kernel(const float* __restrict__ z, long long n, int w, int id0, int items,
                         const long long* __restrict__ target, const float* __restrict__ za, ItemSets ex,
                         int* __restrict__ counts) {
  __shared__ long long s_range[3];
  const int sp = blockIdx.x, splits = gridDim.x;
  const int per = (w + splits - 1) / splits;
  const int lo = sp * per, hi = min(w, lo + per);
  for (long long r = blockIdx.y; r < n; r += gridDim.y) {
    const long long t = target[r];
    if (t < 0 || t >= items) continue;                        // the same decision in every thread
    const float kt = logit_key(za[r]);
    const float* row = z + r * w;
    int c = 0;
    for (int j = lo + threadIdx.x; j < hi; j += blockDim.x) {
      const int id = id0 + j;
      c += id != (int)t && better(logit_key(row[j]), id, kt, (int)t);
    }
    if (SETS)
      c -= excluded_beaters(ex, r, (long long)id0 + lo, (long long)id0 + hi, kt, (int)t,
                            [&](long long x) { return logit_key(row[x - id0]); }, s_range);
    c = __reduce_add_sync(0xffffffffu, c);
    if ((threadIdx.x & 31) == 0 && c != 0) atomicAdd(counts + r, c);
  }
}

// log pi(t | s) from the row's max M, sum of exp S and the target's logit
__device__ __forceinline__ float target_log_prob(float za, float M, float S) { return (za - M) - logf(S); }

// one thread per row: rank (-1 for a target outside [0, items)) and log pi(t | s)
__global__ void policy_rank_finish_kernel(const int* __restrict__ counts, const float* __restrict__ za,
                                          const float* __restrict__ run_max, const float* __restrict__ run_sum,
                                          const long long* __restrict__ target, long long n, int items,
                                          long long* __restrict__ rank, float* __restrict__ logp) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const bool ok = target[r] >= 0 && target[r] < items;
  rank[r] = ok ? counts[r] : -1;
  logp[r] = ok ? target_log_prob(za[r], run_max[r], run_sum[r]) : 0.f;
}

struct RankWorkspace {
  DiscreteScratch s;           // img, h, z ([n, chunk]), run_max, run_sum and za for the passes
  int* counts;                 // [n] (the unsharded call)
  int64_t bytes;
};
static RankWorkspace rank_carve(const recnn_discrete_dims& d, int64_t n, int chunk, void* base) {
  RankWorkspace w;
  Carve c(base);
  memset(&w.s, 0, sizeof(w.s));
  w.s.img = c.take(n * pad4(d.state_dim));
  w.s.h = c.take(n * d.hidden);
  w.s.z = c.take(n * (int64_t)chunk);
  w.s.run_max = c.take(n);
  w.s.run_sum = c.take(n);
  w.s.za = c.take(n);
  w.counts = c.take<int>(n);
  w.bytes = c.bytes();
  return w;
}

// Pass 2 over the arena's items (global ids id0 + the local item, the last chunk's logits already in s.z): counts +=
// the beating ids of every chunk.  items: the whole vocabulary.
static int rank_count_pass(const recnn_discrete_dims& d, const float* params, int64_t n, const DiscreteScratch& s,
                           int chunk, int id0, int items, const long long* target, const float* za, const ItemSets& ex,
                           int* counts, cudaStream_t st) {
  const int I = d.num_items;
  const int n_chunks = (int)ceil_div(I, chunk);
  auto count = ex.ids ? policy_rank_count_kernel<true> : policy_rank_count_kernel<false>;
  for (int c = n_chunks - 1; c >= 0; --c) {
    const int c0 = c * chunk, w = I - c0 < chunk ? I - c0 : chunk;
    if (c != n_chunks - 1) RECNN_PROPAGATE(discrete_logits(d, params, n, s, c0, w, s.z, st));
    const dim3 grid((unsigned)topk_splits(n, w, 32), (unsigned)(n < 65535 ? n : 65535));
    count<<<grid, kTopkThreads, 0, st>>>(s.z, n, w, id0 + c0, items, target, za, ex, counts);
    RECNN_CHECK_LAUNCH("policy_rank_count_kernel");
  }
  return RECNN_OK;
}

// A rank's count record (vocabulary-parallel rank): the header {lo, hi, num_items, n_rows}, then n int32 counts of the
// rank's block.
__host__ __device__ __forceinline__ int64_t rank_record_floats(int64_t n) { return kShardHeader + n; }

__global__ void rank_record_init_kernel(float* __restrict__ rec, long long n, ShardPlan p) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) reinterpret_cast<int*>(shard_plane(rec, n, 0))[i] = 0;
  if (i == 0) shard_header_write(rec, p, n);
}

// gathered stats records -> za[r], the target's logit: the rank-order sum of shard_merge_row (every plane but the
// owner's holds 0)
__global__ void shard_target_logit_kernel(const float* __restrict__ g, long long n, int W, float* __restrict__ za) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const long long stride = shard_record_floats(n);
  float z = 0.f;
  for (int q = 0; q < W; ++q) z += shard_plane(g, n, 2, q, stride)[r];
  za[r] = z;
}

// gathered stats and count records -> every rank's (rank, log pi): M, S and za merged in rank order (shard_merge_row),
// the counts summed in rank order.  *flag |= 2 when either set of headers does not tile the vocabulary with this rank's
// block, |= 1 for a target outside [0, items).
__global__ void shard_rank_finish_kernel(const float* __restrict__ gs, const float* __restrict__ gc, long long n,
                                         ShardPlan p, const long long* __restrict__ target, long long* __restrict__ rank,
                                         float* __restrict__ logp, int* flag) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r == 0 && (shard_plan_bad(gs, shard_record_floats(n), p, n) || shard_plan_bad(gc, rank_record_floats(n), p, n)))
    atomicOr(flag, 2);
  if (r >= n) return;
  const long long t = target[r];
  if (t < 0 || t >= p.items) {
    atomicOr(flag, 1);
    rank[r] = -1;
    logp[r] = 0.f;
    return;
  }
  float M, S, za;
  shard_merge_row(gs, p.world, n, r, M, S, za);
  long long c = 0;
  for (int q = 0; q < p.world; ++q)
    c += reinterpret_cast<const int*>(shard_plane(gc, n, 0, q, rank_record_floats(n)))[r];
  rank[r] = c;
  logp[r] = target_log_prob(za, M, S);
}

// ---- log pi(a | s) and log beta(a | s) of given items (off-policy estimation): pass 1 alone, then target_log_prob.

// one thread per row: log-prob of action[r] from the row's statistics (0 for an id outside [0, items), which the
// caller's check flags)
__global__ void log_prob_finish_kernel(const float* __restrict__ za, const float* __restrict__ run_max,
                                       const float* __restrict__ run_sum, const long long* __restrict__ action,
                                       long long n, int items, float* __restrict__ logp) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const bool ok = action[r] >= 0 && action[r] < items;
  logp[r] = ok ? target_log_prob(za[r], run_max[r], run_sum[r]) : 0.f;
}

// gathered stats records (either net's) -> every rank's log-prob: M, S and the action's logit merged in rank order
// (shard_merge_row).  The finish sees no arena, so this rank's block ends where its own header says.  *flag |= 2 when
// the headers do not tile the vocabulary with this rank's first item, |= 1 for an id outside [0, items).
__global__ void vocab_log_prob_finish_kernel(const float* __restrict__ g, long long n, ShardPlan p,
                                             const long long* __restrict__ action, float* __restrict__ logp,
                                             int* flag) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long stride = shard_record_floats(n);
  if (r == 0) {
    p.hi = reinterpret_cast<const int*>(g + p.rank * stride)[1];
    if (shard_plan_bad(g, stride, p, n)) atomicOr(flag, 2);
  }
  if (r >= n) return;
  const long long a = action[r];
  if (a < 0 || a >= p.items) {
    atomicOr(flag, 1);
    logp[r] = 0.f;
    return;
  }
  float M, S, za;
  shard_merge_row(g, p.world, n, r, M, S, za);
  logp[r] = target_log_prob(za, M, S);
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
  if (!discrete_dims_ok(d) || n_rows <= 0 || !chunk_ok(d->num_items, chunk_items)) return 0;
  return discrete_carve(*d, n_rows, chunk_items, nullptr).floats;
}

extern "C" int recnn_discrete_forward(const recnn_discrete_dims* d, const float* params, const float* state,
                                      int64_t n_rows, float* probs_out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && probs_out && scratch, "null pointer / dims");
  if (n_rows <= 0) return RECNN_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const DiscreteScratch s = discrete_carve(*d, n_rows, 0, scratch);
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

extern "C" int recnn_categorical_sample_at(const float* probs, int64_t n_rows, int32_t num_items, int64_t ld,
                                           const float* uniforms, uint64_t seed, int64_t draw, int64_t row_offset,
                                           int64_t* action_out, float* log_prob_out, void* stream) {
  RECNN_REQUIRE(probs && action_out && log_prob_out, "null pointer");
  RECNN_REQUIRE(num_items > 0 && ld >= num_items, "num_items / ld");
  RECNN_REQUIRE(row_offset >= 0, "row_offset");
  if (n_rows <= 0) return RECNN_OK;
  categorical_sample_kernel<<<row_grid(n_rows), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, ld, n_rows, num_items, uniforms, seed, draw, reinterpret_cast<long long*>(action_out), log_prob_out,
      row_offset);
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

// The checks of both policy-gradient entry points after their pointers (and shard plan): the loss, rows and chunk.
static int reinforce_check(const recnn_discrete_dims& d, int64_t n_rows, int method, int top_k,
                           const float* beta_log_prob, int chunk_items) {
  RECNN_REQUIRE(method == RECNN_REINFORCE_BASIC || method == RECNN_REINFORCE_CORRECTED || method == RECNN_REINFORCE_TOPK,
                "unknown REINFORCE method");
  RECNN_REQUIRE(method == RECNN_REINFORCE_BASIC || beta_log_prob, "the corrected losses need the behaviour policy's log-probs");
  RECNN_REQUIRE(method != RECNN_REINFORCE_TOPK || top_k >= 1, "K >= 1");
  RECNN_REQUIRE(n_rows > 0, "no saved rows: select_action was never called since the last update");
  RECNN_REQUIRE(chunk_ok(d.num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  return RECNN_OK;
}

// After the row statistics (s.run_max, s.run_sum, s.za): the row weights, out[0] = the loss, pass 2, then the first
// `flag_words` int32 flags of s.flags into out[1..].  items: the whole vocabulary; a_off as in reinforce_stats_pass.
static int reinforce_finish(const recnn_discrete_dims& d, const float* params, float* grads, int64_t n,
                            const DiscreteScratch& s, int chunk, const long long* act, long long a_off, int items,
                            const float* beta_log_prob, const float* returns, int method, int top_k, const Seg& xs,
                            float* out, int flag_words, cudaStream_t st) {
  reinforce_row_weights_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(
      n, items, act, s.run_max, s.run_sum, s.za, beta_log_prob, returns, method, top_k, s.g, s.row_loss, s.flags);
  RECNN_CHECK_LAUNCH("reinforce_row_weights_kernel");
  sum_rows_kernel<<<1, 1024, 0, st>>>(s.row_loss, n, 1.f, out);
  RECNN_CHECK_LAUNCH("sum_rows_kernel");
  RECNN_PROPAGATE(reinforce_grad_pass(d, params, grads, n, s, chunk, act, a_off, xs, st));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(out + 1, s.flags, flag_words * sizeof(int), cudaMemcpyDeviceToDevice, st));
  return RECNN_OK;
}

// out[0] = policy loss, out[1] = 1.0 if an action id was outside [0, num_items) (that row contributes nothing)
extern "C" int recnn_reinforce_policy_grad_chunked(const recnn_discrete_dims* d, const float* params, float* grads,
                                                   const float* state, const int64_t* action, const float* beta_log_prob,
                                                   const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                                   int32_t chunk_items, float* out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && grads && state && action && returns && out && scratch,
                "null pointer / dims");
  RECNN_PROPAGATE(reinforce_check(*d, n_rows, method, top_k, beta_log_prob, chunk_items));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* act = reinterpret_cast<const long long*>(action);
  const DiscreteScratch s = discrete_carve(*d, n_rows, chunk_items, scratch);
  RECNN_CHECK_CUDA(cudaMemsetAsync(s.flags, 0, 4 * sizeof(int), st));
  Seg xs;
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, s, st, &xs));
  RECNN_PROPAGATE(reinforce_stats_pass(*d, params, n_rows, s, chunk_items, act, 0, s.run_max, s.run_sum, s.za, st));
  return reinforce_finish(*d, params, grads, n_rows, s, chunk_items, act, 0, d->num_items, beta_log_prob, returns,
                          method, top_k, xs, out, 1, st);
}

extern "C" int recnn_reinforce_policy_grad(const recnn_discrete_dims* d, const float* params, float* grads,
                                           const float* state, const int64_t* action, const float* beta_log_prob,
                                           const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                           float* out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d), "null pointer / dims");
  return recnn_reinforce_policy_grad_chunked(d, params, grads, state, action, beta_log_prob, returns, n_rows, method,
                                             top_k, d->num_items, out, scratch, stream);
}

// ---- the vocabulary-sharded policy: the phases around the two all-gathers (see the header) ----------------------
extern "C" int64_t recnn_vocab_record_floats(int64_t n_rows) { return n_rows > 0 ? shard_record_floats(n_rows) : 0; }

static int shard_record_init(const ShardPlan& p, float* record, int64_t n, cudaStream_t st) {
  shard_record_init_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(record, n, p);
  RECNN_CHECK_LAUNCH("shard_record_init_kernel");
  return RECNN_OK;
}

extern "C" int recnn_reinforce_shard_stats(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                           const float* state, const int64_t* action, int64_t n_rows,
                                           int32_t chunk_items, float* record, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && action && record && scratch, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "no saved rows: select_action was never called since the last update");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const DiscreteScratch s = discrete_carve(*d, n_rows, chunk_items, scratch);
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, s, st, nullptr));
  RECNN_PROPAGATE(shard_record_init(p, record, n_rows, st));
  return reinforce_stats_pass(*d, params, n_rows, s, chunk_items, reinterpret_cast<const long long*>(action), p.lo,
                              shard_plane(record, n_rows, 0), shard_plane(record, n_rows, 1),
                              shard_plane(record, n_rows, 2), st);
}

extern "C" int recnn_reinforce_shard_grad(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                          float* grads, const float* state, const int64_t* action,
                                          const float* beta_log_prob, const float* returns, int64_t n_rows,
                                          int32_t method, int32_t top_k, int32_t chunk_items, const float* gathered,
                                          float* out, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && grads && state && action && returns && gathered && out && scratch,
                "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_PROPAGATE(reinforce_check(*d, n_rows, method, top_k, beta_log_prob, chunk_items));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* act = reinterpret_cast<const long long*>(action);
  const DiscreteScratch s = discrete_carve(*d, n_rows, chunk_items, scratch);
  RECNN_CHECK_CUDA(cudaMemsetAsync(s.flags, 0, 4 * sizeof(int), st));
  // the stats phase left the state image (when one was needed) in s.img
  const Seg xs = state_seg(d->state_dim, state, 0, s.img);
  shard_merge_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(gathered, n_rows, p, s.run_max, s.run_sum, s.za,
                                                                      s.flags + 1);
  RECNN_CHECK_LAUNCH("shard_merge_kernel");
  return reinforce_finish(*d, params, grads, n_rows, s, chunk_items, act, p.lo, p.items, beta_log_prob, returns,
                          method, top_k, xs, out, 2, st);
}

extern "C" int recnn_discrete_shard_forward(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                            const float* params, const float* state, int64_t n_rows, float* probs_out,
                                            float* record, float* scratch, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && probs_out && record && scratch, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int I = d->num_items;
  const DiscreteScratch s = discrete_carve(*d, n_rows, 0, scratch);
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, s, st, nullptr));
  RECNN_PROPAGATE(discrete_logits(*d, params, n_rows, s, 0, I, probs_out, st));
  RECNN_PROPAGATE(shard_record_init(p, record, n_rows, st));
  logit_stats_kernel<<<row_grid(n_rows), kRowThreads, 0, st>>>(probs_out, I, n_rows, I, 0, nullptr, 0,
                                                                shard_plane(record, n_rows, 0),
                                                                shard_plane(record, n_rows, 1), nullptr);
  RECNN_CHECK_LAUNCH("logit_stats_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                           const float* gathered, int64_t n_rows, float* probs, int32_t* error_flag,
                                           void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && gathered && probs && error_flag, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  if (n_rows <= 0) return RECNN_OK;
  shard_softmax_finish_kernel<<<row_grid(n_rows), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, n_rows, d->num_items, gathered, p, error_flag);
  RECNN_CHECK_LAUNCH("shard_softmax_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_sample(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                           const float* gathered, const float* probs, int64_t n_rows,
                                           const float* uniforms, uint64_t seed, int64_t draw, float* draw_record,
                                           void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && gathered && probs && draw_record, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  if (n_rows <= 0) return RECNN_OK;
  shard_sample_kernel<<<row_grid(n_rows), kRowThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, n_rows, d->num_items, gathered, p, uniforms, seed, draw, draw_record);
  RECNN_CHECK_LAUNCH("shard_sample_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_log_prob(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                             const float* probs, int64_t n_rows, const int64_t* action,
                                             float* draw_record, int32_t* oob_flag, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && probs && action && draw_record && oob_flag, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  if (n_rows <= 0) return RECNN_OK;
  shard_log_prob_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      probs, n_rows, d->num_items, p.lo, p.items, reinterpret_cast<const long long*>(action), draw_record, oob_flag);
  RECNN_CHECK_LAUNCH("shard_log_prob_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_pick(int32_t world, const float* gathered_draws, int64_t n_rows,
                                         int64_t* action_out, float* log_prob_out, int32_t* error_flag, void* stream) {
  RECNN_REQUIRE(world >= 1 && gathered_draws && action_out && log_prob_out && error_flag, "null pointer / world");
  if (n_rows <= 0) return RECNN_OK;
  shard_pick_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      gathered_draws, world, n_rows, reinterpret_cast<long long*>(action_out), log_prob_out, error_flag);
  RECNN_CHECK_LAUNCH("shard_pick_kernel");
  return RECNN_OK;
}

// ---- the policy's top-k ----------------------------------------------------------------------------------------
static bool topk_args_ok(const recnn_discrete_dims& d, int64_t n, int k, int chunk) {
  return n > 0 && k >= 1 && k <= 64 && chunk_ok(d.num_items, chunk);
}

extern "C" int64_t recnn_discrete_topk_workspace_bytes(const recnn_discrete_dims* d, int64_t n_rows, int32_t k,
                                                       int32_t chunk_items) {
  if (!discrete_dims_ok(d) || !topk_args_ok(*d, n_rows, k, chunk_items)) return 0;
  return topk_carve(*d, n_rows, k, chunk_items, nullptr).bytes;
}

// the rows, k and exclusion checks of every top-k entry point
static int topk_rows_check(int64_t n_rows, int32_t k, const int64_t* exclude, int32_t n_exclude) {
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(k >= 1 && k <= 64, "1 <= k <= 64");
  RECNN_REQUIRE(n_exclude >= 0 && n_exclude <= kMaxExclude && (n_exclude == 0 || exclude), "0 <= n_exclude <= 256");
  return RECNN_OK;
}

// ... and those of the two that run the passes
static int topk_check(const recnn_discrete_dims* d, const float* params, const float* state, int64_t n_rows, int32_t k,
                      const int64_t* exclude, int32_t n_exclude, int32_t chunk_items, void* workspace,
                      int64_t workspace_bytes) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && workspace, "null pointer / dims");
  RECNN_PROPAGATE(topk_rows_check(n_rows, k, exclude, n_exclude));
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  return check_workspace(topk_carve(*d, n_rows, k, chunk_items, nullptr).bytes, workspace_bytes);
}

// the passes and the finish of an unsharded call
static int topk_local(const recnn_discrete_dims& d, const float* params, const float* state, int64_t n_rows, int k,
                      const ItemSets& sets, int chunk_items, float* values_out, int64_t* ids_out,
                      const TopkWorkspace& w, cudaStream_t st) {
  const Cand* lists;
  RECNN_PROPAGATE(policy_topk_pass<LogitKey>(d, params, state, n_rows, k, sets, chunk_items, 0, w, w.run_max,
                                             w.run_sum, &lists, st));
  policy_topk_finish_kernel<<<(unsigned)ceil_div(n_rows * k, 256), 256, 0, st>>>(
      lists, n_rows, k, w.run_max, w.run_sum, values_out, reinterpret_cast<long long*>(ids_out));
  RECNN_CHECK_LAUNCH("policy_topk_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_topk(const recnn_discrete_dims* d, const float* params, const float* state,
                                   int64_t n_rows, int32_t k, const int64_t* exclude, int32_t n_exclude,
                                   int32_t chunk_items, float* values_out, int64_t* ids_out, int32_t* error_flag,
                                   void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(values_out && ids_out && error_flag, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, exclude, n_exclude, chunk_items, workspace, workspace_bytes));
  RECNN_REQUIRE(k <= d->num_items, "k <= num_items");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* ex = reinterpret_cast<const long long*>(exclude);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(exclude_check(ex, n_rows, n_exclude, d->num_items, error_flag, st));
  ItemSets sets;
  RECNN_PROPAGATE(dense_sets(ex, n_rows, n_exclude, w, &sets, st));
  return topk_local(*d, params, state, n_rows, k, sets, chunk_items, values_out, ids_out, w, st);
}

extern "C" int recnn_discrete_topk_sets(const recnn_discrete_dims* d, const float* params, const float* state,
                                        int64_t n_rows, int32_t k, const int64_t* set_ids, int64_t n_set_ids,
                                        const int64_t* set_offsets, int64_t n_sets, const int64_t* row_set,
                                        int32_t chunk_items, float* values_out, int64_t* ids_out, int32_t* error_flag,
                                        void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(values_out && ids_out, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, nullptr, 0, chunk_items, workspace, workspace_bytes));
  RECNN_REQUIRE(k <= d->num_items, "k <= num_items");
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, d->num_items, error_flag, st));
  return topk_local(*d, params, state, n_rows, k, sets, chunk_items, values_out, ids_out, w, st);
}

extern "C" int64_t recnn_vocab_topk_record_floats(int64_t n_rows, int32_t k) {
  return n_rows > 0 && k >= 1 && k <= 64 ? topk_record_floats(n_rows, k) : 0;
}

// the passes over the rank's block and its record
static int topk_shard_local(const recnn_discrete_dims& d, const ShardPlan& p, const float* params, const float* state,
                            int64_t n_rows, int k, const ItemSets& sets, int chunk_items, float* record,
                            const TopkWorkspace& w, cudaStream_t st) {
  const Cand* lists;
  RECNN_PROPAGATE(policy_topk_pass<LogitKey>(d, params, state, n_rows, k, sets, chunk_items, p.lo, w,
                                   shard_plane(record, n_rows, 0), shard_plane(record, n_rows, 1), &lists, st));
  policy_topk_record_kernel<<<(unsigned)ceil_div(n_rows * k, 256), 256, 0, st>>>(lists, n_rows, k, p, record);
  RECNN_CHECK_LAUNCH("policy_topk_record_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_topk(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                         const float* state, int64_t n_rows, int32_t k, const int64_t* exclude,
                                         int32_t n_exclude, int32_t chunk_items, float* record, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(record, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, exclude, n_exclude, chunk_items, workspace, workspace_bytes));
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(k <= p.items, "k <= num_items (the whole vocabulary)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  ItemSets sets;
  RECNN_PROPAGATE(dense_sets(reinterpret_cast<const long long*>(exclude), n_rows, n_exclude, w, &sets, st));
  return topk_shard_local(*d, p, params, state, n_rows, k, sets, chunk_items, record, w, st);
}

extern "C" int recnn_discrete_shard_topk_sets(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                              const float* params, const float* state, int64_t n_rows, int32_t k,
                                              const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                                              int64_t n_sets, const int64_t* row_set, int32_t chunk_items,
                                              float* record, int32_t* error_flag, void* workspace,
                                              int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(record, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, nullptr, 0, chunk_items, workspace, workspace_bytes));
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(k <= p.items, "k <= num_items (the whole vocabulary)");
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, p.items, error_flag, st));   // global ids: every rank agrees
  return topk_shard_local(*d, p, params, state, n_rows, k, sets, chunk_items, record, w, st);
}

extern "C" int recnn_discrete_shard_topk_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                                const float* gathered, int64_t n_rows, int32_t k,
                                                const int64_t* exclude, int32_t n_exclude, float* values_out,
                                                int64_t* ids_out, int32_t* error_flag, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && gathered && values_out && ids_out && error_flag, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(p.world <= 32, "world <= 32");
  RECNN_PROPAGATE(topk_rows_check(n_rows, k, exclude, n_exclude));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(exclude_check(reinterpret_cast<const long long*>(exclude), n_rows, n_exclude, p.items, error_flag,
                                st));
  policy_topk_shard_finish_kernel<<<(unsigned)ceil_div(n_rows, 4), 128, 0, st>>>(
      gathered, n_rows, k, p, values_out, reinterpret_cast<long long*>(ids_out), error_flag);
  RECNN_CHECK_LAUNCH("policy_topk_shard_finish_kernel");
  return RECNN_OK;
}

// ---- the policy's sampled slates: topk's checks, workspace and passes with GumbelKey -----------------------------
static int sample_rows_check(int64_t n_rows, int64_t row_offset) {
  RECNN_REQUIRE(row_offset >= 0 && row_offset <= kMaxSampleRow - n_rows, "0 <= row_offset <= 2^55 - n_rows");
  return RECNN_OK;
}

// the passes and the finish of an unsharded call
static int sample_local(const recnn_discrete_dims& d, const float* params, const float* state, int64_t n_rows, int k,
                        const ItemSets& sets, uint64_t seed, int64_t row_offset, int chunk_items, float* values_out,
                        int64_t* ids_out, const TopkWorkspace& w, cudaStream_t st) {
  const DiscreteLayout l = discrete_layout(d);
  const Cand* lists;
  RECNN_PROPAGATE(policy_topk_pass(d, params, state, n_rows, k, sets, chunk_items, 0, w, w.run_max, w.run_sum, &lists,
                                   st, GumbelKey{seed, row_offset}));
  policy_sample_finish_kernel<<<(unsigned)ceil_div(n_rows * k, 4), 128, 0, st>>>(
      lists, n_rows, k, w.s.h, d.hidden, params + l.w2, l.ld2, params + l.b2, w.run_max, w.run_sum, values_out,
      reinterpret_cast<long long*>(ids_out));
  RECNN_CHECK_LAUNCH("policy_sample_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_sample_topk(const recnn_discrete_dims* d, const float* params, const float* state,
                                          int64_t n_rows, int32_t k, const int64_t* exclude, int32_t n_exclude,
                                          uint64_t seed, int64_t row_offset, int32_t chunk_items, float* values_out,
                                          int64_t* ids_out, int32_t* error_flag, void* workspace,
                                          int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(values_out && ids_out && error_flag, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, exclude, n_exclude, chunk_items, workspace, workspace_bytes));
  RECNN_REQUIRE(k <= d->num_items, "k <= num_items");
  RECNN_PROPAGATE(sample_rows_check(n_rows, row_offset));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* ex = reinterpret_cast<const long long*>(exclude);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(exclude_check(ex, n_rows, n_exclude, d->num_items, error_flag, st));
  ItemSets sets;
  RECNN_PROPAGATE(dense_sets(ex, n_rows, n_exclude, w, &sets, st));
  return sample_local(*d, params, state, n_rows, k, sets, seed, row_offset, chunk_items, values_out, ids_out, w, st);
}

extern "C" int recnn_discrete_sample_topk_sets(const recnn_discrete_dims* d, const float* params, const float* state,
                                               int64_t n_rows, int32_t k, const int64_t* set_ids, int64_t n_set_ids,
                                               const int64_t* set_offsets, int64_t n_sets, const int64_t* row_set,
                                               uint64_t seed, int64_t row_offset, int32_t chunk_items,
                                               float* values_out, int64_t* ids_out, int32_t* error_flag,
                                               void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(values_out && ids_out, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, nullptr, 0, chunk_items, workspace, workspace_bytes));
  RECNN_REQUIRE(k <= d->num_items, "k <= num_items");
  RECNN_PROPAGATE(sample_rows_check(n_rows, row_offset));
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, d->num_items, error_flag, st));
  return sample_local(*d, params, state, n_rows, k, sets, seed, row_offset, chunk_items, values_out, ids_out, w, st);
}

extern "C" int64_t recnn_vocab_sample_topk_record_floats(int64_t n_rows, int32_t k) {
  return n_rows > 0 && k >= 1 && k <= 64 ? sample_record_floats(n_rows, k) : 0;
}

// the passes over the rank's block and its record
static int sample_shard_local(const recnn_discrete_dims& d, const ShardPlan& p, const float* params,
                              const float* state, int64_t n_rows, int k, const ItemSets& sets, uint64_t seed,
                              int64_t row_offset, int chunk_items, float* record, const TopkWorkspace& w,
                              cudaStream_t st) {
  const DiscreteLayout l = discrete_layout(d);
  const Cand* lists;
  RECNN_PROPAGATE(policy_topk_pass(d, params, state, n_rows, k, sets, chunk_items, p.lo, w,
                                   shard_plane(record, n_rows, 0), shard_plane(record, n_rows, 1), &lists, st,
                                   GumbelKey{seed, row_offset}));
  policy_sample_record_kernel<<<(unsigned)ceil_div(n_rows * k, 4), 128, 0, st>>>(
      lists, n_rows, k, w.s.h, d.hidden, params + l.w2, l.ld2, params + l.b2, p, seed, record);
  RECNN_CHECK_LAUNCH("policy_sample_record_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_shard_sample_topk(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                                const float* params, const float* state, int64_t n_rows, int32_t k,
                                                const int64_t* exclude, int32_t n_exclude, uint64_t seed,
                                                int64_t row_offset, int32_t chunk_items, float* record,
                                                void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(record, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, exclude, n_exclude, chunk_items, workspace, workspace_bytes));
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(k <= p.items, "k <= num_items (the whole vocabulary)");
  RECNN_PROPAGATE(sample_rows_check(n_rows, row_offset));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  ItemSets sets;
  RECNN_PROPAGATE(dense_sets(reinterpret_cast<const long long*>(exclude), n_rows, n_exclude, w, &sets, st));
  return sample_shard_local(*d, p, params, state, n_rows, k, sets, seed, row_offset, chunk_items, record, w, st);
}

extern "C" int recnn_discrete_shard_sample_topk_sets(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                                     const float* params, const float* state, int64_t n_rows,
                                                     int32_t k, const int64_t* set_ids, int64_t n_set_ids,
                                                     const int64_t* set_offsets, int64_t n_sets,
                                                     const int64_t* row_set, uint64_t seed, int64_t row_offset,
                                                     int32_t chunk_items, float* record, int32_t* error_flag,
                                                     void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(record, "null pointer");
  RECNN_PROPAGATE(topk_check(d, params, state, n_rows, k, nullptr, 0, chunk_items, workspace, workspace_bytes));
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(k <= p.items, "k <= num_items (the whole vocabulary)");
  RECNN_PROPAGATE(sample_rows_check(n_rows, row_offset));
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const TopkWorkspace w = topk_carve(*d, n_rows, k, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, p.items, error_flag, st));   // global ids: every rank agrees
  return sample_shard_local(*d, p, params, state, n_rows, k, sets, seed, row_offset, chunk_items, record, w, st);
}

extern "C" int recnn_discrete_shard_sample_topk_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                                       const float* gathered, int64_t n_rows, int32_t k,
                                                       const int64_t* exclude, int32_t n_exclude, uint64_t seed,
                                                       float* values_out, int64_t* ids_out, int32_t* error_flag,
                                                       void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && gathered && values_out && ids_out && error_flag, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(p.world <= 32, "world <= 32");
  RECNN_PROPAGATE(topk_rows_check(n_rows, k, exclude, n_exclude));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(exclude_check(reinterpret_cast<const long long*>(exclude), n_rows, n_exclude, p.items, error_flag,
                                st));
  policy_sample_shard_finish_kernel<<<(unsigned)ceil_div(n_rows, 4), 128, 0, st>>>(
      gathered, n_rows, k, p, seed, values_out, reinterpret_cast<long long*>(ids_out), error_flag);
  RECNN_CHECK_LAUNCH("policy_sample_shard_finish_kernel");
  return RECNN_OK;
}

// ---- the exact rank of each row's target ---------------------------------------------------------------------
extern "C" int64_t recnn_discrete_rank_workspace_bytes(const recnn_discrete_dims* d, int64_t n_rows,
                                                       int32_t chunk_items) {
  if (!discrete_dims_ok(d) || n_rows <= 0 || !chunk_ok(d->num_items, chunk_items)) return 0;
  return rank_carve(*d, n_rows, chunk_items, nullptr).bytes;
}

// the checks of every rank entry point that runs a pass
static int rank_check(const recnn_discrete_dims* d, const float* params, const int64_t* target, int64_t n_rows,
                      int32_t chunk_items, const int32_t* error_flag, void* workspace, int64_t workspace_bytes) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && target && error_flag && workspace, "null pointer / dims");
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  return check_workspace(rank_carve(*d, n_rows, chunk_items, nullptr).bytes, workspace_bytes);
}

// pass 1 of an unsharded call: the target check, the hidden layer and the stats pass into w.s (run_max, run_sum, za)
static int rank_stats_local(const recnn_discrete_dims& d, const float* params, const float* state,
                            const long long* target, int64_t n, int chunk, int* flag, const RankWorkspace& w,
                            cudaStream_t st) {
  const DiscreteScratch& s = w.s;
  RECNN_PROPAGATE(rank_target_check(target, n, d.num_items, flag, st));
  RECNN_PROPAGATE(discrete_hidden(d, params, state, n, s, st, nullptr));
  return reinforce_stats_pass(d, params, n, s, chunk, target, 0, s.run_max, s.run_sum, s.za, st);
}

// both passes and the finish of an unsharded call
static int rank_local(const recnn_discrete_dims& d, const float* params, const float* state, const long long* target,
                      int64_t n, const ItemSets& sets, int chunk, int64_t* rank_out, float* log_prob_out, int* flag,
                      const RankWorkspace& w, cudaStream_t st) {
  const DiscreteScratch& s = w.s;
  RECNN_CHECK_CUDA(cudaMemsetAsync(w.counts, 0, n * sizeof(int), st));
  RECNN_PROPAGATE(rank_stats_local(d, params, state, target, n, chunk, flag, w, st));
  RECNN_PROPAGATE(rank_count_pass(d, params, n, s, chunk, 0, d.num_items, target, s.za, sets, w.counts, st));
  policy_rank_finish_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(
      w.counts, s.za, s.run_max, s.run_sum, target, n, d.num_items, reinterpret_cast<long long*>(rank_out),
      log_prob_out);
  RECNN_CHECK_LAUNCH("policy_rank_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_rank(const recnn_discrete_dims* d, const float* params, const float* state,
                                   const int64_t* target, int64_t n_rows, int32_t chunk_items, int64_t* rank_out,
                                   float* log_prob_out, int32_t* error_flag, void* workspace, int64_t workspace_bytes,
                                   void* stream) {
  RECNN_REQUIRE(state && rank_out && log_prob_out, "null pointer");
  RECNN_PROPAGATE(rank_check(d, params, target, n_rows, chunk_items, error_flag, workspace, workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  const ItemSets none = {nullptr, nullptr, nullptr, 0, 0, 0};
  return rank_local(*d, params, state, reinterpret_cast<const long long*>(target), n_rows, none, chunk_items, rank_out,
                    log_prob_out, error_flag, w, st);
}

extern "C" int recnn_discrete_rank_sets(const recnn_discrete_dims* d, const float* params, const float* state,
                                        const int64_t* target, int64_t n_rows, const int64_t* set_ids,
                                        int64_t n_set_ids, const int64_t* set_offsets, int64_t n_sets,
                                        const int64_t* row_set, int32_t chunk_items, int64_t* rank_out,
                                        float* log_prob_out, int32_t* error_flag, void* workspace,
                                        int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(state && rank_out && log_prob_out, "null pointer");
  RECNN_PROPAGATE(rank_check(d, params, target, n_rows, chunk_items, error_flag, workspace, workspace_bytes));
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, d->num_items, error_flag, st));
  return rank_local(*d, params, state, reinterpret_cast<const long long*>(target), n_rows, sets, chunk_items, rank_out,
                    log_prob_out, error_flag, w, st);
}

extern "C" int64_t recnn_vocab_rank_record_floats(int64_t n_rows) { return n_rows > 0 ? rank_record_floats(n_rows) : 0; }

extern "C" int recnn_discrete_shard_rank_stats(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                               const float* params, const float* state, const int64_t* target,
                                               int64_t n_rows, int32_t chunk_items, float* record, void* workspace,
                                               int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && state && target && record && workspace, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  RECNN_PROPAGATE(check_workspace(rank_carve(*d, n_rows, chunk_items, nullptr).bytes, workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  RECNN_PROPAGATE(discrete_hidden(*d, params, state, n_rows, w.s, st, nullptr));
  RECNN_PROPAGATE(shard_record_init(p, record, n_rows, st));
  return reinforce_stats_pass(*d, params, n_rows, w.s, chunk_items, reinterpret_cast<const long long*>(target), p.lo,
                              shard_plane(record, n_rows, 0), shard_plane(record, n_rows, 1),
                              shard_plane(record, n_rows, 2), st);
}

// the count pass over the rank's block from the gathered stats records, into the rank's count record
static int shard_rank_local(const recnn_discrete_dims& d, const ShardPlan& p, const float* params,
                            const long long* target, int64_t n, const ItemSets& sets, int chunk, const float* gathered,
                            float* record, const RankWorkspace& w, cudaStream_t st) {
  shard_target_logit_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(gathered, n, p.world, w.s.za);
  RECNN_CHECK_LAUNCH("shard_target_logit_kernel");
  rank_record_init_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, st>>>(record, n, p);
  RECNN_CHECK_LAUNCH("rank_record_init_kernel");
  return rank_count_pass(d, params, n, w.s, chunk, p.lo, p.items, target, w.s.za, sets,
                         reinterpret_cast<int*>(shard_plane(record, n, 0)), st);
}

extern "C" int recnn_discrete_shard_rank(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                         const int64_t* target, int64_t n_rows, int32_t chunk_items,
                                         const float* gathered, float* record, void* workspace,
                                         int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && target && gathered && record && workspace, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  RECNN_PROPAGATE(check_workspace(rank_carve(*d, n_rows, chunk_items, nullptr).bytes, workspace_bytes));
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  const ItemSets none = {nullptr, nullptr, nullptr, 0, 0, 0};
  return shard_rank_local(*d, p, params, reinterpret_cast<const long long*>(target), n_rows, none, chunk_items,
                          gathered, record, w, static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_discrete_shard_rank_sets(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                              const float* params, const int64_t* target, int64_t n_rows,
                                              const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                                              int64_t n_sets, const int64_t* row_set, int32_t chunk_items,
                                              const float* gathered, float* record, int32_t* error_flag,
                                              void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && params && target && gathered && record && workspace, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  RECNN_REQUIRE(chunk_ok(d->num_items, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  RECNN_PROPAGATE(check_workspace(rank_carve(*d, n_rows, chunk_items, nullptr).bytes, workspace_bytes));
  ItemSets sets;
  RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n_rows, error_flag, &sets));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(item_sets_check(sets, n_rows, p.items, error_flag, st));   // global ids: every rank agrees
  return shard_rank_local(*d, p, params, reinterpret_cast<const long long*>(target), n_rows, sets, chunk_items,
                          gathered, record, w, st);
}

extern "C" int recnn_discrete_shard_rank_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                                const float* gathered_stats, const float* gathered_counts,
                                                const int64_t* target, int64_t n_rows, int64_t* rank_out,
                                                float* log_prob_out, int32_t* error_flag, void* stream) {
  RECNN_REQUIRE(discrete_dims_ok(d) && gathered_stats && gathered_counts && target && rank_out && log_prob_out &&
                    error_flag, "null pointer / dims");
  ShardPlan p;
  RECNN_PROPAGATE(shard_plan(d->num_items, v, &p));
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  shard_rank_finish_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(
      gathered_stats, gathered_counts, n_rows, p, reinterpret_cast<const long long*>(target),
      reinterpret_cast<long long*>(rank_out), log_prob_out, error_flag);
  RECNN_CHECK_LAUNCH("shard_rank_finish_kernel");
  return RECNN_OK;
}

// ---- log-probs of given items (off-policy estimation) ---------------------------------------------------------
extern "C" int recnn_discrete_log_prob(const recnn_discrete_dims* d, const float* params, const float* state,
                                       const int64_t* action, int64_t n_rows, int32_t chunk_items, float* log_prob_out,
                                       int32_t* error_flag, void* workspace, int64_t workspace_bytes, void* stream) {
  RECNN_REQUIRE(state && log_prob_out, "null pointer");
  RECNN_PROPAGATE(rank_check(d, params, action, n_rows, chunk_items, error_flag, workspace, workspace_bytes));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const RankWorkspace w = rank_carve(*d, n_rows, chunk_items, workspace);
  const long long* act = reinterpret_cast<const long long*>(action);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  RECNN_PROPAGATE(rank_stats_local(*d, params, state, act, n_rows, chunk_items, error_flag, w, st));
  log_prob_finish_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(w.s.za, w.s.run_max, w.s.run_sum, act,
                                                                          n_rows, d->num_items, log_prob_out);
  RECNN_CHECK_LAUNCH("log_prob_finish_kernel");
  return RECNN_OK;
}

extern "C" int recnn_vocab_log_prob_finish(const recnn_vocab_shard* v, const float* gathered, const int64_t* action,
                                           int64_t n_rows, float* log_prob_out, int32_t* error_flag, void* stream) {
  RECNN_REQUIRE(gathered && action && log_prob_out && error_flag, "null pointer");
  RECNN_REQUIRE(v && v->num_items > 0 && v->world >= 1 && v->rank >= 0 && v->rank < v->world &&
                    v->item_offset >= 0 && v->item_offset < v->num_items,
                "shard: rank / world / item_offset outside the vocabulary");
  RECNN_REQUIRE(n_rows > 0, "n_rows");
  const ShardPlan p{v->world, v->rank, v->item_offset, -1, v->num_items};      // hi: from the rank's own header
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  vocab_log_prob_finish_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(
      gathered, n_rows, p, reinterpret_cast<const long long*>(action), log_prob_out, error_flag);
  RECNN_CHECK_LAUNCH("vocab_log_prob_finish_kernel");
  return RECNN_OK;
}
