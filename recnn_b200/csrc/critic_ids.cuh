// REINFORCE critic with item-id actions: the critic half of recnn/nn/update/reinforce.py:92-102 (misc.py:10-55 with a
// DiscreteActor target policy) without any [rows, num_items] matrix.  Included at the end of step.cu after
// reinforce.cuh: it reuses the four contraction helpers, the DiscreteActor layout and the critic-head kernels.
//
// The critic's layer 1 is W1 [H, S + num_items] applied to [state | action].  Its action block W1a = W1[:, S:] is never
// multiplied by a dense matrix:
//   * online critic, action = one-hot(a):   W1a onehot(a) = W1[:, S + a]    -> a gathered [rows, H] addend
//   * target critic, action = softmax(z):   W1a softmax(z) = Y, streamed over item chunks (one pass, online rescaling):
//       per chunk c:  P_c = exp(z_c - M_new),  Y <- Y exp(M_old - M_new) + P_c W1a[:, c]^T,  sum <- ...;  Y /= sum
//   * gradient of the online W1a:            column S + j <- sum over rows m with a_m = j of dz1[m, :]
//     (sort of (id, row) keys, then one ascending-row sum per distinct id: deterministic, no atomics)
// Layer 1 then runs over the state block only (K = S) with the addend in the EPI_HIDDEN epilogue.  Sharded over the
// item vocabulary (recnn_discrete_value_shard_*), each rank computes both terms over the ids it holds and the ranks'
// parts are summed; the rest of the step is the same code.
#pragma once

namespace recnn {

// split count of one chunk's projection GEMM Y_part[rows, H] = P_c W1a_c^T (K = lead + chunk): the [rows, H] output is
// only ceil(rows/128) * ceil(H/128) tiles, so the chunk's K is split to fill the SMs (>= 4 k-blocks of 32 per split).
static int proj_splits(int64_t n, int H, int K) {
  const int64_t tiles = ceil_div(n, 128) * ceil_div(H, 128);
  int64_t s = kNumSMs / tiles;
  const int64_t max_s = ceil_div(K, 32) / 4;
  if (s > max_s) s = max_s;
  return (int)(s < 1 ? 1 : s);
}

struct ProjScratch {
  float *img, *ph;               // policy source: re-pitched state, policy hidden layer [n, Hp]
  float *P;                      // [n, ldP] one chunk, `lead` zero columns in front
  float *run_max, *run_sum, *scale;
  float* partial;                // [splits, n, H]
  long long ldP;
};
static ProjScratch proj_carve(const recnn_dims& cd, const recnn_discrete_dims* pd, int64_t n, int chunk, Carve& c) {
  ProjScratch s;
  const int lead = cd.state_dim % 4;
  s.ldP = pad4(lead + chunk);
  s.img = s.ph = nullptr;
  if (pd) {
    s.img = c.take(n * pad4(pd->state_dim));
    s.ph = c.take(n * pd->hidden);
  }
  s.P = c.take(n * s.ldP);
  s.run_max = c.take(n);
  s.run_sum = c.take(n);
  s.scale = c.take(n);
  s.partial = c.take((int64_t)proj_splits(n, cd.hidden, lead + chunk) * n * cd.hidden);
  return s;
}

// One chunk of logits (columns [lead, lead + w) of each row) -> exp(z - M_new) in place; per row: M, sum of exp and the
// factor exp(M_old - M_new) that rescales the rows of Y accumulated so far (0 on the first chunk).  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
chunk_softmax_fold_kernel(float* __restrict__ P, long long ldP, int lead, long long n, int w, int first,
                          float* __restrict__ run_max, float* __restrict__ run_sum, float* __restrict__ scale) {
  __shared__ float red[32];
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float* row = P + r * ldP + lead;
    float m = -INFINITY;
    for (int j = threadIdx.x; j < w; j += blockDim.x) m = fmaxf(m, row[j]);
    const float M = block_max(m, red);
    const float M0 = first ? -INFINITY : run_max[r];
    const float Mn = fmaxf(M0, M);
    float s = 0.f;
    for (int j = threadIdx.x; j < w; j += blockDim.x) {
      const float e = expf(row[j] - Mn);
      row[j] = e;
      s += e;
    }
    const float S = block_sum(s, red);
    if (threadIdx.x == 0) {
      const float sc = first ? 0.f : expf(M0 - Mn);
      run_sum[r] = (first ? 0.f : run_sum[r] * sc) + S;
      run_max[r] = Mn;
      scale[r] = sc;
    }
    __syncthreads();
  }
}

// Y = (first ? 0 : Y * scale[row]) + sum over splits of part;  then / run_sum[row] on the last chunk (when given).
__global__ void proj_fold_kernel(float* __restrict__ Y, const float* __restrict__ part, int splits, long long n, int H,
                                 const float* __restrict__ scale, const float* __restrict__ run_sum, int first, int last) {
  const long long total = n * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long r = i / H;
    float s = 0.f;
    for (int z = 0; z < splits; ++z) s += part[(long long)z * total + i];
    float y = first ? s : Y[i] * (scale ? scale[r] : 1.f) + s;
    if (last && run_sum) y /= run_sum[r];
    Y[i] = y;
  }
}

static unsigned elem_grid(int64_t count, int threads = 256) {
  const int64_t b = ceil_div(count, threads);
  return (unsigned)(b < (int64_t)kNumSMs * 16 ? b : (int64_t)kNumSMs * 16);
}

// part[z] = P_c[:, 0:K] W[:, 0:K]^T over split z of K (W: the critic's W1 from column S - lead + c0, row pitch ldw)
static int proj_gemm(const float* P, long long ldP, int K, const float* W, long long ldw, int H, int64_t n, int req,
                     float* part, int* splits_out, cudaStream_t st) {
  Epilogue e = base_epi();
  e.out = part; e.ldo = H;
  const bool tc_ok = math_tc() && aligned16(P) && aligned16(W) && ldP % 4 == 0 && ldw % 4 == 0;
  if (tc_ok) {
    tc::Operand a0 = {P, ldP, 0, 0}, a1 = {nullptr, 0, 0, 0}, b = {W, ldw, H, K};
    tc::Problem p;
    memset(&p, 0, sizeof(p));
    p.M = (int)n; p.N = H; p.K0 = K; p.b_k1_offset = K;
    const int r = tc::launch<false, false, EPI_PARTIAL>(a0, a1, b, p, req, H > 64 ? 128 : 64, e, st);
    if (r < 0) return r;
    *splits_out = r;
    return RECNN_OK;
  }
  RECNN_PROPAGATE((launch_gemm_simt<true, true, EPI_PARTIAL>(mat(P, ldP), mat(W, ldw), (int)n, H, K, req, e, st)));
  const int k_chunk = (int)round_up(ceil_div(K, req), 16);        // the launcher's rounding of the split
  *splits_out = (int)ceil_div(K, k_chunk);
  return RECNN_OK;
}

// Y[n, H] = softmax(policy logits) W1a^T (policy source: pparams != null, xs = the policy's input) or probs W1a^T
// (dense source [n, ld_probs]), over item chunks of width W.  normalise = false (policy source only) leaves
// Y = sum exp(z - run_max) W1a^T without the final division by run_sum: a vocabulary shard's part, merged later.
static int action_term_chunked(const recnn_dims& cd, const float* cparams, const recnn_discrete_dims* pd,
                               const float* pparams, const Seg& xs, const float* probs, long long ld_probs, int64_t n,
                               int W, const ProjScratch& s, float* Y, cudaStream_t st, bool normalise = true) {
  const NetLayout lc = critic_layout(cd);
  const int S = cd.state_dim, I = cd.action_dim, H = cd.hidden, lead = S % 4;
  const int n_chunks = (int)ceil_div(I, W);
  if (lead) RECNN_CHECK_CUDA(cudaMemset2DAsync(s.P, (size_t)s.ldP * 4, 0, (size_t)lead * 4, n, st));
  DiscreteLayout lp;
  if (pparams) {
    lp = discrete_layout(*pd);
    Rng rng = {nullptr, 0, nullptr};
    RECNN_PROPAGATE(hidden_layer(xs, kNoSeg, pparams + lp.w1, lp.ld1, pparams + lp.b1, pd->hidden, n, false, nullptr,
                                 rng, 0, s.ph, st));
  }
  for (int c = 0; c < n_chunks; ++c) {
    const int c0 = c * W, w = I - c0 < W ? I - c0 : W;
    if (pparams) {
      const Seg sh = {s.ph, pd->hidden, pd->hidden, 0};
      RECNN_PROPAGATE(linear_out(sh, pparams + lp.w2 + (int64_t)c0 * lp.ld2, lp.ld2, pparams + lp.b2 + c0, w, n, 0,
                                 nullptr, s.P + lead, s.ldP, st));
      chunk_softmax_fold_kernel<<<row_grid(n), kRowThreads, 0, st>>>(s.P, s.ldP, lead, n, w, c == 0, s.run_max,
                                                                      s.run_sum, s.scale);
      RECNN_CHECK_LAUNCH("chunk_softmax_fold_kernel");
    } else {
      RECNN_CHECK_CUDA(cudaMemcpy2DAsync(s.P + lead, (size_t)s.ldP * 4, probs + c0, (size_t)ld_probs * 4, (size_t)w * 4,
                                         n, cudaMemcpyDeviceToDevice, st));
    }
    int splits = 1;
    const int K = lead + w;
    RECNN_PROPAGATE(proj_gemm(s.P, s.ldP, K, cparams + lc.w1 + (S - lead) + c0, lc.ld1, H, n, proj_splits(n, H, K),
                              s.partial, &splits, st));
    proj_fold_kernel<<<elem_grid(n * H), 256, 0, st>>>(Y, s.partial, splits, n, H, pparams ? s.scale : nullptr,
                                                       pparams && normalise ? s.run_sum : nullptr, c == 0,
                                                       c == n_chunks - 1);
    RECNN_CHECK_LAUNCH("proj_fold_kernel");
  }
  return RECNN_OK;
}

// add[m, :] = W1[:, S + a_m - lo] (the one-hot product) when a_m is one of the `items` ids [lo, lo + items) whose
// columns this arena holds, else a zero row; an id outside [0, num_items) flags *oob.  Unsharded: lo 0, items ==
// num_items.
__global__ void gather_action_columns_kernel(const float* __restrict__ w1, long long ld1, int S, int H, int lo,
                                             int items, int num_items, const long long* __restrict__ action,
                                             long long n, float* __restrict__ add, unsigned* oob) {
  const long long total = n * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / H;
    const int h = (int)(i - m * H);
    const long long a = action[m];
    const long long j = a - lo;
    add[i] = (j >= 0 && j < items) ? __ldg(w1 + (long long)h * ld1 + S + j) : 0.f;
    if ((a < 0 || a >= num_items) && h == 0) *oob = 1u;
  }
}

// keys[i] = (id - lo << 32) | row for i < n (an id outside the arena's block [lo, lo + items) sorts last as
// 0xFFFFFFFF and is skipped), UINT64_MAX in the padding
__global__ void action_keys_kernel(const long long* __restrict__ action, long long n, long long n2, int lo, int items,
                                   unsigned long long* __restrict__ keys) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    if (i < n) {
      const long long j = action[i] - lo;
      const unsigned long long id = (j >= 0 && j < items) ? (unsigned long long)j : 0xFFFFFFFFull;
      keys[i] = (id << 32) | (unsigned long long)i;
    } else {
      keys[i] = ~0ull;
    }
  }
}

// one compare-exchange stage (k, j) of a bitonic sort of n2 (a power of two) distinct keys, ascending
__global__ void bitonic_step_kernel(unsigned long long* __restrict__ keys, long long n2, long long j, long long k) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n2; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i ^ j;
    if (p > i) {
      const unsigned long long a = keys[i], b = keys[p];
      if ((a > b) == ((i & k) == 0)) {
        keys[i] = b;
        keys[p] = a;
      }
    }
  }
}

// gw1a[h * ld1 + j] = sum over the rows m with id j, ascending, of dz1[m, h].  One CTA per run of equal ids in the
// sorted keys (the CTA at the run's first position); a column no row selected is left as it is (zeroed before).
__global__ void scatter_action_grad_kernel(const unsigned long long* __restrict__ keys, long long n,
                                           const float* __restrict__ dz1, int H, float* __restrict__ gw1a, long long ld1) {
  for (long long i = blockIdx.x; i < n; i += gridDim.x) {
    const unsigned id = (unsigned)(keys[i] >> 32);
    if (id == 0xFFFFFFFFu || (i > 0 && (unsigned)(keys[i - 1] >> 32) == id)) continue;
    long long end = i + 1;
    while (end < n && (unsigned)(keys[end] >> 32) == id) ++end;
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      float s = 0.f;
      for (long long t = i; t < end; ++t) s += dz1[(long long)(keys[t] & 0xFFFFFFFFull) * H + h];
      gw1a[(long long)h * ld1 + id] = s;
    }
  }
}

// Vocabulary-sharded critic, after the all-gather of the records: terms[0] = Y_r exp(m_r - M) / S (this rank's part of
// the target action term, merged in rank order as shard_merge_row does for the policy) and terms[1] = add_r.  At W = 1
// the factor is exp(0) = 1 and S = s_0, and the division is proj_fold_kernel's: the unsharded bits.  One CTA per row.
__global__ void __launch_bounds__(kRowThreads)
critic_shard_merge_kernel(const float* __restrict__ g, long long n, ShardPlan p, const float* __restrict__ local_max,
                          const float* __restrict__ Y, const float* __restrict__ add, int H, float* __restrict__ terms,
                          unsigned* plan_bad) {
  if (blockIdx.x == 0 && threadIdx.x == 0 && shard_plan_bad(g, shard_record_floats(n), p, n)) *plan_bad = 1u;
  for (long long r = blockIdx.x; r < n; r += gridDim.x) {
    float M, S, za;
    shard_merge_row(g, p.world, n, r, M, S, za);
    const float f = expf(local_max[r] - M);
    for (int h = threadIdx.x; h < H; h += blockDim.x) {
      const long long i = r * H + h;
      float y = Y[i] * f;
      y /= S;
      terms[i] = y;
      terms[n * H + i] = add[i];
    }
  }
}

static int64_t pow2_at_least(int64_t n) {
  int64_t p = 1;
  while (p < n) p <<= 1;
  return p;
}

// ---------------------------------------------------------------- the critic step with item-id actions
struct DvWorkspace {
  float *S, *S2;                              // [n, ldS] state images
  float *c1, *c2, *dz2, *dz1, *t1, *t2, *add, *Y;   // [n, H]
  float *y, *qtmp, *dq;                       // [n]
  float* partial;
  float* block_partials;
  unsigned* tickets;
  unsigned long long* keys;                   // [pow2(n)]
  ProjScratch proj;
  int64_t bytes;
};

static DvWorkspace dv_carve(const recnn_dims& d, const recnn_discrete_dims& pd, int64_t n, int chunk, void* base) {
  DvWorkspace w;
  Carve c(base);
  const int ldS = pad4(d.state_dim), H = d.hidden;
  w.S = c.take(n * ldS);
  w.S2 = c.take(n * ldS);
  float** hb[8] = {&w.c1, &w.c2, &w.dz2, &w.dz1, &w.t1, &w.t2, &w.add, &w.Y};
  for (auto b : hb) *b = c.take(n * H);
  w.y = c.take(n);
  w.qtmp = c.take(n);
  w.dq = c.take(n);
  int64_t part = head_partial_floats(H, n);
  const int shapes[3][2] = {{H, d.state_dim}, {H, H}, {1, H}};
  for (auto& s : shapes) part = std::max(part, dw_partial_floats(s[0], s[1], n));
  w.partial = c.take(part);
  w.block_partials = c.take(1024);
  w.tickets = c.take<unsigned>(8);
  w.keys = c.take<unsigned long long>(pow2_at_least(n));
  w.proj = proj_carve(d, &pd, n, chunk, c);
  w.bytes = c.bytes();
  return w;
}

static bool dv_dims_ok(const recnn_dims& d, const recnn_discrete_dims& pd) {
  return d.state_dim > 0 && d.hidden > 0 && d.action_dim > 0 && pd.hidden > 0 && pd.state_dim == d.state_dim &&
         pd.num_items == d.action_dim;
}

}  // namespace recnn

using namespace recnn;

extern "C" int64_t recnn_critic_action_term_scratch_floats(const recnn_dims* d, const recnn_discrete_dims* pd,
                                                           int64_t n_rows, int32_t chunk_items) {
  if (!d || n_rows <= 0 || d->state_dim <= 0 || d->hidden <= 0 || !chunk_ok(d->action_dim, chunk_items)) return 0;
  Carve c(nullptr);
  proj_carve(*d, pd, n_rows, chunk_items, c);
  return c.floats();
}

extern "C" int recnn_critic_action_term_chunked(const recnn_dims* d, const float* critic_params,
                                                const recnn_discrete_dims* pd, const float* policy_params,
                                                const float* state, const float* probs, int64_t probs_ld,
                                                int64_t n_rows, int32_t chunk_items, float* out, float* scratch,
                                                void* stream) {
  RECNN_REQUIRE(d && critic_params && out && scratch, "null pointer");
  RECNN_REQUIRE(d->state_dim > 0 && d->hidden > 0 && d->action_dim > 0, "dims");
  RECNN_REQUIRE((policy_params != nullptr) != (probs != nullptr), "give a policy (policy_params, state) or probs");
  RECNN_REQUIRE(!policy_params || (pd && state && dv_dims_ok(*d, *pd)), "policy dims / state");
  RECNN_REQUIRE(!probs || probs_ld >= d->action_dim, "probs_ld");
  RECNN_REQUIRE(chunk_ok(d->action_dim, chunk_items), "chunk_items must be num_items or a positive multiple of 128 below it");
  if (n_rows <= 0) return RECNN_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  Carve c(scratch);
  const ProjScratch s = proj_carve(*d, policy_params ? pd : nullptr, n_rows, chunk_items, c);
  Seg xs = kNoSeg;
  if (policy_params) RECNN_PROPAGATE(repitch_state(pd->state_dim, state, n_rows, s.img, &xs, st));
  return action_term_chunked(*d, critic_params, pd, policy_params, xs, probs, probs_ld, n_rows, chunk_items, s, out, st);
}

extern "C" int recnn_critic_forward_action_term(const recnn_dims* d, const float* params, const float* state,
                                                const float* action_term, int64_t n_rows, const uint8_t* mask1,
                                                const uint8_t* mask2, float* value_out, float* scratch, void* stream) {
  RECNN_REQUIRE(d && params && state && action_term && value_out && scratch, "null pointer");
  RECNN_REQUIRE((mask1 == nullptr) == (mask2 == nullptr), "give both masks or neither");
  if (n_rows <= 0) return RECNN_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const NetLayout l = critic_layout(*d);
  const int H = d->hidden;
  const ForwardScratch s = forward_carve(*d, n_rows, false, scratch);
  Rng rng = {nullptr, 0, nullptr};
  const bool train = mask1 != nullptr;
  Seg xs;
  RECNN_PROPAGATE(repitch_state(d->state_dim, state, n_rows, s.img, &xs, st));
  const Seg s1 = {s.h1, H, H, 0};
  RECNN_PROPAGATE(hidden_layer(xs, kNoSeg, params + l.w1, l.ld1, params + l.b1, H, n_rows, train, mask1, rng, 0, s.h1,
                               st, action_term));
  RECNN_PROPAGATE(hidden_layer(s1, kNoSeg, params + l.w2, l.ld2, params + l.b2, H, n_rows, train, mask2, rng, 1, s.h2, st));
  HeadArgs h;
  memset(&h, 0, sizeof(h));
  h.h2 = s.h2; h.w3 = params + l.w3; h.b3 = params + l.b3; h.n_rows = n_rows; h.n_rows_global = n_rows;
  h.hidden = H; h.mode = HEAD_PLAIN; h.out = value_out;
  return launch_critic_head(h, st);
}

extern "C" int64_t recnn_discrete_value_workspace_bytes(const recnn_dims* d, const recnn_discrete_dims* pd,
                                                        int64_t n_rows, int32_t chunk_items) {
  if (!d || !pd || n_rows <= 0 || !dv_dims_ok(*d, *pd) || !chunk_ok(d->action_dim, chunk_items)) return 0;
  return dv_carve(*d, *pd, n_rows, chunk_items, nullptr).bytes;
}

extern "C" int64_t recnn_sizeof_discrete_value_args(void) { return (int64_t)sizeof(recnn_discrete_value_args); }

// The argument checks of the step and of its sharded phases (dims are the arena's: local ones on a shard); *w <- the
// carved workspace.
static int dv_check(const recnn_discrete_value_args* a, DvWorkspace* w) {
  RECNN_REQUIRE(a != nullptr, "args");
  RECNN_REQUIRE(dv_dims_ok(a->dims, a->policy_dims), "dims (critic action_dim == policy num_items, equal state_dim)");
  RECNN_REQUIRE(a->n_rows > 0, "n_rows");
  const int S = a->dims.state_dim, H = a->dims.hidden;
  RECNN_REQUIRE(chunk_ok(a->dims.action_dim, a->chunk_items),
                "chunk_items must be num_items or a positive multiple of 128 below it");
  int64_t widest = pad4(S) > H ? pad4(S) : H;
  if (pad4(S % 4 + a->chunk_items) > widest) widest = pad4(S % 4 + a->chunk_items);
  RECNN_REQUIRE(a->n_rows < (1ll << 31) / (widest + 1), "n_rows too large for int32 tile indexing");
  RECNN_REQUIRE(a->state && a->next_state && a->action && a->reward && a->done, "batch");
  RECNN_REQUIRE(a->value.params && a->target_value.params && a->target_policy, "nets");
  RECNN_REQUIRE(!a->learn || a->value.grads, "value net needs a grad arena when learn=1");
  RECNN_REQUIRE(a->losses && a->workspace && a->rng_step, "losses / workspace / rng_step");
  RECNN_REQUIRE((a->masks[0] == nullptr) == (a->masks[1] == nullptr), "give both masks or neither");
  *w = dv_carve(a->dims, a->policy_dims, a->n_rows, a->chunk_items, a->workspace);
  return check_workspace(w->bytes, a->workspace_bytes);
}

// The action terms of layer 1: the error tickets zeroed, the state images, then
//   w.Y   = next_action = target_policy_net(next_state) (misc.py:28), consumed only as W1a' next_action -- without its
//           division by the row sums (normalise = false) on a vocabulary shard;
//   w.add = W1a one-hot(action) (misc.py:37) over the ids [lo, lo + action_dim) this arena holds.
static int dv_action_terms(const recnn_discrete_value_args* a, const DvWorkspace& w, int lo, int num_items,
                           bool normalise, cudaStream_t st) {
  const recnn_dims& d = a->dims;
  const int S = d.state_dim, H = d.hidden, ldS = pad4(S);
  const int64_t n = a->n_rows;
  const NetLayout lc = critic_layout(d);
  RECNN_CHECK_CUDA(cudaMemsetAsync(w.tickets, 0, 8 * sizeof(unsigned), st));
  RECNN_CHECK_CUDA(cudaMemcpy2DAsync(w.S, (size_t)ldS * 4, a->state, (size_t)S * 4, (size_t)S * 4, n,
                                     cudaMemcpyDeviceToDevice, st));
  RECNN_CHECK_CUDA(cudaMemcpy2DAsync(w.S2, (size_t)ldS * 4, a->next_state, (size_t)S * 4, (size_t)S * 4, n,
                                     cudaMemcpyDeviceToDevice, st));
  const Seg ss2 = {w.S2, S, ldS, 0};
  RECNN_PROPAGATE(action_term_chunked(d, a->target_value.params, &a->policy_dims, a->target_policy, ss2, nullptr, 0, n,
                                      a->chunk_items, w.proj, w.Y, st, normalise));
  gather_action_columns_kernel<<<elem_grid(n * H), 256, 0, st>>>(a->value.params + lc.w1, lc.ld1, S, H, lo, d.action_dim,
                                                                 num_items, reinterpret_cast<const long long*>(a->action),
                                                                 n, w.add, w.tickets + kTicketOob);
  RECNN_CHECK_LAUNCH("gather_action_columns_kernel");
  return RECNN_OK;
}

// misc.py:29-44 from the action terms Y and add on, in the reference's order: target critic -> TD target (clamped),
// online critic, MSE, backward, optimizer.  lo: the global id of the arena's first action column (0 unsharded).
static int dv_tail(const recnn_discrete_value_args* a, const DvWorkspace& w, const float* Y, const float* add, int lo,
                   cudaStream_t st) {
  const recnn_dims& d = a->dims;
  const int S = d.state_dim, I = d.action_dim, H = d.hidden;
  const int64_t n = a->n_rows;
  const NetLayout lc = critic_layout(d);
  const int ldS = pad4(S);
  const bool train = a->dropout != 0;
  const float gate = train ? 2.0f : 1.0f;
  Rng rng = {nullptr, a->seed, (const long long*)a->rng_step};
  const long long* act = reinterpret_cast<const long long*>(a->action);
  unsigned* oob = w.tickets + kTicketOob;
  const Seg ss = {w.S, S, ldS, 0}, ss2 = {w.S2, S, ldS, 0};
  const float* Pt = a->target_value.params;
  const float* P = a->value.params;
  // target critic, eval mode (misc.py:29)
  const Seg st1 = {w.t1, H, H, 0};
  RECNN_PROPAGATE(hidden_layer(ss2, kNoSeg, Pt + lc.w1, lc.ld1, Pt + lc.b1, H, n, false, nullptr, rng, 0, w.t1, st, Y));
  RECNN_PROPAGATE(hidden_layer(st1, kNoSeg, Pt + lc.w2, lc.ld2, Pt + lc.b2, H, n, false, nullptr, rng, 1, w.t2, st));
  // online critic on (state, one-hot(action)) (misc.py:37)
  const Seg sc1 = {w.c1, H, H, 0};
  RECNN_PROPAGATE(hidden_layer(ss, kNoSeg, P + lc.w1, lc.ld1, P + lc.b1, H, n, train, train ? a->masks[0] : nullptr, rng,
                               0, w.c1, st, add));
  RECNN_PROPAGATE(hidden_layer(sc1, kNoSeg, P + lc.w2, lc.ld2, P + lc.b2, H, n, train, train ? a->masks[1] : nullptr, rng,
                               1, w.c2, st));
  // TD target and clamp (misc.py:30-35), MSE (:39), its gradient through the head
  float* G = a->value.grads;
  if (value_head_fusable(H)) {
    ValueHeadArgs v;
    memset(&v, 0, sizeof(v));
    v.h2 = w.c2; v.w3 = P + lc.w3; v.b3 = P + lc.b3;
    v.th2 = w.t2; v.tw3 = Pt + lc.w3; v.tb3 = Pt + lc.b3;
    v.reward = a->reward; v.done = a->done;
    v.gamma = a->gamma; v.min_value = a->min_value; v.max_value = a->max_value;
    v.y = w.y; v.n_rows = n; v.n_rows_global = n; v.hidden = H;
    v.learn = a->learn ? 1 : 0; v.gate_scale = gate; v.dz2 = w.dz2;
    v.gw3 = a->learn ? G + lc.w3 : nullptr; v.gb3 = a->learn ? G + lc.b3 : nullptr;
    v.loss = a->losses;
    v.block_partials = w.partial;
    v.ticket = w.tickets + 2;
    RECNN_PROPAGATE(launch_value_head_fused(v, st));
  } else {
    HeadArgs h;
    memset(&h, 0, sizeof(h));
    h.w3 = Pt + lc.w3; h.b3 = Pt + lc.b3; h.h2 = w.t2;
    h.n_rows = n; h.n_rows_global = n; h.hidden = H; h.mode = HEAD_TARGET_DDPG;
    h.reward = a->reward; h.done = a->done; h.gamma = a->gamma; h.min_value = a->min_value; h.max_value = a->max_value;
    h.y = w.y; h.tmp = w.qtmp; h.dq = w.dq; h.block_partials = w.block_partials; h.ticket = w.tickets;
    RECNN_PROPAGATE(launch_critic_head(h, st));
    h.w3 = P + lc.w3; h.b3 = P + lc.b3; h.h2 = w.c2; h.mode = HEAD_VALUE; h.loss = a->losses;
    RECNN_PROPAGATE(launch_critic_head(h, st));
    if (a->learn) {
      const int splits = (int)ceil_div(n, kHeadGradRowsPerSplit);
      RECNN_PROPAGATE(launch_head_grad_partials(w.dq, w.c2, n, H, kHeadGradRowsPerSplit, splits, w.partial, st));
      RECNN_PROPAGATE(launch_reduce_partials(w.partial, splits, 1, H + 1, G + lc.w3, lc.ld3, G + lc.b3, st));
      RECNN_PROPAGATE(launch_critic_head_bwd(w.dq, 0.f, P + lc.w3, w.c2, gate, w.dz2, n, H, st));
    }
  }
  if (a->learn) {
    // layers 2 and 1 (state block) through the dense weight gradients, each reduced here; then the action block
    RECNN_PROPAGATE(weight_grad(w.dz2, H, sc1, kNoSeg, n, G + lc.w2, lc.ld2, G + lc.b2, w.partial, st));
    RECNN_PROPAGATE(backprop_hidden(w.dz2, H, P + lc.w2, lc.ld2, H, 0, H, n, w.c1, gate, w.dz1, st));
    RECNN_PROPAGATE(weight_grad(w.dz1, H, ss, kNoSeg, n, G + lc.w1, lc.ld1, G + lc.b1, w.partial, st));
    RECNN_CHECK_CUDA(cudaMemset2DAsync(G + lc.w1 + S, (size_t)lc.ld1 * 4, 0, (size_t)I * 4, H, st));
    const int64_t n2 = pow2_at_least(n);
    action_keys_kernel<<<elem_grid(n2), 256, 0, st>>>(act, n, n2, lo, I, w.keys);
    RECNN_CHECK_LAUNCH("action_keys_kernel");
    for (int64_t k = 2; k <= n2; k <<= 1)
      for (int64_t j = k >> 1; j > 0; j >>= 1) {
        bitonic_step_kernel<<<elem_grid(n2), 256, 0, st>>>(w.keys, n2, j, k);
        RECNN_CHECK_LAUNCH("bitonic_step_kernel");
      }
    const unsigned blocks = (unsigned)(n < (int64_t)kNumSMs * 16 ? n : (int64_t)kNumSMs * 16);
    scatter_action_grad_kernel<<<blocks, H < 256 ? 128 : 256, 0, st>>>(w.keys, n, w.dz1, H, G + lc.w1 + S, lc.ld1);
    RECNN_CHECK_LAUNCH("scatter_action_grad_kernel");
    if (a->value_optim.kind != RECNN_OPT_EXTERNAL)
      RECNN_PROPAGATE(launch_optimizer(a->value_optim, a->value, lc.count, nullptr, st, w.tickets + 3));
  }
  // ++rng_step; losses[4] <- error bits (1: an action id outside [0, num_items): its row read a zero action column and
  // its gradient column was skipped; 2: the gathered shard records disagree with the plan)
  RECNN_PROPAGATE(launch_finish((long long*)a->rng_step, oob, w.tickets + kTicketDpMismatch, a->losses + 4, st));
  if (a->losses_host)
    RECNN_CHECK_CUDA(cudaMemcpyAsync(a->losses_host, a->losses, 8 * sizeof(float), cudaMemcpyDeviceToHost, st));
  return RECNN_OK;
}

// misc.py:10-55: the action terms, then the rest.  Everything on `stream`, no allocation, no synchronisation.
extern "C" int recnn_discrete_value_step(const recnn_discrete_value_args* a, void* stream) {
  DvWorkspace w;
  RECNN_PROPAGATE(dv_check(a, &w));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_PROPAGATE(dv_action_terms(a, w, 0, a->dims.action_dim, true, st));
  return dv_tail(a, w, w.Y, w.add, 0, st);
}

// ---- the vocabulary-sharded critic: the phases around the all-gather and the all-reduce (see the header) ---------
static int dv_shard_check(const recnn_discrete_value_args* a, const recnn_vocab_shard* v, DvWorkspace* w,
                          ShardPlan* p) {
  RECNN_PROPAGATE(dv_check(a, w));
  return shard_plan(a->policy_dims.num_items, v, p);
}

extern "C" int recnn_discrete_value_shard_begin(const recnn_discrete_value_args* a, const recnn_vocab_shard* v,
                                                float* record, void* stream) {
  DvWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(dv_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(record != nullptr, "record");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = a->n_rows;
  RECNN_PROPAGATE(dv_action_terms(a, w, p.lo, p.items, false, st));
  RECNN_PROPAGATE(shard_record_init(p, record, n, st));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(shard_plane(record, n, 0), w.proj.run_max, n * sizeof(float),
                                   cudaMemcpyDeviceToDevice, st));
  RECNN_CHECK_CUDA(cudaMemcpyAsync(shard_plane(record, n, 1), w.proj.run_sum, n * sizeof(float),
                                   cudaMemcpyDeviceToDevice, st));
  return RECNN_OK;
}

extern "C" int recnn_discrete_value_shard_merge(const recnn_discrete_value_args* a, const recnn_vocab_shard* v,
                                                const float* gathered, float* terms, void* stream) {
  DvWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(dv_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(gathered && terms, "gathered / terms");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t n = a->n_rows;
  critic_shard_merge_kernel<<<row_grid(n), kRowThreads, 0, st>>>(gathered, n, p, w.proj.run_max, w.Y, w.add,
                                                                  a->dims.hidden, terms, w.tickets + kTicketDpMismatch);
  RECNN_CHECK_LAUNCH("critic_shard_merge_kernel");
  return RECNN_OK;
}

extern "C" int recnn_discrete_value_shard_end(const recnn_discrete_value_args* a, const recnn_vocab_shard* v,
                                              const float* terms, void* stream) {
  DvWorkspace w;
  ShardPlan p;
  RECNN_PROPAGATE(dv_shard_check(a, v, &w, &p));
  RECNN_REQUIRE(terms != nullptr, "terms");
  return dv_tail(a, w, terms, terms + a->n_rows * a->dims.hidden, p.lo, static_cast<cudaStream_t>(stream));
}
