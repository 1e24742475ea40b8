// Serving through the DDPG / TD3 critic (the Wolpertinger policy, PAPERS.md): score items by Q(s_r, e_j) and keep the
// k best per row, or count the items that beat a row's target.  Included at the end of step.cu: every contraction goes
// through gemm_nt (hidden_layer / linear_out), so RECNN_B200_MATH=simt reaches it like the update step.
//
// Layer 1 is linear in [state | action], so the work splits (eval mode: no dropout):
//   u_r = W1[:, :S] s_r + b1                 once per row                 [N, H]
//   v_j = W1[:, S-lead : S+A] [0^lead | e_j]  once per item (or candidate)  [., H]
//   h1  = relu(u_r + v_j)                    pair kernel                  [pairs, H]
//   h2  = relu(W2 h1 + b2)                   layer 2 (EPI_HIDDEN), M = pairs
//   q   = w3 . h2 + b3                       one warp per pair
// then a top-k select (topk.cuh's register lists, running per-row lists across chunks) or a count of beaters.
//
// A block is nr rows x w columns of the call.  A column is an item id: c0 + j over the whole table, or cand[r, c0 + j]
// of a row's candidates (-1: padding).  Every pair's arithmetic is the same code at every position (the GEMMs run with
// split-K 1 and one back end per call), so Q of a pair is the same bits at any chunk width, in either mode and whatever
// other rows share the call: rank equals the position in topk, and the two modes agree on a pair.
#pragma once

namespace recnn {

constexpr int kServeSplitsMax = 31;      // column ranges per row of a select: lane 31 of the merge holds the running list
constexpr int kServeCandRepeat = 8;      // error bit: an id repeated within a row's candidates

// pairs of one block: h1 and h2 [pairs, H] together in 32 MB of the 50 MB L2 (slab_rows' reasoning in retrieval.cu),
// so layer 2 reads h1 and the score kernel reads h2 from L2
static int64_t serve_pairs(int H) {
  int64_t p = (32ll << 20) / ((int64_t)H * 8);
  p = p / 128 * 128;
  return p < 128 ? 128 : (p > 65536 ? 65536 : p);
}

// columns per chunk: `chunk` (0: 4096), at most the call's width.  Does not depend on the width beyond that cap, so an
// all-items call's workspace stops growing with the table at 4096 items.
static int serve_chunk(int64_t width, int chunk) {
  const int64_t c = chunk > 0 ? chunk : 4096;
  return (int)(c < width ? c : width);
}

struct ServePlan {
  int S, A, H, lead, k;
  long long ldS, ldE;
  int64_t n, width;      // rows; columns of the call (candidates per row, or n_items)
  int C;                 // columns per chunk
  int64_t R;             // rows per block: R * C pairs
};

static ServePlan serve_plan(const recnn_dims& d, int64_t n, int64_t width, int k, int chunk) {
  ServePlan p;
  p.S = d.state_dim; p.A = d.action_dim; p.H = d.hidden; p.lead = p.S % 4; p.k = k;
  p.ldS = pad4(p.S);
  p.ldE = pad4(p.A + p.lead);
  p.n = n; p.width = width;
  p.C = serve_chunk(width, chunk);
  int64_t R = serve_pairs(p.H) / p.C;
  p.R = R < 1 ? 1 : (R > n ? n : R);
  return p;
}

struct ServeWs {
  float *img, *u;        // state image [n, ldS]; row term [n, H]
  float *E, *v;          // staged embeddings [R*C, ldE] (`lead` zero columns in front); item term [R*C, H]
  float *h1, *h2, *q;    // one block: [R*C, H], [R*C, H], [R*C]
  float* qt;             // rank: Q of each row's target [n]
  int* present;          // rank with candidates: the target is among the row's candidates [n]
  Cand *part, *run;      // topk: [R, splits, k] of one block; the running lists [n, k]
  int64_t bytes;
};

// k > 0: a topk call, k == 0: a rank call
static ServeWs serve_carve(const ServePlan& p, void* base) {
  ServeWs w;
  Carve c(base);
  const int64_t V = p.R * p.C;
  w.img = c.take(p.n * p.ldS);
  w.u = c.take(p.n * p.H);
  w.E = c.take(V * p.ldE);
  w.v = c.take(V * p.H);
  w.h1 = c.take(V * p.H);
  w.h2 = c.take(V * p.H);
  w.q = c.take(V);
  w.qt = p.k == 0 ? c.take(p.n) : nullptr;
  w.present = p.k == 0 ? c.take<int>(p.n) : nullptr;
  w.part = p.k > 0 ? c.take<Cand>(p.R * kServeSplitsMax * p.k) : nullptr;
  w.run = p.k > 0 ? c.take<Cand>(p.n * p.k) : nullptr;
  w.bytes = c.bytes();
  return w;
}

// the item of column j of row r in a block: c0 + j over the whole table, else the row's candidate (-1: padding)
__device__ __forceinline__ long long serve_id(const long long* __restrict__ ids, long long ld_ids, long long r,
                                              long long col) {
  return ids ? __ldg(ids + r * ld_ids + col) : col;
}

// smaller is better: -Q, a NaN or -inf Q as FLT_MAX (finite_key, as metric_key)
__device__ __forceinline__ float serve_key(float q) { return finite_key(-q); }

// One CTA per row of the candidates: *flag |= 1 for an id outside [-1, items), |= kServeCandRepeat for an id that
// appears twice in the row (the row is compared with itself tile by tile in shared memory: O(M^2) compares, cheap next
// to the M H^2 of the row's layer 2).  target: present[r] = the row's target is one of its candidates.
static __global__ void __launch_bounds__(256)
serve_cand_check_kernel(const long long* __restrict__ cand, int M, long long items, const long long* __restrict__ target,
                        int* __restrict__ present, int* flag) {
  constexpr int kTile = 2048;
  __shared__ long long s[kTile];
  __shared__ int s_bits;
  const long long r = blockIdx.x;
  const long long* row = cand + r * M;
  const long long t = target ? target[r] : -2;
  if (threadIdx.x == 0) s_bits = 0;
  int bits = 0;
  for (int j = threadIdx.x; j < M; j += blockDim.x) {
    const long long x = row[j];
    if (x < -1 || x >= items) bits |= 1;
    if (x >= 0 && x == t) bits |= 16;                       // 16: local only, the target was found
  }
  for (int t0 = 0; t0 < M; t0 += kTile) {
    const int tn = M - t0 < kTile ? M - t0 : kTile;
    __syncthreads();
    for (int i = threadIdx.x; i < tn; i += blockDim.x) s[i] = row[t0 + i];
    __syncthreads();
    for (int j = threadIdx.x; j < M; j += blockDim.x) {
      const long long x = row[j];
      if (x < 0 || j <= t0) continue;
      const int lim = j - t0 < tn ? j - t0 : tn;            // earlier columns only: each pair is compared once
      for (int i = 0; i < lim; ++i)
        if (s[i] == x) { bits |= kServeCandRepeat; break; }
    }
  }
  if (bits) atomicOr(&s_bits, bits);
  __syncthreads();
  if (threadIdx.x == 0) {
    if (s_bits & (1 | kServeCandRepeat)) atomicOr(flag, s_bits & (1 | kServeCandRepeat));
    if (present) present[r] = (s_bits & 16) != 0;
  }
}

// E[p, :] = [0^lead | table[id] | 0...] for the pairs p = rr * w + j of rows r0 .. r0 + nr, columns c0 .. c0 + w; an id
// outside [0, items) (padding, or a malformed list the check reports) stages a zero row.  One warp per pair.
static __global__ void __launch_bounds__(256)
serve_stage_kernel(const float* __restrict__ table, long long items, int A, const long long* __restrict__ ids,
                   long long ld_ids, long long c0, int w, long long r0, long long nr, int lead, long long ldE,
                   float* __restrict__ E) {
  const long long np = nr * w;
  const int lane = threadIdx.x & 31;
  for (long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < np;
       p += (long long)gridDim.x * (blockDim.x >> 5)) {
    const long long rr = p / w, j = p - rr * w;
    const long long id = serve_id(ids, ld_ids, r0 + rr, c0 + j);
    const bool ok = id >= 0 && id < items;
    const float* src = table + (ok ? id : 0) * A;
    float* dst = E + p * ldE;
    for (long long a = lane; a < ldE; a += 32) {
      const long long e = a - lead;
      dst[a] = (ok && e >= 0 && e < A) ? __ldg(src + e) : 0.f;
    }
  }
}

// h1[p, :] = relu(u[r0 + p / w, :] + v[vrow, :]), vrow = p (one staged row per pair) or p % w (one per column)
static __global__ void __launch_bounds__(256)
serve_pair_kernel(const float* __restrict__ u, const float* __restrict__ v, long long r0, long long nr, int w,
                  int v_per_pair, int H, float* __restrict__ h1) {
  const long long total = nr * w * H;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i / H;
    const int h = (int)(i - p * H);
    const long long rr = p / w;
    const long long vrow = v_per_pair ? p : p - rr * w;
    h1[i] = fmaxf(__ldg(u + (r0 + rr) * H + h) + __ldg(v + vrow * H + h), 0.f);
  }
}

// q[(p / w) * ldq + p % w] = w3 . h2[p, :] + b3, one warp per pair in a fixed order (lane-strided FMAs, then the
// butterfly sum): the same bits for a pair at any position
static __global__ void __launch_bounds__(256)
serve_score_kernel(const float* __restrict__ h2, long long np, int H, const float* __restrict__ w3,
                   const float* __restrict__ b3, int w, long long ldq, float* __restrict__ q) {
  const int lane = threadIdx.x & 31;
  for (long long p = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); p < np;
       p += (long long)gridDim.x * (blockDim.x >> 5)) {
    const float* row = h2 + p * H;
    float s = 0.f;
    for (int h = lane; h < H; h += 32) s = fmaf(row[h], __ldg(w3 + h), s);
    s = warp_sum(s);
    if (lane == 0) {
      const long long rr = p / w;
      q[rr * ldq + (p - rr * w)] = s + __ldg(b3);
    }
  }
}

// grid (splits, nr): the k best (key, id) of row r0 + y over its share of the block's w columns -> part, ascending.  With
// SETS the row's excluded set is tested only for a candidate that would enter a thread's list.
template <int KMAX, bool SETS>
__global__ void __launch_bounds__(kTopkThreads)
serve_topk_kernel(const float* __restrict__ q, long long ldq, const long long* __restrict__ ids, long long ld_ids,
                  long long c0, int w, long long items, long long r0, ItemSets ex, int stage_cap, int k,
                  Cand* __restrict__ part) {
  extern __shared__ int s_set[];
  const int y = blockIdx.y, sp = blockIdx.x, splits = gridDim.x;
  const long long r = r0 + y;
  const long long per = (w + splits - 1) / splits;
  const long long lo = sp * per, hi = min((long long)w, lo + per);
  SetView set = {nullptr, 0, true};
  if (SETS) {
    set = set_stage(ex, r, s_set, stage_cap);
    __syncthreads();
  }
  float keys[KMAX];
  int idl[KMAX];
  list_clear(keys, idl);
  for (long long j = lo + threadIdx.x; j < hi; j += blockDim.x) {
    const long long id = serve_id(ids, ld_ids, r, c0 + j);
    if (id < 0 || id >= items) continue;
    const float key = serve_key(q[(long long)y * ldq + j]);
    if (better(key, (int)id, keys[KMAX - 1], idl[KMAX - 1]) && (!SETS || set.n == 0 || !set_has(set, s_set, (int)id)))
      list_insert(keys, idl, key, (int)id);
  }
  block_merge(keys, idl, k, part + ((long long)y * splits + sp) * k);
}

// one warp per row of the block: run[r] <- the k best of the row's running list and its `splits` block lists
static __global__ void __launch_bounds__(128)
serve_merge_kernel(const Cand* __restrict__ part, int splits, int k, long long r0, long long nr, Cand* __restrict__ run) {
  __shared__ Cand s_out[4][64];
  const long long y = (long long)blockIdx.x * 4 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31, wi = threadIdx.x >> 5;
  if (y >= nr) return;
  const Cand* mine = lane == kServeSplitsMax ? run + (r0 + y) * k : part + (y * splits + lane) * k;
  const bool owns = lane < splits || lane == kServeSplitsMax;
  warp_merge<1>(k, [&](int, int pos) { return owns && pos < k ? mine[pos] : Cand{FLT_MAX, kNoId}; },
                [&](int i, float key, int id, int) {
                  if (lane == 0) { s_out[wi][i].key = key; s_out[wi][i].id = id; }
                });
  __syncwarp();
  for (int i = lane; i < k; i += 32) run[(r0 + y) * k + i] = s_out[wi][i];
}

static __global__ void serve_run_init_kernel(Cand* __restrict__ run, long long count) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) { run[i].key = FLT_MAX; run[i].id = kNoId; }
}

// the outputs: values = Q (-key), ids; an empty slot is id -1, value -FLT_MAX
static __global__ void serve_out_kernel(const Cand* __restrict__ run, long long count, float* __restrict__ values,
                                        int64_t* __restrict__ ids) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const Cand c = run[i];
  ids[i] = c.id == kNoId ? -1 : (int64_t)c.id;
  values[i] = c.id == kNoId ? -FLT_MAX : -c.key;
}

// rank[r] <- 0, or -1 and *flag |= 1 for a target outside [0, items)
static __global__ void serve_rank_init_kernel(const long long* __restrict__ target, long long n, long long items,
                                              long long* __restrict__ rank, int* flag) {
  const long long r = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const bool ok = target[r] >= 0 && target[r] < items;
  rank[r] = ok ? 0 : -1;
  if (!ok) atomicOr(flag, 1);
}

// grid (splits, nr): rank[r] += the eligible items of the block that beat row r's target (higher Q, equal Q the smaller
// id), r = r0 + y.  The target never counts itself and is never excluded.  A target missing from its row's candidates
// (present[r] == 0) is beaten by every eligible candidate.
template <bool SETS>
__global__ void __launch_bounds__(kTopkThreads)
serve_count_kernel(const float* __restrict__ q, long long ldq, const long long* __restrict__ ids, long long ld_ids,
                   long long c0, int w, long long items, long long r0, const long long* __restrict__ target,
                   const int* __restrict__ present, const float* __restrict__ qt, ItemSets ex, int stage_cap,
                   long long* __restrict__ rank) {
  extern __shared__ int s_set[];
  const int y = blockIdx.y, sp = blockIdx.x, splits = gridDim.x;
  const long long r = r0 + y;
  const long long t = target[r];
  if (t < 0 || t >= items) return;
  const bool in = present == nullptr || present[r] != 0;
  const float kt = in ? serve_key(qt[r]) : FLT_MAX;
  const int ti = in ? (int)t : kNoId;
  const long long per = (w + splits - 1) / splits;
  const long long lo = sp * per, hi = min((long long)w, lo + per);
  SetView set = {nullptr, 0, true};
  if (SETS) {
    set = set_stage(ex, r, s_set, stage_cap);
    __syncthreads();
  }
  int c = 0;
  for (long long j = lo + threadIdx.x; j < hi; j += blockDim.x) {
    const long long id = serve_id(ids, ld_ids, r, c0 + j);
    if (id < 0 || id >= items || id == t) continue;
    if (better(serve_key(q[(long long)y * ldq + j]), (int)id, kt, ti) &&
        (!SETS || set.n == 0 || !set_has(set, s_set, (int)id)))
      ++c;
  }
  c = __reduce_add_sync(0xffffffffu, c);
  if ((threadIdx.x & 31) == 0 && c != 0)
    atomicAdd(reinterpret_cast<unsigned long long*>(rank + r), (unsigned long long)(long long)c);
}

struct ServeCall {
  const recnn_dims* d;
  const float* params;
  const float* table;
  int64_t n_items;
  const long long* cand;     // [n, M] or null (every item)
  int64_t M;
  ItemSets ex;
  ServePlan p;
  ServeWs w;
  NetLayout l;
  cudaStream_t st;
};

// E <- the embeddings of the block's pairs; v = E W1[:, S - lead : S + A]^T
static int serve_item_term(const ServeCall& c, const long long* ids, long long ld_ids, long long c0, int w, long long r0,
                           long long nr) {
  const ServePlan& p = c.p;
  const int64_t np = nr * w;
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(np, 8), (int64_t)kNumSMs * 16);
  serve_stage_kernel<<<grid, 256, 0, c.st>>>(c.table, c.n_items, p.A, ids, ld_ids, c0, w, r0, nr, p.lead, p.ldE, c.w.E);
  RECNN_CHECK_LAUNCH("serve_stage_kernel");
  Epilogue e = base_epi();
  e.out = c.w.v; e.ldo = p.H;
  const Seg xe = {c.w.E, p.A + p.lead, p.ldE, 0};      // the lead pads meet W1's last state columns: exact zeros
  return gemm_nt<EPI_STORE>(xe, kNoSeg, c.params + c.l.w1 + (p.S - p.lead), c.l.ld1, p.H, np, e, c.st);
}

// q[rr * ldq + j] = Q(row r0 + rr, staged item of pair rr * w + j) for the block's nr x w pairs
static int serve_pairs_q(const ServeCall& c, long long r0, long long nr, int w, bool v_per_pair, float* q,
                         long long ldq) {
  const ServePlan& p = c.p;
  const int64_t np = nr * w;
  serve_pair_kernel<<<elem_grid(np * p.H), 256, 0, c.st>>>(c.w.u, c.w.v, r0, nr, w, v_per_pair ? 1 : 0, p.H, c.w.h1);
  RECNN_CHECK_LAUNCH("serve_pair_kernel");
  const Rng rng = {nullptr, 0, nullptr};
  const Seg s1 = {c.w.h1, p.H, p.H, 0};
  RECNN_PROPAGATE(hidden_layer(s1, kNoSeg, c.params + c.l.w2, c.l.ld2, c.params + c.l.b2, p.H, np, false, nullptr, rng,
                               0, c.w.h2, c.st));
  const unsigned grid = (unsigned)std::min<int64_t>(ceil_div(np, 8), (int64_t)kNumSMs * 32);
  serve_score_kernel<<<grid, 256, 0, c.st>>>(c.w.h2, np, p.H, c.params + c.l.w3, c.params + c.l.b3, w, ldq, q);
  RECNN_CHECK_LAUNCH("serve_score_kernel");
  return RECNN_OK;
}

// The chunk loop of both calls: Q of every block of the call into w.q, then after(r0, nr, c0, w, ids, ld_ids) selects
// or counts.  Every item: the item term of each column chunk once, then every row block.  Candidates: row blocks, then
// the candidates' chunks, each gathering the rows of its pairs.
template <class After>
static int serve_blocks(const ServeCall& c, After after) {
  const ServePlan& p = c.p;
  if (!c.cand) {
    for (int64_t c0 = 0; c0 < c.n_items; c0 += p.C) {
      const int w = (int)std::min<int64_t>(p.C, c.n_items - c0);
      RECNN_PROPAGATE(serve_item_term(c, nullptr, 0, c0, w, 0, 1));
      for (int64_t r0 = 0; r0 < p.n; r0 += p.R) {
        const int64_t nr = std::min<int64_t>(p.R, p.n - r0);
        RECNN_PROPAGATE(serve_pairs_q(c, r0, nr, w, false, c.w.q, w));
        RECNN_PROPAGATE(after(r0, nr, c0, w, (const long long*)nullptr, 0ll));
      }
    }
    return RECNN_OK;
  }
  for (int64_t r0 = 0; r0 < p.n; r0 += p.R) {
    const int64_t nr = std::min<int64_t>(p.R, p.n - r0);
    for (int64_t c0 = 0; c0 < c.M; c0 += p.C) {
      const int w = (int)std::min<int64_t>(p.C, c.M - c0);
      RECNN_PROPAGATE(serve_item_term(c, c.cand, c.M, c0, w, r0, nr));
      RECNN_PROPAGATE(serve_pairs_q(c, r0, nr, w, true, c.w.q, w));
      RECNN_PROPAGATE(after(r0, nr, c0, w, c.cand, (long long)c.M));
    }
  }
  return RECNN_OK;
}

// argument checks, the workspace, the flag, the table and candidate checks, the row term.  k == 0: a rank call.
static int serve_begin(ServeCall& c, const recnn_dims* d, const float* params, const float* state, int64_t n,
                       const float* table, int64_t n_items, const int64_t* candidates, int64_t M, int k,
                       const int64_t* target, const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                       int64_t n_sets, const int64_t* row_set, int chunk, int32_t* error_flag, void* workspace,
                       int64_t workspace_bytes, cudaStream_t st) {
  RECNN_REQUIRE(d && params && state && table && error_flag && workspace, "null pointer");
  RECNN_REQUIRE(d->state_dim > 0 && d->action_dim > 0 && d->hidden > 0, "dims");
  RECNN_REQUIRE(n >= 0 && n_items > 0 && n_items < (1ll << 31) - 1, "0 < n_items < 2^31 - 1");
  RECNN_REQUIRE(candidates ? (M > 0 && M < (1ll << 31)) : M == 0, "n_candidates > 0 with a candidate list, else 0");
  RECNN_REQUIRE(chunk >= 0, "chunk >= 0 (0: auto)");
  RECNN_REQUIRE(k >= 0 && k <= 64, "1 <= k <= 64");
  c.d = d; c.params = params; c.table = table; c.n_items = n_items;
  c.cand = reinterpret_cast<const long long*>(candidates); c.M = M;
  c.st = st;
  c.l = critic_layout(*d);
  if (set_offsets) {
    RECNN_PROPAGATE(item_sets_args(set_ids, n_set_ids, set_offsets, n_sets, row_set, n, error_flag, &c.ex));
  } else {
    c.ex = ItemSets{nullptr, nullptr, nullptr, 0, 0, 0};
  }
  c.p = serve_plan(*d, n > 0 ? n : 1, candidates ? M : n_items, k, chunk);
  c.w = serve_carve(c.p, workspace);
  RECNN_PROPAGATE(check_workspace(c.w.bytes, workspace_bytes));
  RECNN_CHECK_CUDA(cudaMemsetAsync(error_flag, 0, sizeof(int32_t), st));
  if (n == 0) return RECNN_OK;
  if (c.ex.ids || c.ex.offsets) RECNN_PROPAGATE(item_sets_check(c.ex, n, n_items, error_flag, st));
  if (candidates) {
    serve_cand_check_kernel<<<(unsigned)n, 256, 0, st>>>(c.cand, (int)M, n_items,
                                                          reinterpret_cast<const long long*>(target), c.w.present,
                                                          error_flag);
    RECNN_CHECK_LAUNCH("serve_cand_check_kernel");
  }
  Seg xs;
  RECNN_PROPAGATE(repitch_state(c.p.S, state, n, c.w.img, &xs, st));
  return linear_out(xs, params + c.l.w1, c.l.ld1, params + c.l.b1, c.p.H, n, 0, nullptr, c.w.u, c.p.H, st);
}

// one back end for every GEMM of a call: the tensor cores need h1's row pitch H to be a 16-byte multiple
static bool serve_simt(const recnn_dims* d) { return d && d->hidden % 4 != 0; }

}  // namespace recnn

extern "C" int64_t recnn_critic_serve_workspace_bytes(const recnn_dims* d, int64_t n_rows, int64_t n_candidates,
                                                      int64_t n_items, int32_t k, int32_t chunk) {
  if (!d || n_rows <= 0 || n_items <= 0 || n_candidates < 0 || k < 0 || k > 64 || chunk < 0) return 0;
  if (d->state_dim <= 0 || d->action_dim <= 0 || d->hidden <= 0) return 0;
  const ServePlan p = serve_plan(*d, n_rows, n_candidates > 0 ? n_candidates : n_items, k, chunk);
  return serve_carve(p, nullptr).bytes;
}

extern "C" int recnn_critic_topk(const recnn_dims* d, const float* params, const float* state, int64_t n_rows,
                                 const float* table, int64_t n_items, const int64_t* candidates, int64_t n_candidates,
                                 int32_t k, const int64_t* set_ids, int64_t n_set_ids, const int64_t* set_offsets,
                                 int64_t n_sets, const int64_t* row_set, int32_t chunk, float* values_out,
                                 int64_t* ids_out, int32_t* error_flag, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  RECNN_REQUIRE(values_out && ids_out, "null pointer");
  RECNN_REQUIRE(k >= 1 && k <= 64, "1 <= k <= 64");
  SimtScope simt(serve_simt(d));
  ServeCall c;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_PROPAGATE(serve_begin(c, d, params, state, n_rows, table, n_items, candidates, n_candidates, k, nullptr,
                              set_ids, n_set_ids, set_offsets, n_sets, row_set, chunk, error_flag, workspace,
                              workspace_bytes, st));
  if (n_rows == 0) return RECNN_OK;
  const int64_t slots = n_rows * k;
  serve_run_init_kernel<<<(unsigned)ceil_div(slots, 256), 256, 0, st>>>(c.w.run, slots);
  RECNN_CHECK_LAUNCH("serve_run_init_kernel");
  const int stage = set_stage_bytes(c.ex);
  auto kernel = k <= 16 ? (stage ? serve_topk_kernel<16, true> : serve_topk_kernel<16, false>)
                        : (stage ? serve_topk_kernel<64, true> : serve_topk_kernel<64, false>);
  RECNN_PROPAGATE(serve_blocks(c, [&](int64_t r0, int64_t nr, int64_t c0, int w, const long long* ids, long long ld) {
    const int splits = topk_splits(nr, w, kServeSplitsMax);
    kernel<<<dim3((unsigned)splits, (unsigned)nr), kTopkThreads, stage, st>>>(
        c.w.q, w, ids, ld, c0, w, n_items, r0, c.ex, stage / (int)sizeof(int), k, c.w.part);
    RECNN_CHECK_LAUNCH("serve_topk_kernel");
    serve_merge_kernel<<<(unsigned)ceil_div(nr, 4), 128, 0, st>>>(c.w.part, splits, k, r0, nr, c.w.run);
    RECNN_CHECK_LAUNCH("serve_merge_kernel");
    return RECNN_OK;
  }));
  serve_out_kernel<<<(unsigned)ceil_div(slots, 256), 256, 0, st>>>(c.w.run, slots, values_out, ids_out);
  RECNN_CHECK_LAUNCH("serve_out_kernel");
  return RECNN_OK;
}

extern "C" int recnn_critic_rank(const recnn_dims* d, const float* params, const float* state, int64_t n_rows,
                                 const float* table, int64_t n_items, const int64_t* candidates, int64_t n_candidates,
                                 const int64_t* target, const int64_t* set_ids, int64_t n_set_ids,
                                 const int64_t* set_offsets, int64_t n_sets, const int64_t* row_set, int32_t chunk,
                                 int64_t* rank_out, int32_t* error_flag, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  RECNN_REQUIRE(target && rank_out, "null pointer");
  SimtScope simt(serve_simt(d));
  ServeCall c;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  RECNN_PROPAGATE(serve_begin(c, d, params, state, n_rows, table, n_items, candidates, n_candidates, 0, target,
                              set_ids, n_set_ids, set_offsets, n_sets, row_set, chunk, error_flag, workspace,
                              workspace_bytes, st));
  if (n_rows == 0) return RECNN_OK;
  const long long* tgt = reinterpret_cast<const long long*>(target);
  long long* rank = reinterpret_cast<long long*>(rank_out);
  serve_rank_init_kernel<<<(unsigned)ceil_div(n_rows, 256), 256, 0, st>>>(tgt, n_rows, n_items, rank, error_flag);
  RECNN_CHECK_LAUNCH("serve_rank_init_kernel");
  // Q of each row's target: the pair (r, target[r]) through the same code as every other pair, so the same bits
  const int64_t V = c.p.R * c.p.C;
  for (int64_t r0 = 0; r0 < n_rows; r0 += V) {
    const int64_t nr = std::min<int64_t>(V, n_rows - r0);
    RECNN_PROPAGATE(serve_item_term(c, tgt, 1, 0, 1, r0, nr));
    RECNN_PROPAGATE(serve_pairs_q(c, r0, nr, 1, true, c.w.qt + r0, 1));
  }
  const int stage = set_stage_bytes(c.ex);
  auto kernel = stage ? serve_count_kernel<true> : serve_count_kernel<false>;
  const int* present = candidates ? c.w.present : nullptr;
  return serve_blocks(c, [&](int64_t r0, int64_t nr, int64_t c0, int w, const long long* ids, long long ld) {
    const int splits = topk_splits(nr, w, kServeSplitsMax);
    kernel<<<dim3((unsigned)splits, (unsigned)nr), kTopkThreads, stage, st>>>(
        c.w.q, w, ids, ld, c0, w, n_items, r0, tgt, present, c.w.qt, c.ex, stage / (int)sizeof(int), rank);
    RECNN_CHECK_LAUNCH("serve_count_kernel");
    return RECNN_OK;
  });
}
