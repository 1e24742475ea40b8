// Peer-memory all-reduce of the gradient arenas (data-parallel update step, one process per GPU).
//
// The reference is single-process; BASELINE north_star asks for the minibatch to be sharded over the
// GPUs of one box with an all-reduce of the Actor/Critic gradients over NVLink.  Calling NCCL between
// the phases of the step costs three host-launched collectives and cuts the step's CUDA graph in three;
// instead every rank maps its peers' staging buffers (cudaIpc, NVLink/NVSwitch peer access) and ONE
// kernel per gradient arena does a TWO-SHOT all-reduce made of remote STORES only, in the style of NCCL's
// low-latency protocol: every payload float travels as an 8-byte word {value, epoch}, so the receiver polls
// the payload itself -- there are no flags, no system-scope fences and no arrival counters on the path
// (a system fence and a flag per peer and step cost more latency than the small payloads take to move).
//
//   A  reduce-scatter, push side: rank r owns slice r of the arena.  Every rank sums its split-K partials on the
//      fly (GradSource) and stores slice s of its gradient into rank s's contribution buffer [my rank], plus its few
//      "aux" words (loss partial sums, the global row count it assumed) into every peer.
//   B  owner side: for every element of my slice wait for the W contributions, sum them IN RANK ORDER (the same bits
//      on every rank), store the reduced element into every peer's result buffer (+ this CTA's partial L1 norm).
//   C  every rank waits for the elements of the whole reduced gradient as it consumes them: clip coefficient from
//      the L1 partials in a fixed order (actor), global loss means from the aux words, gradient written back
//      (scaled by the coefficient when there is one) and the built-in optimizer applied in the same pass.
//
// Bytes on NVLink per rank and arena: 2 x 2 (W-1)/W x 1.72 MB (the epoch tags double the payload; 6 MB at W = 8).
// It is an ordinary kernel on the step's stream, so the whole data-parallel step is captured in one CUDA graph
// exactly like the single-GPU step.  All sums are taken in rank order on every rank, so all replicas hold
// bit-identical gradients (and therefore weights) after every step.
//
// Protocol (epoch e = number of collectives issued so far on this communicator + 1; all on one stream):
//   * all buffers are double buffered by e & 1.  A rank can only be one epoch ahead of any peer (it needs every
//     peer's words of epoch e to finish e), so when it writes buffers (e+2) & 1 = e & 1 during epoch e+2 every peer
//     has completed its epoch-e kernel and no longer reads them.
//   * polls are bounded (~20 s of %globaltimer): a lost peer makes the kernel trap instead of hanging the GPU.
//   * ranks that disagree on n_rows_global (uneven shards without batch["n_rows_global"]) raise *err_flag.
#include <string.h>

#include <type_traits>

#include "common.cuh"
#include "pointwise.cuh"

namespace recnn {

constexpr int kMaxRanks = 8;
constexpr int kCommThreads = 512;
constexpr int kMaxAux = 8;
typedef unsigned long long ll_word;     // {epoch (high 32 bits), fp32 value (low 32 bits)}

struct CommDev {                       // lives at the head of every rank's shared allocation
  unsigned epoch;                      // collectives completed by this rank           (local)
  unsigned done;                       // CTAs that finished (wraps to 0)              (local)
  unsigned pad[30];
  ll_word aux[2][kMaxRanks][kMaxAux + 1];          // [e & 1][src]: aux floats, then the row count src assumed
  ll_word l1[2][kMaxRanks][kNumSMs];               // [e & 1][src][cta]: partial L1 norms of src's reduced slice
};

struct CommPeers {                     // kernel parameter
  CommDev* ctrl[kMaxRanks];
  ll_word* contrib[kMaxRanks];         // [2][W][slice_cap] words: contributions to THAT rank's slice
  ll_word* result[kMaxRanks];          // [2][capacity] words: the reduced gradient, assembled by the owners
  long long capacity, slice_cap;
  int rank, world;
};

struct CommOpt {                       // optional fused optimizer (kind == RECNN_OPT_EXTERNAL: none)
  int kind;
  OptConsts k;
  double beta1, beta2, lr, wd, n_sma_threshold;
  int k_look;
  float *p, *m, *v, *slow;
  int* t;
};

}  // namespace recnn

struct recnn_comm {
  recnn::CommPeers peers;
  void* local_base;
  void* opened[recnn::kMaxRanks];
  cudaIpcMemHandle_t handle;
  bool connected;
};

namespace recnn {

__device__ __forceinline__ unsigned long long comm_gtimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ ll_word ll_pack(float v, unsigned e) {
  return ((ll_word)e << 32) | (ll_word)__float_as_uint(v);
}
__device__ __forceinline__ void st_ll(ll_word* p, float v, unsigned e) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(ll_pack(v, e)) : "memory");
}
__device__ __forceinline__ void st_ll2(ll_word* p, float v0, float v1, unsigned e) {      // p 16-byte aligned
  asm volatile("st.relaxed.sys.global.v2.u64 [%0], {%1, %2};" ::"l"(p), "l"(ll_pack(v0, e)), "l"(ll_pack(v1, e)) : "memory");
}
__device__ __forceinline__ ll_word ld_ll(const ll_word* p) {
  ll_word w;
  asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(w) : "l"(p) : "memory");
  return w;
}
__device__ __forceinline__ void comm_timeout(int rank, unsigned e, const char* what) {
  printf("recnn_b200 allreduce: rank %d timed out waiting for %s (epoch %u)\n", rank, what, e);
  __trap();
}
// spin until the word carries epoch e; returns its payload bits
__device__ __forceinline__ unsigned wait_ll_bits(const ll_word* p, unsigned e, int rank, const char* what) {
  ll_word w = ld_ll(p);
  if ((unsigned)(w >> 32) == e) return (unsigned)w;
  const unsigned long long t0 = comm_gtimer();
  unsigned spins = 0;
  for (;;) {
    w = ld_ll(p);
    if ((unsigned)(w >> 32) == e) return (unsigned)w;
    if ((++spins & 1023u) == 0 && comm_gtimer() - t0 > 20000000000ull) comm_timeout(rank, e, what);
  }
}
__device__ __forceinline__ float wait_ll(const ll_word* p, unsigned e, int rank, const char* what) {
  return __uint_as_float(wait_ll_bits(p, e, rank, what));
}
__device__ __forceinline__ void wait_ll2(const ll_word* p, unsigned e, int rank, const char* what, float& v0, float& v1) {
  const unsigned long long t0 = comm_gtimer();
  unsigned spins = 0;
  for (;;) {
    ll_word w0, w1;
    asm volatile("ld.relaxed.sys.global.v2.u64 {%0, %1}, [%2];" : "=l"(w0), "=l"(w1) : "l"(p) : "memory");
    if ((unsigned)(w0 >> 32) == e && (unsigned)(w1 >> 32) == e) {
      v0 = __uint_as_float((unsigned)w0);
      v1 = __uint_as_float((unsigned)w1);
      return;
    }
    if ((++spins & 1023u) == 0 && comm_gtimer() - t0 > 20000000000ull) comm_timeout(rank, e, what);
  }
}

// grid <= number of SMs (all CTAs must be co-resident: they wait for words other CTAs -- of other ranks -- produce).
// VEC = 2: n even and buf 8-byte aligned (the arenas): two elements = one 16-byte store of two words; VEC = 1: anything.
template <int VEC>
__global__ void __launch_bounds__(kCommThreads, 1)
allreduce_kernel(CommPeers c, float* __restrict__ buf, long long n, float max_norm, float* coef_out, float* l1_out,
                 const float* aux_in, float* aux_out, int n_aux, float check_val, int* err_flag, CommOpt opt,
                 GradSource src) {
  __shared__ float red[32];
  __shared__ unsigned s_epoch;
  __shared__ bool s_last;
  __shared__ float s_coef;
  __shared__ OptStep s_st;
  CommDev* me = c.ctrl[c.rank];
  if (threadIdx.x == 0) s_epoch = *((volatile unsigned*)&me->epoch) + 1;
  __syncthreads();
  const unsigned e = s_epoch;
  const int par = (int)(e & 1u);
  const int W = c.world;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  const long long units = n / VEC;                               // VEC == 2 => n % 2 == 0
  const long long slice = units > 0 ? (units + W - 1) / W : 1;   // units per owner (the last slice may be short)

  // ---- A: push slice s of my gradient to owner s, aux words to everyone (remote stores, nothing to wait for)
  for (long long i = tid; i < units; i += nth) {
    const int s = (int)(i / slice);
    ll_word* dst = c.contrib[s] + ((long long)par * W + c.rank) * c.slice_cap + (i - (long long)s * slice) * VEC;
    if constexpr (VEC == 2) {
      float g0, g1;
      if (src.n_layers) {            // the local gradient is still in split-K partials: reduce them on the way out
        const float4 q = grad4_at(src, buf, (unsigned)((2 * i) & ~3ll));
        g0 = (i & 1) ? q.z : q.x;
        g1 = (i & 1) ? q.w : q.y;
      } else {
        const float2 q = reinterpret_cast<const float2*>(buf)[i];
        g0 = q.x; g1 = q.y;
      }
      st_ll2(dst, g0, g1, e);
    } else {
      st_ll(dst, src.n_layers ? grad_at(src, buf, i) : buf[i], e);
    }
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < W) {
    ll_word* dst = c.ctrl[threadIdx.x]->aux[par][c.rank];
    for (int j = 0; j < n_aux; ++j) st_ll(dst + j, aux_in[j], e);
    st_ll(dst + kMaxAux, check_val, e);
  }
  // ---- B: owner: every element of my slice: wait for the W contributions, sum in rank order, push to everyone
  if (units > 0) {
    const long long lo = (long long)c.rank * slice;
    const long long cnt = units - lo < slice ? (units - lo > 0 ? units - lo : 0) : slice;
    const ll_word* mine = c.contrib[c.rank] + (long long)par * W * c.slice_cap;
    float l1 = 0.f;
    for (long long i = tid; i < cnt; i += nth) {
      float s0 = 0.f, s1 = 0.f;
      for (int p = 0; p < W; ++p) {
        const ll_word* w = mine + (long long)p * c.slice_cap + i * VEC;
        if constexpr (VEC == 2) {
          float v0, v1;
          wait_ll2(w, e, c.rank, "a contribution", v0, v1);
          s0 = p == 0 ? v0 : s0 + v0;
          s1 = p == 0 ? v1 : s1 + v1;
        } else {
          const float v0 = wait_ll(w, e, c.rank, "a contribution");
          s0 = p == 0 ? v0 : s0 + v0;
        }
      }
      l1 += fabsf(s0) + (VEC == 2 ? fabsf(s1) : 0.f);
      for (int p = 0; p < W; ++p) {
        ll_word* dst = c.result[p] + (long long)par * c.capacity + (lo + i) * VEC;
        if constexpr (VEC == 2) st_ll2(dst, s0, s1, e);
        else st_ll(dst, s0, e);
      }
    }
    if (coef_out) {
      l1 = block_sum(l1, red);
      if ((int)threadIdx.x < W) st_ll(&c.ctrl[threadIdx.x]->l1[par][c.rank][blockIdx.x], l1, e);
    }
  }
  // ---- C: everyone: scalars first (clip coefficient, loss sums, optimizer step constants)
  if (threadIdx.x < 32) {
    float coef = 1.0f;
    if (coef_out) {
      // ||g||_1 from the owners' per-CTA partials: lane l takes entries l, l+32, ... of the (rank-major, CTA-minor)
      // list, then a shuffle tree -- the same order on every rank and CTA, so every replica gets the same bits
      const int total = W * (int)gridDim.x;
      float t = 0.f;
      for (int k = (int)threadIdx.x; k < total; k += 32)
        t += wait_ll(&me->l1[par][k / (int)gridDim.x][k % (int)gridDim.x], e, c.rank, "an L1 partial");
      t = warp_sum(t);
      coef = fminf(max_norm / (t + 1e-6f), 1.0f);     // clip_grad_norm_: max_norm / (total_norm + 1e-6), <= 1
      if (blockIdx.x == 0 && threadIdx.x == 0) {
        *coef_out = coef;
        if (l1_out) *l1_out = t;
      }
    }
    if (threadIdx.x == 0) {
      s_coef = coef;
      if (opt.kind != RECNN_OPT_EXTERNAL)
        s_st = opt_step_scalars(opt.kind, opt.beta1, opt.beta2, opt.lr, opt.wd, opt.n_sma_threshold, opt.k_look, *opt.t + 1);
      if (blockIdx.x == 0) {
        bool bad = false;
        for (int p = 0; p < W; ++p) bad = bad || wait_ll(&me->aux[par][p][kMaxAux], e, c.rank, "a peer's row count") != check_val;
        if (bad && err_flag) *err_flag = 1;
        for (int j = 0; j < n_aux; ++j) {
          float t = 0.f;
          for (int p = 0; p < W; ++p) t += wait_ll(&me->aux[par][p][j], e, c.rank, "a peer's loss sum");
          aux_out[j] = t;
        }
      }
    }
  }
  __syncthreads();
  // ---- the reduced gradient, element by element as it arrives: write back (scaled) and apply the optimizer
  {
    const float coef = s_coef;
    const bool scale = coef_out != nullptr;
    const int t_next = opt.kind != RECNN_OPT_EXTERNAL ? *opt.t + 1 : 0;
    const OptStep ost = s_st;
    const ll_word* res = c.result[c.rank] + (long long)par * c.capacity;
    for (long long i = tid; i < units; i += nth) {
      float g0, g1 = 0.f;
      if constexpr (VEC == 2) wait_ll2(res + i * 2, e, c.rank, "a reduced element", g0, g1);
      else g0 = wait_ll(res + i, e, c.rank, "a reduced element");
      if (scale) {
        g0 = __fmul_rn(g0, coef);
        g1 = __fmul_rn(g1, coef);
      }
      if constexpr (VEC == 2) reinterpret_cast<float2*>(buf)[i] = make_float2(g0, g1);   // the caller-visible .grad
      else buf[i] = g0;
      if (opt.kind != RECNN_OPT_EXTERNAL) {
        opt_apply(opt.kind, opt.k, ost, t_next, opt.p, opt.m, opt.v, opt.slow, i * VEC, g0);
        if constexpr (VEC == 2) opt_apply(opt.kind, opt.k, ost, t_next, opt.p, opt.m, opt.v, opt.slow, i * VEC + 1, g1);
      }
    }
  }
  // ---- D: the last CTA closes the epoch (and advances the optimizer's step count)
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicInc(&me->done, gridDim.x - 1) == gridDim.x - 1;
  __syncthreads();
  if (s_last && threadIdx.x == 0) {
    if (opt.kind != RECNN_OPT_EXTERNAL) *opt.t = *opt.t + 1;
    *((volatile unsigned*)&me->epoch) = e;
  }
}

// All-gather in the same word protocol: every rank stores its n words, as raw bits, into slot [my rank] of the
// contribution buffer of every peer (epoch e, buffer e & 1), then waits for the W slots of its own buffer and writes
// them out rank-major.  It takes an epoch from the same counter as allreduce_kernel, so the two interleave freely.
// grid <= number of SMs (all CTAs of all ranks resident at once), n <= slice_cap.
__global__ void __launch_bounds__(kCommThreads, 1)
allgather_kernel(CommPeers c, const unsigned* __restrict__ local, long long n, unsigned* __restrict__ gathered) {
  __shared__ unsigned s_epoch;
  __shared__ bool s_last;
  CommDev* me = c.ctrl[c.rank];
  if (threadIdx.x == 0) s_epoch = *((volatile unsigned*)&me->epoch) + 1;
  __syncthreads();
  const unsigned e = s_epoch;
  const int par = (int)(e & 1u);
  const int W = c.world;
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, nth = (long long)gridDim.x * blockDim.x;
  for (long long i = tid; i < n; i += nth) {
    const ll_word w = ((ll_word)e << 32) | (ll_word)local[i];
    for (int p = 0; p < W; ++p) {
      ll_word* dst = c.contrib[p] + ((long long)par * W + c.rank) * c.slice_cap + i;
      asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(dst), "l"(w) : "memory");
    }
  }
  const ll_word* mine = c.contrib[c.rank] + (long long)par * W * c.slice_cap;
  for (long long i = tid; i < n; i += nth)
    for (int q = 0; q < W; ++q) gathered[q * n + i] = wait_ll_bits(mine + (long long)q * c.slice_cap + i, e, c.rank, "a peer's slot");
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) s_last = atomicInc(&me->done, gridDim.x - 1) == gridDim.x - 1;
  __syncthreads();
  if (s_last && threadIdx.x == 0) *((volatile unsigned*)&me->epoch) = e;
}

// every CTA must be resident at once: at most one per SM of THIS device (and no more than the L1-partials array holds)
static int comm_grid(int64_t n, int* grid) {
  int dev = 0, sms = 0;
  RECNN_CHECK_CUDA(cudaGetDevice(&dev));
  RECNN_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int cap = sms < kNumSMs ? sms : kNumSMs;
  const int64_t blocks = ceil_div(n, (int64_t)kCommThreads * 8);   // eight words per thread
  *grid = (int)(blocks < 1 ? 1 : (blocks > cap ? cap : blocks));
  return RECNN_OK;
}

int launch_comm_allgather(const recnn_comm* comm, const float* local, int64_t n, float* gathered, cudaStream_t st) {
  RECNN_REQUIRE(comm != nullptr && comm->connected, "communicator is not connected");
  RECNN_REQUIRE(n >= 0 && n * comm->peers.world <= comm->peers.capacity,
                "all-gather larger than the communicator's staging capacity (n * world > capacity)");
  RECNN_REQUIRE(n == 0 || (local != nullptr && gathered != nullptr), "local / gathered");
  int grid = 1;
  RECNN_PROPAGATE(comm_grid(n, &grid));
  allgather_kernel<<<grid, kCommThreads, 0, st>>>(comm->peers, reinterpret_cast<const unsigned*>(local), n,
                                                   reinterpret_cast<unsigned*>(gathered));
  RECNN_CHECK_LAUNCH("allgather_kernel");
  return RECNN_OK;
}

int launch_comm_allreduce(const recnn_comm* comm, float* buf, int64_t n, const CommReduce& r, cudaStream_t st) {
  RECNN_REQUIRE(comm != nullptr && comm->connected, "communicator is not connected");
  RECNN_REQUIRE(n >= 0 && n <= comm->peers.capacity, "all-reduce larger than the communicator's staging capacity");
  RECNN_REQUIRE(n == 0 || buf != nullptr, "buf");
  RECNN_REQUIRE(r.n_aux >= 0 && r.n_aux <= kMaxAux && (r.n_aux == 0 || (r.aux_in && r.aux_out)), "aux floats");
  CommOpt opt;
  memset(&opt, 0, sizeof(opt));
  opt.kind = RECNN_OPT_EXTERNAL;
  if (r.optim && r.optim->kind != RECNN_OPT_EXTERNAL) {
    RECNN_REQUIRE(r.net && r.net->params && r.net->opt_t, "fused optimizer needs params and the step counter");
    RECNN_REQUIRE(r.optim->kind == RECNN_OPT_SGD || r.optim->kind == RECNN_OPT_ADAM || r.optim->kind == RECNN_OPT_RANGER ||
                      r.optim->kind == RECNN_OPT_RADAM,
                  "built-in optimizer kind must be SGD, ADAM, RANGER or RADAM");
    if (r.optim->kind == RECNN_OPT_ADAM || r.optim->kind == RECNN_OPT_RADAM)
      RECNN_REQUIRE(r.net->opt_m && r.net->opt_v, "Adam / RAdam need exp_avg / exp_avg_sq arenas");
    if (r.optim->kind == RECNN_OPT_RANGER) RECNN_REQUIRE(r.net->opt_m && r.net->opt_v && r.net->opt_slow, "Ranger needs exp_avg / exp_avg_sq / slow arenas");
    if (r.optim->kind == RECNN_OPT_SGD && r.optim->momentum != 0.f) RECNN_REQUIRE(r.net->opt_m, "SGD momentum needs a buffer arena");
    opt.kind = r.optim->kind;
    opt.k = opt_consts(*r.optim);
    opt.beta1 = r.optim->beta1; opt.beta2 = r.optim->beta2; opt.lr = r.optim->lr;
    opt.wd = r.optim->weight_decay; opt.n_sma_threshold = r.optim->n_sma_threshold; opt.k_look = r.optim->k;
    opt.p = r.net->params; opt.m = r.net->opt_m; opt.v = r.net->opt_v; opt.slow = r.net->opt_slow; opt.t = r.net->opt_t;
  }
  GradSource gsrc;
  memset(&gsrc, 0, sizeof(gsrc));
  if (r.src) gsrc = *r.src;
  int grid = 1;
  RECNN_PROPAGATE(comm_grid(n, &grid));
  // partial-sourced gradients are read four at a time: the arena case (n % 4 == 0, 16-byte aligned)
  const bool vec = (n & 1) == 0 && ((reinterpret_cast<uintptr_t>(buf) & 7) == 0) &&
                   (!r.src || ((n & 3) == 0 && (reinterpret_cast<uintptr_t>(buf) & 15) == 0));
  RECNN_REQUIRE(vec || !r.src, "partial-sourced gradients need a 16-byte aligned arena");
  if (vec)
    allreduce_kernel<2><<<grid, kCommThreads, 0, st>>>(comm->peers, buf, n, r.max_norm, r.coef, r.l1_out, r.aux_in,
                                                        r.aux_out, r.n_aux, r.check_val, r.err_flag, opt, gsrc);
  else
    allreduce_kernel<1><<<grid, kCommThreads, 0, st>>>(comm->peers, buf, n, r.max_norm, r.coef, r.l1_out, r.aux_in,
                                                        r.aux_out, r.n_aux, r.check_val, r.err_flag, opt, gsrc);
  RECNN_CHECK_LAUNCH("allreduce_kernel");
  return RECNN_OK;
}

}  // namespace recnn

using namespace recnn;

// staging layout of one rank: CommDev | contrib [2][W][slice_cap] | result [2][capacity]   (8-byte words)
static size_t comm_ctrl_bytes() { return (size_t)round_up((int64_t)sizeof(CommDev), 256); }
static void comm_carve(recnn_comm* c, int p, void* base) {
  char* b = static_cast<char*>(base);
  c->peers.ctrl[p] = reinterpret_cast<CommDev*>(b);
  c->peers.contrib[p] = reinterpret_cast<ll_word*>(b + comm_ctrl_bytes());
  c->peers.result[p] = c->peers.contrib[p] + 2ll * c->peers.world * c->peers.slice_cap;
}

extern "C" int recnn_comm_create(int32_t rank, int32_t world, int64_t capacity_floats, recnn_comm** out) {
  RECNN_REQUIRE(out != nullptr, "out");
  RECNN_REQUIRE(world >= 1 && world <= kMaxRanks && rank >= 0 && rank < world, "rank/world (at most 8 ranks)");
  RECNN_REQUIRE(capacity_floats > 0, "capacity");
  capacity_floats = round_up(capacity_floats, 4);
  recnn_comm* c = new recnn_comm();
  c->connected = false;
  for (int i = 0; i < kMaxRanks; ++i) {
    c->opened[i] = nullptr; c->peers.ctrl[i] = nullptr; c->peers.contrib[i] = nullptr; c->peers.result[i] = nullptr;
  }
  c->peers.capacity = capacity_floats;
  c->peers.slice_cap = round_up(ceil_div(capacity_floats, world), 4) + 4;
  c->peers.rank = rank;
  c->peers.world = world;
  const size_t bytes = comm_ctrl_bytes() +
                       sizeof(ll_word) * (size_t)(2 * world * c->peers.slice_cap + 2 * capacity_floats);
  cudaError_t e = cudaMalloc(&c->local_base, bytes);
  if (e != cudaSuccess) {
    delete c;
    set_error("cudaMalloc of the all-reduce staging buffer (%zu bytes) failed: %s", bytes, cudaGetErrorString(e));
    return RECNN_E_CUDA;
  }
  cudaMemset(c->local_base, 0, bytes);
  e = cudaIpcGetMemHandle(&c->handle, c->local_base);
  if (e != cudaSuccess) {
    cudaFree(c->local_base);
    delete c;
    set_error("cudaIpcGetMemHandle failed: %s", cudaGetErrorString(e));
    return RECNN_E_CUDA;
  }
  cudaDeviceSynchronize();
  *out = c;
  return RECNN_OK;
}

extern "C" int32_t recnn_comm_handle_bytes(void) { return (int32_t)sizeof(cudaIpcMemHandle_t); }

extern "C" int recnn_comm_local_handle(const recnn_comm* c, void* out) {
  RECNN_REQUIRE(c && out, "args");
  memcpy(out, &c->handle, sizeof(cudaIpcMemHandle_t));
  return RECNN_OK;
}

// all_handles: world consecutive handles in rank order (this rank's own entry is ignored)
extern "C" int recnn_comm_connect(recnn_comm* c, const void* all_handles) {
  RECNN_REQUIRE(c && all_handles, "args");
  RECNN_REQUIRE(!c->connected, "already connected");
  const char* hs = static_cast<const char*>(all_handles);
  for (int p = 0; p < c->peers.world; ++p) {
    void* base = c->local_base;
    if (p != c->peers.rank) {
      cudaIpcMemHandle_t h;
      memcpy(&h, hs + (size_t)p * sizeof(h), sizeof(h));
      cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        set_error("cudaIpcOpenMemHandle(rank %d) failed: %s", p, cudaGetErrorString(e));
        for (int q = 0; q < p; ++q)
          if (c->opened[q]) { cudaIpcCloseMemHandle(c->opened[q]); c->opened[q] = nullptr; }
        (void)cudaGetLastError();
        return RECNN_E_CUDA;
      }
      c->opened[p] = base;
    }
    comm_carve(c, p, base);
  }
  c->connected = true;
  return RECNN_OK;
}

extern "C" int recnn_comm_allreduce(const recnn_comm* c, float* buf, int64_t n, void* stream) {
  return launch_comm_allreduce(c, buf, n, CommReduce(), static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_comm_allgather(const recnn_comm* c, const float* local, int64_t n, float* gathered, void* stream) {
  return launch_comm_allgather(c, local, n, gathered, static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_comm_destroy(recnn_comm* c) {
  if (!c) return RECNN_OK;
  cudaDeviceSynchronize();
  for (int p = 0; p < kMaxRanks; ++p)
    if (c->opened[p]) cudaIpcCloseMemHandle(c->opened[p]);
  if (c->local_base) cudaFree(c->local_base);
  delete c;
  return RECNN_OK;
}
