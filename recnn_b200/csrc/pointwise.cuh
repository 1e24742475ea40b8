// Declarations of the non-GEMM kernels' host launchers (pointwise.cu).
#pragma once
#include "common.cuh"

namespace recnn {

// ---- where a gradient element comes from -------------------------------------------------------------------
// The weight-gradient GEMMs leave split-K partials [splits][C][K1] (column K1-1 = the bias gradient, written by the
// column-sum kernel).  Instead of a reduce kernel per layer followed by the optimizer pass, the optimizer (and the
// data-parallel all-reduce) read the partials directly: grad_at() sums the splits of the element's layer in a fixed
// order; elements outside the listed layers (the critic's head, written by the fused value-head kernel) come from
// the gradient arena itself.  Two launches and one pass over the arena less on the step's serial tail.
struct PartialLayer {
  const float* part;       // [splits][C][K1]
  int splits, C, K1;
  int ld;                  // row pitch of the weight in the arena
  long long w_off, b_off;  // arena offsets of the weight [C, ld] and of the bias [C]
};
struct GradSource {
  PartialLayer l[2];
  int n_layers;            // 0: every element comes from the gradient arena
};
#ifdef __CUDACC__
// four consecutive arena elements starting at i (i % 4 == 0; weight rows and bias segments start on multiples of 4,
// so the four never straddle a row or a segment).  32-bit index arithmetic: an arena has far fewer than 2^31 elements.
__device__ __forceinline__ float4 grad4_at(const GradSource& s, const float* __restrict__ direct, unsigned i) {
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (k >= s.n_layers) break;
    const PartialLayer& L = s.l[k];
    const unsigned tot = (unsigned)L.C * (unsigned)L.K1;
    const unsigned ew = i - (unsigned)L.w_off, eb = i - (unsigned)L.b_off;
    if (ew < (unsigned)L.C * (unsigned)L.ld) {
      const unsigned r = ew / (unsigned)L.ld, c = ew - r * (unsigned)L.ld;
      const float* p0 = L.part + (size_t)r * L.K1 + c;
      float g[4] = {0.f, 0.f, 0.f, 0.f};
      const int valid = (int)(L.K1 - 1) - (int)c;              // columns c .. c+3 that are real weights (the rest: pitch padding)
      // eight splits per round with all their loads issued before the first add (the serial tail of the step waits
      // for this pass: a load-add chain per split made it latency-bound)
      for (int z0 = 0; z0 < L.splits; z0 += 8) {
        float v[8][4];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float* p = p0 + (size_t)(z0 + u) * tot;
#pragma unroll
          for (int j = 0; j < 4; ++j) v[u][j] = (z0 + u < L.splits && j < valid) ? p[j] : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u)
#pragma unroll
          for (int j = 0; j < 4; ++j) g[j] += v[u][j];
      }
      return make_float4(g[0], g[1], g[2], g[3]);
    }
    if (eb < (unsigned)(((L.C + 3) / 4) * 4)) {
      float g[4] = {0.f, 0.f, 0.f, 0.f};
      for (int z = 0; z < L.splits; ++z) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (eb + j < (unsigned)L.C) g[j] += L.part[(size_t)z * tot + (size_t)(eb + j) * L.K1 + (L.K1 - 1)];
      }
      return make_float4(g[0], g[1], g[2], g[3]);
    }
  }
  return *reinterpret_cast<const float4*>(direct + i);
}
__device__ __forceinline__ float grad_at(const GradSource& s, const float* __restrict__ direct, long long i) {
  const float4 v = grad4_at(s, direct, (unsigned)(i & ~3ll));
  const int j = (int)(i & 3);
  return j == 0 ? v.x : j == 1 ? v.y : j == 2 ? v.z : v.w;
}
#endif

enum HeadMode {
  HEAD_PLAIN = 0,        // out[n] = q
  HEAD_TARGET_DDPG = 1,  // y[n] = clamp(r + (1-d)*gamma*q, min, max)            misc.py:30-35
  HEAD_TARGET_TD3_A = 2, // tmp[n] = q                                            td3.py:81
  HEAD_TARGET_TD3_B = 3, // y[n] = r + (1-d)*gamma*min(tmp[n], q)  (no clamp)     td3.py:82-86
  HEAD_VALUE = 4,        // diff=q-y; dq[n]=2*diff/Ng; loss += diff^2/Ng          misc.py:37-39
  HEAD_POLICY = 5        // loss += -q/Ng                                          ddpg.py:79,87
};

struct HeadArgs {
  const float* h2;      // [N, H]
  const float* w3;      // [H]
  const float* b3;      // [1]
  int64_t n_rows;
  int64_t n_rows_global;
  int hidden;
  int mode;
  const float* reward;  // [N]
  const float* done;    // [N]
  float gamma, min_value, max_value;
  float* y;             // TD target in/out
  float* tmp;           // TD3 first critic
  float* out;           // HEAD_PLAIN / q copy (may be null)
  float* dq;            // HEAD_VALUE
  float* loss;          // device scalar to write (VALUE / POLICY)
  float* block_partials;  // >= gridDim floats
  unsigned* ticket;       // zero-initialised, self-resetting
};
int launch_critic_head(const HeadArgs& a, cudaStream_t st);

// Everything between the critic's last hidden layer and its backward GEMMs in ONE kernel (was five launches
// on the step's critical path): q = h2 w3 + b3; TD target y from the target critic's hidden layer (DDPG,
// misc.py:28-35) or a precomputed y (TD3's min of two targets); MSE loss; dq = 2 (q - y) / N_global;
// dz2 = dq w3 * gate(h2); dW3 = dq^T h2 and db3 = sum dq (deterministic two-level reductions).
struct ValueHeadArgs {
  const float *h2, *w3, *b3;         // online critic: hidden2 [N, H], head weights
  const float *th2, *tw3, *tb3;      // target critic (fused TD target) or null (y is an input)
  const float *reward, *done;
  float gamma, min_value, max_value;
  float* y;                          // [N] TD target: written when th2 != null, read otherwise
  int64_t n_rows, n_rows_global;
  int hidden;
  int learn;                         // 0: loss only
  float gate_scale;
  float* dz2;                        // [N, H]
  float* gw3;                        // [H] gradient of the head weights
  float* gb3;                        // [1]
  float* loss;
  float* block_partials;             // >= kNumSMs * (H + 2) floats
  unsigned* ticket;
};
bool value_head_fusable(int hidden);
int launch_value_head_fused(const ValueHeadArgs& a, cudaStream_t st);

// dz2[n,c] = dq_n * w3[c] * (h2[n,c] > 0 ? gate_scale : 0); dq_n = dq ? dq[n] : dq_const
int launch_critic_head_bwd(const float* dq, float dq_const, const float* w3, const float* h2,
                           float gate_scale, float* dz2, int64_t n_rows, int hidden, cudaStream_t st);

// grad arena <- sum over split-K partials; part is [splits][C][K1] where column K1-1 is the
// bias gradient: w_dst[c*ldw+k] for k<K1-1 (ldw = arena row pitch), b_dst[c] for k==K1-1.
int launch_reduce_partials(const float* part, int splits, int C, int K1, float* w_dst, long long ldw,
                           float* b_dst, cudaStream_t st);
int launch_head_grad_partials(const float* dq, const float* h2, int64_t n_rows, int H, int64_t rows_per_split,
                              int splits, float* part, cudaStream_t st);
int launch_colsum_partials(const float* dz, int64_t n_rows, int C, int64_t rows_per_split, int splits,
                           float* part, int K1, cudaStream_t st);

// *coef = min(max_norm / (||g||_1 + 1e-6), 1)  (clip_grad_norm_(.., -1, 1): ddpg.py:92);  *l1_out = ||g||_1
int launch_l1_clip_coef(const float* grads, int64_t count, float max_norm, float* coef, float* l1_out,
                        float* block_partials, unsigned* ticket, cudaStream_t st);

// comm.cu: buf <- sum over the communicator's ranks (in place, rank order), two-shot over NVLink peer memory.
// Optional riders of the same kernel: the L1 norm of the summed gradient and its clip coefficient (as
// launch_l1_clip_coef would give them; the gradient is then left scaled by the coefficient), up to 8 "aux" floats
// summed over the ranks (loss partial sums), a consistency check of a value every rank must agree on (the
// global row count), and the built-in optimizer's update of `net` with the reduced gradient (step count included).
struct CommReduce {
  float max_norm = 0.f;
  float* coef = nullptr;
  float* l1_out = nullptr;
  const float* aux_in = nullptr;
  float* aux_out = nullptr;
  int n_aux = 0;
  float check_val = 0.f;
  int* err_flag = nullptr;
  const recnn_optim* optim = nullptr;
  const recnn_net* net = nullptr;
  const GradSource* src = nullptr;     // local gradient = split-K partials (see GradSource) instead of `buf`
};
int launch_comm_allreduce(const recnn_comm* comm, float* buf, int64_t n, const CommReduce& r, cudaStream_t st);

// zero the `lead` leading and the trailing pad columns of up to three [n_rows, ld] buffers whose data columns are
// [lead, lead + cols) (the lead-padded action images of the step); one launch instead of three full memsets
int launch_zero_pad_columns(float* b0, float* b1, float* b2, int64_t n_rows, int ld, int lead, int cols, cudaStream_t st);
int launch_scale_inplace(float* x, int64_t count, const float* scale, cudaStream_t st);

// ---- fused optimizers: per-element update shared by optimizer_kernel and the all-reduce kernel (comm.cu) ----
struct OptConsts {
  float lr, one_minus_b1, b1, b2, one_minus_b2, eps, wd, momentum, alpha;
};
static inline OptConsts opt_consts(const recnn_optim& o) {
  OptConsts k;
  k.lr = (float)o.lr;
  k.one_minus_b1 = (float)(1.0 - o.beta1);
  k.b1 = (float)o.beta1;
  k.b2 = (float)o.beta2;
  k.one_minus_b2 = (float)(1.0 - o.beta2);
  k.eps = (float)o.eps;
  k.wd = (float)o.weight_decay;
  k.momentum = (float)o.momentum;
  k.alpha = (float)o.alpha;
  return k;
}
// the step-dependent scalars of one optimizer step (python-float arithmetic in double, cast where torch casts)
struct OptStep {
  float step_size;     // Adam: lr / (1 - beta1^t); Ranger: -(rectified step size) * lr as torch_optimizer forms it
  float bc2_sqrt;      // Adam: sqrt(1 - beta2^t)
  float wd_lr;         // Ranger: -weight_decay * lr
  int adaptive;        // Ranger / RAdam: N_sma past the threshold (use the variance term)
  int lookahead;       // Ranger: t % k == 0 (interpolate towards / reset to the slow weights)
  int first;           // Ranger: first step (slow weights start as a copy of the parameters)
};
#ifdef __CUDACC__
__device__ __forceinline__ OptStep opt_step_scalars(int kind, double beta1, double beta2, double lr, double wd,
                                                    double n_sma_threshold, int k_look, int t) {
  OptStep s;
  s.step_size = 0.f; s.bc2_sqrt = 1.f; s.wd_lr = 0.f; s.adaptive = 0; s.lookahead = 0; s.first = (t == 1);
  if (kind == RECNN_OPT_ADAM) {
    const double bc1 = 1.0 - pow(beta1, (double)t);
    const double bc2 = 1.0 - pow(beta2, (double)t);
    s.step_size = (float)(lr / bc1);
    s.bc2_sqrt = (float)sqrt(bc2);
  } else if (kind == RECNN_OPT_RANGER || kind == RECNN_OPT_RADAM) {
    const double beta2_t = pow(beta2, (double)t);
    const double n_sma_max = 2.0 / (1.0 - beta2) - 1.0;
    const double n_sma = n_sma_max - 2.0 * t * beta2_t / (1.0 - beta2_t);
    // torch_optimizer.RAdam rectifies from N_sma >= 5 on; Ranger past its N_sma_threshhold
    const bool rectify = kind == RECNN_OPT_RADAM ? n_sma >= 5.0 : n_sma > n_sma_threshold;
    double step_size;
    if (rectify) {
      step_size = sqrt((1.0 - beta2_t) * (n_sma - 4.0) / (n_sma_max - 4.0) * (n_sma - 2.0) / n_sma * n_sma_max /
                       (n_sma_max - 2.0)) / (1.0 - pow(beta1, (double)t));
      s.adaptive = 1;
    } else {
      step_size = 1.0 / (1.0 - pow(beta1, (double)t));
    }
    s.step_size = (float)(-step_size * lr);
    s.wd_lr = (float)(-wd * lr);
    s.lookahead = (kind == RECNN_OPT_RANGER && k_look > 0 && t % k_look == 0) ? 1 : 0;
  }
  return s;
}
// one element of torch.optim.SGD / Adam (torch 2.11 single-tensor op order), torch_optimizer.Ranger or its RAdam half
// alone (RECNN_OPT_RADAM: no Lookahead, no slow arena); `grad` already carries any clip scale
__device__ __forceinline__ void opt_apply(int kind, const OptConsts& k, const OptStep& st, int t,
                                          float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                          float* __restrict__ slow, long long i, float grad) {
  const float w = p[i];
  if (kind == RECNN_OPT_RANGER || kind == RECNN_OPT_RADAM) {
    // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1-beta2); exp_avg.mul_(beta1).add_(grad, alpha=1-beta1)
    float vi = __fmul_rn(v[i], k.b2);
    vi = __fadd_rn(vi, __fmul_rn(__fmul_rn(k.one_minus_b2, grad), grad));
    float mi = __fmul_rn(m[i], k.b1);
    mi = __fadd_rn(mi, __fmul_rn(k.one_minus_b1, grad));
    v[i] = vi;
    m[i] = mi;
    float x = w;
    if (k.wd != 0.f) x = __fadd_rn(x, __fmul_rn(st.wd_lr, x));             // p.add_(p, alpha=-wd*lr)
    if (st.adaptive) {
      const float denom = __fadd_rn(__fsqrt_rn(vi), k.eps);                  // exp_avg_sq.sqrt().add_(eps)
      x = __fadd_rn(x, __fdiv_rn(__fmul_rn(st.step_size, mi), denom));       // p.addcdiv_(exp_avg, denom, value=-step_size*lr)
    } else {
      x = __fadd_rn(x, __fmul_rn(st.step_size, mi));                         // p.add_(exp_avg, alpha=-step_size*lr)
    }
    if (kind == RECNN_OPT_RANGER) {
      float sl = st.first ? w : slow[i];               // slow_buffer starts as a copy of the (un-stepped) weights
      if (st.lookahead) {
        sl = __fadd_rn(sl, __fmul_rn(k.alpha, __fsub_rn(x, sl)));            // slow.add_(p - slow, alpha=alpha); p = slow
        x = sl;
      }
      if (st.lookahead || st.first) slow[i] = sl;
    }
    p[i] = x;
    return;
  }
  if (k.wd != 0.f) grad = __fadd_rn(grad, __fmul_rn(k.wd, w));
  if (kind == RECNN_OPT_SGD) {
    if (k.momentum != 0.f) {
      const float buf = (t == 1) ? grad : __fadd_rn(__fmul_rn(k.momentum, m[i]), grad);
      m[i] = buf;
      grad = buf;
    }
    p[i] = __fsub_rn(w, __fmul_rn(k.lr, grad));
  } else {
    float mi = m[i], vi = v[i];
    mi = __fadd_rn(mi, __fmul_rn(k.one_minus_b1, __fsub_rn(grad, mi)));       // lerp_
    vi = __fadd_rn(__fmul_rn(vi, k.b2), __fmul_rn(__fmul_rn(k.one_minus_b2, grad), grad));
    m[i] = mi;
    v[i] = vi;
    const float denom = __fadd_rn(__fdiv_rn(__fsqrt_rn(vi), st.bc2_sqrt), k.eps);
    p[i] = __fsub_rn(w, __fmul_rn(st.step_size, __fdiv_rn(mi, denom)));
  }
}
#endif

// ticket: zero-initialised self-resetting counter; when given, the kernel itself increments *net.opt_t.
// skip: optional device word; when it is non-zero at run time the step does nothing (t included; needs a ticket)
int launch_optimizer(const recnn_optim& o, const recnn_net& net, int64_t count, const float* grad_scale,
                     cudaStream_t st, unsigned* ticket = nullptr, const GradSource* src = nullptr,
                     const unsigned* skip = nullptr);

int launch_bump64(long long* t, cudaStream_t st);
int launch_finish(long long* rng_step, const unsigned* oob, const unsigned* dp_mismatch, float* flags_out,
                  cudaStream_t st);
int launch_polyak(float* target, const float* net, int64_t count, double tau, cudaStream_t st);

}  // namespace recnn
