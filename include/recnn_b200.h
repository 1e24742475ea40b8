/*
 * recnn_b200 -- C ABI of the H100-native RecNN DDPG/TD3 update hot path.
 *
 * The reference (awarebayes/RecNN) is pure Python on PyTorch and has NO FFI:
 * its seams for this path are Python call sites (SURVEY.md 8b).  Each entry
 * point below names the reference function (file:line under /root/reference)
 * whose work it replaces; the Python host layer in recnn_b200/ binds them with
 * ctypes and keeps the reference's own signatures on top (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C types only; every pointer is a DEVICE pointer unless it says host;
 *   - every call takes the CUDA stream to launch on (cudaStream_t as void*);
 *     nothing synchronises, nothing allocates: scratch comes from the caller
 *     (recnn_step_workspace_bytes);
 *   - workspace / scratch pointers may be any address: the size a
 *     *_workspace_bytes / *_scratch_floats query reports includes alignment
 *     slack.  A call that takes workspace_bytes returns RECNN_E_WORKSPACE when
 *     it is below the reported size, before launching anything;
 *   - return 0 on success, a negative RECNN_E_* code otherwise;
 *     recnn_b200_last_error() returns a thread-local message;
 *   - all floating point data is fp32, item indices are int64 (as the
 *     reference's LongTensor), dropout masks are uint8 {0,1}.
 *   - a "net" is one 3-layer MLP stored as ONE flat fp32 arena in
 *     nn.Module.parameters() order: linear1.weight [H,in], linear1.bias [H],
 *     linear2.weight [H,H], linear2.bias [H], linear3.weight [out,H],
 *     linear3.bias [out]  (nn.Linear layout, y = x W^T + b;
 *     recnn/nn/models.py:41-57 Actor, :187-203 Critic).  Every matrix row and every
 *     segment is padded to a multiple of 4 floats (16 bytes, the TMA granule):
 *     recnn_net_layout() returns the offsets and row pitches; pad elements are 0.
 */
#ifndef RECNN_B200_H
#define RECNN_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RECNN_B200_ABI_VERSION 3

#if defined(__GNUC__)
#define RECNN_API __attribute__((visibility("default")))
#else
#define RECNN_API
#endif

enum {
  RECNN_OK = 0,
  RECNN_E_INVALID = -1,   /* bad argument (null pointer, non-positive size ...) */
  RECNN_E_CUDA = -2,      /* a CUDA runtime call / launch failed */
  RECNN_E_WORKSPACE = -3, /* workspace too small */
  RECNN_E_UNSUPPORTED = -4
};

RECNN_API int recnn_b200_abi_version(void);
RECNN_API const char* recnn_b200_last_error(void);
/* number of kernels this library has launched in this process (bench accounting) */
RECNN_API int64_t recnn_b200_launch_count(void);
/* struct-layout probes so a foreign binding can verify its mirror of recnn_step_args */
RECNN_API int64_t recnn_sizeof_step_args(void);
RECNN_API int64_t recnn_offsetof_step_args(int field);

/* ------------------------------------------------------------------ data path */

/* recnn/data/utils.py:51-68 batch_tensor_embeddings: gather table rows for the
 * F+1 items of every sample and assemble state / next_state / action / reward.
 *   table  fp32[n_items, dim] row-major      items   int64[n_rows, frame+1]
 *   ratings fp32[n_rows, frame+1]
 *   state, next_state fp32[n_rows, frame*dim+frame]; action fp32[n_rows, dim];
 *   reward fp32[n_rows].  Any output pointer may be NULL (skipped).
 * Bit-exact copy semantics.  Indices are checked on device; an out-of-range
 * index sets *oob_flag (device int32, may be NULL) and the row reads item 0. */
RECNN_API int recnn_frame_gather(const float* table, int64_t n_items, int dim,
                       const int64_t* items, const float* ratings,
                       int64_t n_rows, int frame,
                       float* state, float* next_state, float* action, float* reward,
                       int* oob_flag, void* stream);

/* recnn/data/utils.py:70-71: done = zeros(n_rows); done[cumsum(sizes-frame)-1] = 1.
 * sizes int64[n_users] (device). */
RECNN_API int recnn_done_from_sizes(const int64_t* sizes, int64_t n_users, int frame,
                          float* done, int64_t n_rows, void* stream);

/* Device-resident FrameEnv feed.  The reference builds every minibatch on the host, inside a
 * DataLoader worker: UserDataset.__getitem__ (recnn/data/env.py:47-64) hands out one user's
 * time-ordered items / ratings, and the collate function cuts ALL length-(frame+1) sliding
 * windows of every user of the batch and concatenates them (rolling_window, recnn/data/utils.py:7-10;
 * prepare_batch_static_size, :161-181; ratings cast with .float(), :178).  Here the histories stay in
 * HBM as a CSR over users
 *     hist_items int64[total]   hist_ratings fp32[total] (the .float() cast, done once)
 *     hist_offsets int64[n_users+1]
 * and the windows are cut on the device: the only per-minibatch input is the list of users.
 * Outputs are exactly what the collate hands to embed_batch: items int64[n_rows, frame+1],
 * ratings fp32[n_rows, frame+1] (feed them to recnn_frame_gather or to the frame form of
 * recnn_ddpg_step / recnn_td3_step), plus done fp32[n_rows] (recnn/data/utils.py:70-71:
 * 1 on the last window of every user) and sizes int64[n_batch] (history lengths, :171).
 * Any output pointer may be NULL.  Bit-exact (copies only).
 *   batch_users int64[n_batch]    positions of the minibatch's users in the CSR, in batch order
 *   row_offsets int64[n_batch+1]  exclusive prefix sum of (length - frame) over batch_users;
 *                                 n_rows == row_offsets[n_batch] (host-side plan: lengths are
 *                                 known to the caller, so no device->host sync is needed)
 * A user index out of range, or a plan that disagrees with the resident lengths, sets *err_flag
 * (device int32, may be NULL) and zero-fills the affected rows. */
RECNN_API int recnn_window_gather_users(const int64_t* hist_items, const float* hist_ratings,
                              const int64_t* hist_offsets, int64_t n_users,
                              const int64_t* batch_users, const int64_t* row_offsets, int64_t n_batch,
                              int frame, int64_t n_rows,
                              int64_t* items, float* ratings, float* done, int64_t* sizes,
                              int* err_flag, void* stream);

/* Fixed-size minibatch over the same CSR: row n is the window with GLOBAL id window_ids[n], windows
 * being numbered user by user in storage order (win_offsets int64[n_users+1] = exclusive prefix sum
 * of max(length - frame, 0)).  Equals rows window_ids of the reference collate over ALL users
 * (prepare_batch_static_size over the whole UserDataset, recnn/data/utils.py:161-181), so a
 * replay-style sampler can draw a constant number of rows per step (constant shapes keep the update
 * step one CUDA graph).  users_out int64[n_rows] (optional) = CSR position of each row's user;
 * done = 1 where the window is its user's last.  Out-of-range ids set *err_flag and zero-fill. */
RECNN_API int recnn_window_gather_ids(const int64_t* hist_items, const float* hist_ratings,
                            const int64_t* hist_offsets, const int64_t* win_offsets, int64_t n_users,
                            const int64_t* window_ids, int frame, int64_t n_rows,
                            int64_t* items, float* ratings, float* done, int64_t* users_out,
                            int* err_flag, void* stream);

/* ------------------------------------------------------------------ networks */

typedef struct recnn_dims {
  int32_t state_dim;   /* S = frame*dim + frame (1290) */
  int32_t action_dim;  /* A (128) */
  int32_t hidden;      /* H (256) */
  int32_t reserved;
} recnn_dims;

/* number of fp32 in an Actor / Critic arena for these dims (padding included) */
RECNN_API int64_t recnn_actor_param_count(const recnn_dims* d);
RECNN_API int64_t recnn_critic_param_count(const recnn_dims* d);

/* arena geometry: offsets (in floats) of w1,b1,w2,b2,w3,b3 then the row pitches of w1,w2,w3,
 * then the total count -> out[10].  is_critic selects in = S+A / out = 1. */
RECNN_API int recnn_net_layout(const recnn_dims* d, int is_critic, int64_t* out);

/* recnn/nn/models.py:59-73 Actor.forward.  masks: two uint8[n_rows,H] arrays
 * (train mode: h = relu(z) * mask * 2) or NULL,NULL for eval().  apply_tanh as
 * the reference's `tanh` argument.  scratch: fp32[recnn_forward_scratch_floats(d, n_rows, 0)]
 * (two hidden activations + a 16-byte-pitch image of `state` when its row pitch is not a 16-byte multiple,
 * so that every layer runs on the tensor cores). */
RECNN_API int64_t recnn_forward_scratch_floats(const recnn_dims* d, int64_t n_rows, int is_critic);
RECNN_API int recnn_actor_forward(const recnn_dims* d, const float* params, const float* state,
                        int64_t n_rows, const uint8_t* mask1, const uint8_t* mask2,
                        int apply_tanh, float* action_out, float* scratch, void* stream);

/* recnn/nn/models.py:205-213 Critic.forward (concat is virtual).  value_out fp32[n_rows];
 * scratch: fp32[recnn_forward_scratch_floats(d, n_rows, 1)]. */
RECNN_API int recnn_critic_forward(const recnn_dims* d, const float* params, const float* state,
                         const float* action, int64_t n_rows,
                         const uint8_t* mask1, const uint8_t* mask2,
                         float* value_out, float* scratch, void* stream);

/* One nn.Linear (+ optional ReLU) on its own: out[n_rows,out_dim] = act(x W^T + b)
 * (recnn/nn/models.py:52-54 layers; exposed so a single layer can be timed / reused). */
RECNN_API int recnn_linear_forward(const float* x, int64_t n_rows, int in_dim, const float* weight,
                         const float* bias, int out_dim, int relu, float* out, void* stream);

/* Generic contraction C[M,N] (pitch ldc) = A . B^T, the building block of every Linear
 * forward/backward in this path (torch addmm sites: recnn/nn/models.py:66-70, :207-212 and
 * their autograd backward).  a_mn=0: A is [M,K] row-major, a_mn=1: A is stored [K,M];
 * same for B with N.  recnn_gemm_tf32x3 runs on the Hopper tensor cores (wgmma) with
 * error-compensated 3xTF32 (fp32-grade accuracy; pitches and bases must be 16-byte
 * multiples; tile_n in {0 (auto), 64, 128}); recnn_gemm_fp32 is the exact-fp32
 * CUDA-core path for arbitrary shapes. */
RECNN_API int recnn_gemm_tf32x3(int M, int N, int K, const float* A, int64_t lda, int a_mn, const float* B,
                      int64_t ldb, int b_mn, float* C, int64_t ldc, int tile_n, void* stream);
RECNN_API int recnn_gemm_fp32(int M, int N, int K, const float* A, int64_t lda, int a_mn, const float* B,
                    int64_t ldb, int b_mn, float* C, int64_t ldc, void* stream);

/* recnn/utils/misc.py:1-5 soft_update over one flat arena:
 * target = target*(1-tau) + net*tau   (tau==1 is an exact copy, as in the reference) */
RECNN_API int recnn_polyak_update(float* target, const float* net, int64_t count, double tau, void* stream);

/* ------------------------------------------------------------------ update step */

typedef struct recnn_net {
  float* params;      /* arena */
  float* grads;       /* arena, same layout; NULL for target nets */
  float* opt_m;       /* Adam exp_avg / SGD momentum buffer (built-in optimizers), else NULL */
  float* opt_v;       /* Adam exp_avg_sq, else NULL */
  int32_t* opt_t;     /* device int32: number of optimizer steps taken so far */
  float* opt_slow;    /* Ranger: Lookahead slow weights (arena), else NULL */
} recnn_net;

/* RANGER = RAdam + Lookahead as in torch_optimizer.Ranger, the optimizer recnn.nn.DDPG/TD3 construct by default
 * (recnn/nn/algo.py:84-89, :139-147).  torch_optimizer is an un-vendored third-party dependency of the reference
 * (requirements.txt:7, unpinned) and absent from this environment: the restatement follows the published algorithm
 * (Liu et al. 2019 rectified Adam with the N_sma_threshhold switch; Zhang et al. 2019 Lookahead every k steps) and
 * its parity with the package is UNPINNED (DESIGN.md section 2). */
/* RADAM = Ranger's RAdam half alone (torch_optimizer.RAdam: rectified from N_sma >= 5, decoupled weight decay, no
 * Lookahead and no slow arena), the optimizer of the Top-K notebook's behaviour policy (recnn_beta_step).  Pinned
 * against torch.optim.RAdam(decoupled_weight_decay=True); parity with the package is UNPINNED as for Ranger. */
enum { RECNN_OPT_EXTERNAL = 0, RECNN_OPT_SGD = 1, RECNN_OPT_ADAM = 2, RECNN_OPT_RANGER = 3, RECNN_OPT_RADAM = 4 };

typedef struct recnn_optim {   /* torch.optim.SGD / torch.optim.Adam / torch_optimizer.Ranger semantics */
  int32_t kind;
  int32_t k;          /* Ranger: Lookahead period (6) */
  /* doubles: torch keeps these as python floats and rounds to fp32 only where the
   * tensor op consumes them (e.g. step_size = lr / (1 - beta1**t) is formed in double) */
  double lr, beta1, beta2, eps, weight_decay, momentum;
  double alpha;            /* Ranger: Lookahead interpolation (0.5) */
  double n_sma_threshold;  /* Ranger: rectification switch (5) */
} recnn_optim;

/* what one call executes; OR them.  A drop-in single-GPU step passes RECNN_PH_ALL.
 * Multi-GPU data parallel and external torch optimizers split the step at the
 * two points where gradients are complete. */
enum {
  RECNN_PH_VALUE_GRAD = 1,   /* targets, TD target, value loss, critic backward        */
  RECNN_PH_VALUE_OPT = 2,    /* built-in critic optimizer step(s)                      */
  RECNN_PH_POLICY_LOSS = 4,  /* pi(s), Q(s,pi(s)) with the *updated* critic, loss      */
  RECNN_PH_POLICY_GRAD = 8,  /* actor backward through the critic (policy steps only)  */
  RECNN_PH_POLICY_OPT = 16,  /* L1 "clip" quirk (+ built-in actor optimizer step)      */
  RECNN_PH_SOFT_UPDATE = 32, /* Polyak target updates (policy steps only)              */
  RECNN_PH_GATHER = 64,      /* frame form: materialise state/next_state/action into the
                              * workspace (split-phase callers pass it once per step)  */
  RECNN_PH_FINISH = 128,     /* end of step: error bits -> losses[4], copy losses to losses_host (if set), ++*rng_step */
  RECNN_PH_ALL = 255
};

enum { RECNN_ALGO_DDPG = 0, RECNN_ALGO_TD3 = 1 };

/* Peer-memory communicator of the data-parallel step (see "data parallel" below); opaque. */
typedef struct recnn_comm recnn_comm;

typedef struct recnn_step_args {
  int32_t algo;            /* RECNN_ALGO_* */
  int32_t phases;          /* RECNN_PH_* mask */
  int32_t learn;           /* reference `learn` flag */
  int32_t do_policy_step;  /* learn && step % policy_step == 0 (ddpg.py:89 / td3.py:130) */
  recnn_dims dims;

  /* batch: EITHER dense (state,next_state,action) OR frames (table,items,ratings).
   * reward/done fp32[n_rows] may be NULL in frame form for reward (= ratings[:,F]). */
  int64_t n_rows;          /* rows in this call (this rank's shard)          */
  int64_t n_rows_global;   /* denominator of the batch means (all ranks)     */
  const float* state;
  const float* next_state;
  const float* action;
  const float* table;
  int64_t n_items;
  int32_t frame;
  int32_t emb_dim;
  const int64_t* items;
  const float* ratings;
  const float* reward;
  const float* done;

  /* nets.  DDPG: value[0], target_value[0].  TD3: [0] and [1]. */
  recnn_net policy, target_policy;
  recnn_net value[2], target_value[2];
  recnn_optim policy_optim, value_optim;

  /* hyper-parameters (recnn/nn/algo.py:103-109, :164-174) */
  float gamma, min_value, max_value, noise_std, noise_clip;
  int32_t dropout;         /* 1: online nets are in train() mode (Dropout p=.5 active) */
  double soft_tau;

  /* randomness.  Parity mode: explicit masks (uint8[n_rows,H]) in the reference's
   * drop_layer call order -- DDPG: value(2) policy(2) value(2); TD3: value1(2)
   * value2(2) policy(2) value1(2) -- and the raw N(0,noise_std) draw fp32[n_rows,A].
   * Perf mode: all NULL; Philox4x32-10 keyed by (seed, *rng_step) on device. */
  const uint8_t* masks[8];
  const float* noise;
  uint64_t seed;
  int64_t* rng_step;         /* device int64 counter; read by every phase, incremented by RECNN_PH_FINISH */

  /* outputs */
  float* losses;           /* device, 8 words: fp32 value(1), value2, policy, ||actor grad||_1; then one int32 of
                            * error bits written by RECNN_PH_FINISH (1: an item id of the frame-form batch was outside
                            * [0, n_items) -- such rows read table row 0; 2: the ranks of a data-parallel step
                            * disagree on n_rows_global); 3 spare words */
  float* losses_host;      /* optional PINNED host buffer of 8 words: RECNN_PH_FINISH copies `losses` here (async) */
  float* next_action_out;  /* optional fp32[n_rows,A] (debug["next_action"]) */
  float* gen_action_out;   /* optional fp32[n_rows,A] (debug["gen_action"])  */
  /* optional fp32[n_rows,A]: the target policy's action on next_state, computed by the caller.  When given the
   * step does not run a target policy of its own (policy / target_policy may then be all-NULL for a call made only of
   * the VALUE phases): this is how misc.py:28 is served when the policy is not an Actor -- the REINFORCE critic is
   * updated against DiscreteActor probabilities (recnn/nn/update/reinforce.py:92-102). */
  const float* next_action_in;

  void* workspace;
  int64_t workspace_bytes;

  /* data parallel (optional, NULL on one GPU): when set, the step all-reduces (sums) the gradient
   * arenas over the communicator's ranks before each optimizer update, and the three loss scalars
   * before RECNN_PH_FINISH, with kernels on `stream` -- no host-side collective between phases.
   * Each rank passes its shard (n_rows local, n_rows_global = total). */
  const recnn_comm* comm;
} recnn_step_args;

/* bytes of scratch a step with these shapes needs (frame form included). */
RECNN_API int64_t recnn_step_workspace_bytes(const recnn_dims* d, int64_t n_rows, int32_t algo);

/* recnn/nn/update/ddpg.py:8-104 (with misc.py:10-55 value_update inlined). */
RECNN_API int recnn_ddpg_step(const recnn_step_args* args, void* stream);
/* recnn/nn/update/td3.py:8-150. */
RECNN_API int recnn_td3_step(const recnn_step_args* args, void* stream);

/* built-in optimizer step on one arena, exposed for recnn_b200.optim
 * (torch.optim.Adam/SGD semantics; increments *net->opt_t).
 * grad_scale: optional device scalar the gradient is multiplied by first. */
RECNN_API int recnn_optimizer_step(const recnn_optim* o, const recnn_net* net, int64_t count,
                         const float* grad_scale, void* stream);

/* ---- serving: nearest-item retrieval over the embedding table ----------------------------------
 * The step after Actor.forward in the reference's serving examples: the generated action (a 128-d
 * embedding) is matched against the item matrix -- examples/streamlit_demo.py:189-203 (faiss
 * IndexFlatL2 / IndexFlatIP / IndexFlatIP over L2-normalised rows), recnn/data/db_con.py:45-56
 * (MilvusConnection.search(search_vecs, topk) -> ids, distances).  Exact search: one
 * [n_queries, dim] x [dim, n_items] contraction on the tensor cores (3xTF32) + an exact top-k.
 * Ordering: best first; L2 reports the squared distance (as faiss / Milvus do), IP the inner product,
 * COS the cosine similarity; ties go to the smaller item id.  k <= 64. */
enum { RECNN_METRIC_L2 = 0, RECNN_METRIC_IP = 1, RECNN_METRIC_COS = 2 };
/* out[n_items]: |item|^2 (L2) or 1/|item| (COS); computed once per table ("index build") */
RECNN_API int recnn_item_norms(const float* table, int64_t n_items, int32_t dim, int32_t metric, float* out,
                               void* stream);
RECNN_API int64_t recnn_retrieve_workspace_bytes(int64_t n_queries, int64_t n_items, int32_t k);
/* ids_out int64[n_queries, k], dist_out fp32[n_queries, k]; norms from recnn_item_norms (NULL for IP);
 * workspace: any address, workspace_bytes >= recnn_retrieve_workspace_bytes (else RECNN_E_WORKSPACE) */
RECNN_API int recnn_retrieve_topk(const float* queries, int64_t n_queries, int32_t dim, const float* table,
                                  int64_t n_items, const float* norms, int32_t metric, int32_t k,
                                  int64_t* ids_out, float* dist_out, void* workspace, int64_t workspace_bytes,
                                  void* stream);

/* ---- REINFORCE with (Top-K) off-policy correction: the policy side (SURVEY 8f-2) ------------------
 * DiscreteActor (recnn/nn/models.py:76-99): probs = softmax(W2 relu(W1 s + b1) + b2), one output per item.
 * Parameter arena in nn.Module.parameters() order -- linear1.weight [H, S], linear1.bias, linear2.weight
 * [num_items, H], linear2.bias -- matrix rows padded to 16-byte multiples (recnn_discrete_layout). */
typedef struct recnn_discrete_dims {
  int32_t state_dim, hidden, num_items, reserved;
} recnn_discrete_dims;
/* out[7]: offsets of w1, b1, w2, b2; row pitches of w1, w2; total float count */
RECNN_API int recnn_discrete_layout(const recnn_discrete_dims* d, int64_t* out);
/* floats of scratch for n_rows rows: forward only (backward = 0) or recnn_reinforce_policy_grad (backward = 1) */
RECNN_API int64_t recnn_discrete_scratch_floats(const recnn_discrete_dims* d, int64_t n_rows, int32_t backward);
/* DiscreteActor.forward (models.py:95-99): probs_out fp32 [n_rows, num_items] dense */
RECNN_API int recnn_discrete_forward(const recnn_discrete_dims* d, const float* params, const float* state,
                                     int64_t n_rows, float* probs_out, float* scratch, void* stream);
/* Categorical(probs).sample() + .log_prob(sample) (models.py:107-110, 121-143): inverse CDF on `uniforms`
 * [n_rows] in [0,1) when given (replayable), else on Philox(seed, draw, row).  probs fp32 [n_rows, ld >= num_items];
 * rows are normalised by their sum and clamped to [eps, 1-eps] before the log, as torch does. */
RECNN_API int recnn_categorical_sample(const float* probs, int64_t n_rows, int32_t num_items, int64_t ld,
                                       const float* uniforms, uint64_t seed, int64_t draw, int64_t* action_out,
                                       float* log_prob_out, void* stream);
/* Categorical(probs).log_prob(action) for given actions; *oob_flag (may be NULL) is set when an id is out of range */
RECNN_API int recnn_categorical_log_prob(const float* probs, int64_t n_rows, int32_t num_items, int64_t ld,
                                         const int64_t* action, float* log_prob_out, int32_t* oob_flag, void* stream);
/* ChooseREINFORCE (recnn/nn/update/reinforce.py:10-65): the three policy losses */
enum { RECNN_REINFORCE_BASIC = 0, RECNN_REINFORCE_CORRECTED = 1, RECNN_REINFORCE_TOPK = 2 };
/* Policy loss and its gradient over the n_rows rows saved since the last policy update (the reference's
 * saved_log_probs / correction / lambda_k lists, concatenated): state [n_rows, state_dim], action int64 [n_rows]
 * (the sampled item), beta_log_prob [n_rows] (NULL for BASIC), returns [n_rows] (the normalised discounted return of
 * the env step the row was saved at, reinforce.py:44-52).  Recomputes the forward, writes the gradient of every
 * parameter into `grads` (arena geometry; overwritten, i.e. zero_grad + backward), out[0] = loss (fp32),
 * out[1] = int32 flag: an action id was outside [0, num_items) (that row contributed nothing). */
RECNN_API int recnn_reinforce_policy_grad(const recnn_discrete_dims* d, const float* params, float* grads,
                                          const float* state, const int64_t* action, const float* beta_log_prob,
                                          const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                          float* out, float* scratch, void* stream);
/* The same gradient without the [n_rows, num_items] logits: the items are visited in chunks of chunk_items (num_items,
 * or a positive multiple of 128 below it; the last chunk may be narrower), twice -- per-row softmax statistics, then
 * the chunk's logits recomputed and back-propagated.  Scratch (recnn_reinforce_scratch_floats) holds one
 * [n_rows, chunk_items] chunk and does not grow with num_items.  recnn_reinforce_policy_grad is this call with
 * chunk_items = num_items.  Deterministic: fixed chunk order, no atomics. */
RECNN_API int recnn_reinforce_policy_grad_chunked(const recnn_discrete_dims* d, const float* params, float* grads,
                                                  const float* state, const int64_t* action, const float* beta_log_prob,
                                                  const float* returns, int64_t n_rows, int32_t method, int32_t top_k,
                                                  int32_t chunk_items, float* out, float* scratch, void* stream);
/* floats of scratch for recnn_reinforce_policy_grad_chunked; 0 when chunk_items is not accepted */
RECNN_API int64_t recnn_reinforce_scratch_floats(const recnn_discrete_dims* d, int64_t n_rows, int32_t chunk_items);

/* ---- REINFORCE: the policy sharded over the item vocabulary across the GPUs of one node -----------
 * Rank `rank` of `world` holds rows [item_offset, item_offset + d->num_items) of linear2 (weight and bias) in its
 * arena: d is the LOCAL dims, so recnn_discrete_layout applies unchanged; linear1 is replicated.  Action ids stay
 * global.  The host issues the phases on one stream with two exchanges between them (recnn_comm_allgather of the
 * records below, and recnn_comm_allreduce of the layer-1 gradient), so a sharded update stays graph-capturable.
 * A record (recnn_vocab_record_floats(n_rows) floats) is a header of four int32 words {lo, hi, num_items, n_rows}
 * followed by three planes of n_rows floats: the local max of the logits, the local sum of exp(z - max) and the logit
 * of the row's action (from the rank that owns it, 0 on the others).  "gathered" is the W records in rank order.
 * Every rank merges them in rank order, so all ranks compute the same bits; at world 1 every phase computes exactly
 * what the unsharded call does. */
typedef struct recnn_vocab_shard {
  int32_t item_offset;   /* the global id of the rank's first item */
  int32_t num_items;     /* the whole vocabulary */
  int32_t rank, world;
} recnn_vocab_shard;
RECNN_API int64_t recnn_vocab_record_floats(int64_t n_rows);
/* Policy gradient, phase 1: the hidden layer, then pass 1 over the local items in chunks of chunk_items -> record.
 * scratch: fp32[recnn_reinforce_scratch_floats(d, n_rows, chunk_items)] (local dims; it does not grow with the
 * vocabulary once chunk_items < d->num_items); phase 2 must get the same scratch, untouched in between. */
RECNN_API int recnn_reinforce_shard_stats(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                          const float* state, const int64_t* action, int64_t n_rows,
                                          int32_t chunk_items, float* record, float* scratch, void* stream);
/* Phase 2, after the all-gather: merge the gathered records, row weights and loss, pass 2 over the local chunks
 * (dW2 / db2 of the local rows), then this rank's share of the layer-1 gradient into grads[0 : w2 offset) -- the
 * caller all-reduces that block (recnn_comm_allreduce) to get dW1 / db1.  out[0] = loss (same bits on every rank);
 * out[1] = int32 flag: an action id was outside [0, num_items) (that row contributed nothing); out[2] = int32 flag:
 * the gathered headers do not tile the vocabulary in rank order with this rank's rows (the ranks disagree on the
 * shard plan or on n_rows; the gradient is then meaningless). */
RECNN_API int recnn_reinforce_shard_grad(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                         float* grads, const float* state, const int64_t* action,
                                         const float* beta_log_prob, const float* returns, int64_t n_rows,
                                         int32_t method, int32_t top_k, int32_t chunk_items, const float* gathered,
                                         float* out, float* scratch, void* stream);
/* Forward: the local logits into probs_out [n_rows, d->num_items] and the record (action-logit plane 0).
 * scratch: fp32[recnn_discrete_scratch_floats(d, n_rows, 0)] */
RECNN_API int recnn_discrete_shard_forward(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                           const float* params, const float* state, int64_t n_rows, float* probs_out,
                                           float* record, float* scratch, void* stream);
/* ... after the all-gather: probs <- exp(z - M) / S, the rank's column block of the softmax over the whole vocabulary.
 * *error_flag <- 1 when the headers disagree (as out[2] above). */
RECNN_API int recnn_discrete_shard_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                          const float* gathered, int64_t n_rows, float* probs, int32_t* error_flag,
                                          void* stream);
/* One draw per row over the whole vocabulary (u as recnn_categorical_sample: uniforms, or Philox(seed, draw, row) --
 * the same u on every rank).  From the gathered records every rank finds the rank whose share of the cumulative mass
 * holds u; that rank draws inside its block at the conditional uniform.  draw_record [2, n_rows]: the global id as
 * int32 bits (-1 on every rank but the owner), then its log-prob.  Exchange it with recnn_comm_allgather and read it
 * with recnn_discrete_shard_pick. */
RECNN_API int recnn_discrete_shard_sample(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                          const float* gathered, const float* probs, int64_t n_rows,
                                          const float* uniforms, uint64_t seed, int64_t draw, float* draw_record,
                                          void* stream);
/* The log-prob of given global ids (probs: the finished block), as a draw record; *oob_flag when an id is out of range */
RECNN_API int recnn_discrete_shard_log_prob(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                            const float* probs, int64_t n_rows, const int64_t* action,
                                            float* draw_record, int32_t* oob_flag, void* stream);
/* gathered draw records [world][2][n_rows] -> action_out int64 [n_rows], log_prob_out [n_rows]; *error_flag <- 1 when
 * a row was claimed by no rank or by several (the ranks used different uniforms, or an id was out of range) */
RECNN_API int recnn_discrete_shard_pick(int32_t world, const float* gathered_draws, int64_t n_rows,
                                        int64_t* action_out, float* log_prob_out, int32_t* error_flag, void* stream);

/* ---- REINFORCE: serving the policy's top-k items ---------------------------------------------------
 * torch.topk(DiscreteActor(state), k) without the [n_rows, num_items] probabilities: the hidden layer once, then the
 * items in chunks of chunk_items (num_items, or a positive multiple of 128 below it; the last chunk may be narrower).
 * Each chunk's logits fold into the row's running max and sum of exp (the reduction of recnn_discrete_forward) and its
 * best candidates merge into a running list of k per row.  Items are ranked by logit, equal logits to the smaller id;
 * values_out fp32 [n_rows, k] = exp(z - M) / S over ALL items (M, S: the row's max and sum of exp), descending;
 * ids_out int64 [n_rows, k].  With one chunk the values equal recnn_discrete_forward's probabilities bit for bit.
 * exclude: NULL or int64 [n_rows, n_exclude] (n_exclude <= 256); those ids are never returned but stay in S (the
 * values are pi's, not renormalised); negative ids are padding.  When a row has fewer than k eligible items the last
 * slots are id -1, value 0.  *error_flag <- bits: 1 = an excluded id is >= num_items.  1 <= k <= min(64, num_items).
 * workspace: any address, workspace_bytes >= recnn_discrete_topk_workspace_bytes (else RECNN_E_WORKSPACE); it holds
 * one [n_rows, chunk_items] logits block and a few [n_rows, k] lists, so it does not grow with num_items once
 * chunk_items < num_items.  Deterministic: fixed chunk order, no atomics on the results. */
RECNN_API int64_t recnn_discrete_topk_workspace_bytes(const recnn_discrete_dims* d, int64_t n_rows, int32_t k,
                                                      int32_t chunk_items);   /* 0 when k is outside [1, 64] or chunk_items is refused */
RECNN_API int recnn_discrete_topk(const recnn_discrete_dims* d, const float* params, const float* state,
                                  int64_t n_rows, int32_t k, const int64_t* exclude, int32_t n_exclude,
                                  int32_t chunk_items, float* values_out, int64_t* ids_out, int32_t* error_flag,
                                  void* workspace, int64_t workspace_bytes, void* stream);
/* The same on a vocabulary-sharded policy (d: the LOCAL dims; k <= the whole vocabulary, and may exceed the rank's
 * block).  shard_topk runs the passes over the rank's items [lo, hi) with global candidate ids and writes a record of
 * recnn_vocab_topk_record_floats(n_rows, k) floats: the header {lo, hi, num_items, n_rows}, the local max and sum-of-exp
 * planes, then k logit planes and k id planes (int32 bits), plane j holding every row's j-th best local candidate (a
 * block of fewer than k eligible items pads with logit -FLT_MAX, id -1).  workspace as recnn_discrete_topk with the
 * local dims.  After recnn_comm_allgather of the records (rank order), shard_topk_finish merges M and S in rank order as
 * recnn_discrete_shard_finish does and k-way merges the W lists (world <= 32): every rank writes the same bits, and at
 * world 1 the pair computes exactly what recnn_discrete_topk does.  *error_flag <- bits: 1 = an excluded id is >=
 * num_items; 2 = the headers do not tile the vocabulary in rank order with this rank's block (the result is then
 * meaningless). */
RECNN_API int64_t recnn_vocab_topk_record_floats(int64_t n_rows, int32_t k);
RECNN_API int recnn_discrete_shard_topk(const recnn_discrete_dims* d, const recnn_vocab_shard* v, const float* params,
                                        const float* state, int64_t n_rows, int32_t k, const int64_t* exclude,
                                        int32_t n_exclude, int32_t chunk_items, float* record, void* workspace,
                                        int64_t workspace_bytes, void* stream);
RECNN_API int recnn_discrete_shard_topk_finish(const recnn_discrete_dims* d, const recnn_vocab_shard* v,
                                               const float* gathered, int64_t n_rows, int32_t k,
                                               const int64_t* exclude, int32_t n_exclude, float* values_out,
                                               int64_t* ids_out, int32_t* error_flag, void* stream);

/* ---- REINFORCE: the critic side with item-id actions ---------------------------------------------
 * The REINFORCE critic is a Critic(S, num_items, H) (recnn/nn/update/reinforce.py:92-102): layer 1 is W1 [H, S + num_items]
 * on [state | action], the action being a one-hot row (the batch) or a probability row (the target policy's output).
 * These calls never form a [n_rows, num_items] matrix: the action block W1a = W1[:, S:] enters layer 1 as an [n_rows, H]
 * "action term" added in its epilogue -- W1[:, S + a] for an item id a, or probs W1a^T streamed over item chunks.
 * d: the critic's dims (action_dim = num_items); pd: the DiscreteActor's (equal state_dim and num_items).
 * chunk_items: num_items, or a positive multiple of 128 below it; scratch does not grow with num_items below it. */
/* out [n_rows, H] = probs W1a^T, with probs = DiscreteActor(policy_params)(state) (softmax folded over the chunks with a
 * running max and sum, one pass) or the dense probs [n_rows, probs_ld] (policy_params NULL).  W1a is critic_params' */
RECNN_API int64_t recnn_critic_action_term_scratch_floats(const recnn_dims* d, const recnn_discrete_dims* pd,
                                                          int64_t n_rows, int32_t chunk_items);
RECNN_API int recnn_critic_action_term_chunked(const recnn_dims* d, const float* critic_params,
                                               const recnn_discrete_dims* pd, const float* policy_params,
                                               const float* state, const float* probs, int64_t probs_ld,
                                               int64_t n_rows, int32_t chunk_items, float* out, float* scratch,
                                               void* stream);
/* Critic.forward (models.py:205-213) with the action block given as its action term [n_rows, H] (from the call above);
 * scratch: fp32[recnn_forward_scratch_floats(d, n_rows, 0)] */
RECNN_API int recnn_critic_forward_action_term(const recnn_dims* d, const float* params, const float* state,
                                               const float* action_term, int64_t n_rows, const uint8_t* mask1,
                                               const uint8_t* mask2, float* value_out, float* scratch, void* stream);

typedef struct recnn_discrete_value_args {
  recnn_dims dims;                  /* the critic: state_dim, action_dim = num_items, hidden */
  recnn_discrete_dims policy_dims;  /* the target DiscreteActor */
  int32_t learn;                    /* 0: loss only */
  int32_t dropout;                  /* 1: the online critic is in train() mode */
  int32_t chunk_items;
  int32_t reserved;
  int64_t n_rows;
  const float* state;               /* [n_rows, state_dim] */
  const float* next_state;          /* [n_rows, state_dim] */
  const int64_t* action;            /* [n_rows] item ids (the batch's one-hot action, as indices) */
  const float* reward;              /* [n_rows] */
  const float* done;                /* [n_rows] */
  recnn_net value, target_value;
  const float* target_policy;       /* DiscreteActor arena (recnn_discrete_layout) */
  recnn_optim value_optim;          /* RECNN_OPT_EXTERNAL: the gradient is left in value.grads */
  float gamma, min_value, max_value;
  int32_t reserved2;
  const uint8_t* masks[2];          /* the online critic's two dropout masks uint8 [n_rows, H], or NULL (Philox) */
  uint64_t seed;
  int64_t* rng_step;                /* device int64, read by the dropout and incremented at the end of the call */
  float* losses;                    /* device, 8 words: [0] value loss, [4] int32 error bits (1: an action id was outside
                                     * [0, num_items) -- its row used a zero action column and added no gradient) */
  float* losses_host;               /* optional pinned host copy of `losses` */
  void* workspace;
  int64_t workspace_bytes;
} recnn_discrete_value_args;
RECNN_API int64_t recnn_sizeof_discrete_value_args(void);
RECNN_API int64_t recnn_discrete_value_workspace_bytes(const recnn_dims* d, const recnn_discrete_dims* pd,
                                                       int64_t n_rows, int32_t chunk_items);
/* misc.py:10-55 with a DiscreteActor target policy and item-id actions: TD target through the chunked action term of
 * the target critic, online critic with the gathered action columns, MSE, backward (the action block of dW1 is zero
 * except in the selected columns, each the ascending-row sum of its rows' dz1: deterministic), optimizer. */
RECNN_API int recnn_discrete_value_step(const recnn_discrete_value_args* args, void* stream);

/* ---- REINFORCE: the item-id critic sharded over the item vocabulary, with the policy ---------------
 * Rank `rank` of `world` holds the action block W1a[:, lo : hi) of the critic and of the target critic, lo =
 * v->item_offset and hi = lo + args->dims.action_dim, and rows [lo, hi) of the target policy (recnn_vocab_shard above,
 * the same plan).  args carries the LOCAL dims: each arena is laid out as a Critic(S, hi - lo, H) / DiscreteActor with
 * hi - lo items; layer 1's state block, its bias and layers 2 and 3 are replicated.  Action ids stay global.  The step
 * is three phases on one stream with two exchanges between them:
 *   begin  -> record (recnn_vocab_record_floats(n_rows): header {lo, hi, num_items, n_rows}, then the local max and
 *             sum of exp of the target policy's logits, and a zero action-logit plane) -> all-gather (recnn_comm_allgather)
 *   merge  -> terms [2, n_rows, H] = {this rank's part of the target action term, rescaled to the merged max and
 *             divided by the merged sum; W1a one-hot(action) over the ids this rank holds (0 rows elsewhere)}
 *          -> all-reduce of terms (recnn_comm_allreduce)
 *   end    -> the rest of recnn_discrete_value_step from the target critic on, with the summed terms.
 * After the all-reduce every rank holds the same terms, so the loss and the gradient of every replicated block are the
 * same bits on every rank and need no exchange; the action block's gradient is rank-local (the columns of the ids it
 * holds).  The phases share args->workspace (recnn_discrete_value_workspace_bytes of the local dims: it does not grow
 * with the vocabulary once chunk_items < action_dim), which must be left untouched between them.  At world 1 the three
 * phases compute exactly what recnn_discrete_value_step does.  losses[4] error bits: 1 as for the step (an id outside
 * [0, v->num_items), flagged on every rank); 2: the gathered headers do not tile the vocabulary in rank order with this
 * rank's block, or the ranks disagree on n_rows (the result is then meaningless). */
RECNN_API int recnn_discrete_value_shard_begin(const recnn_discrete_value_args* args, const recnn_vocab_shard* v,
                                               float* record, void* stream);
RECNN_API int recnn_discrete_value_shard_merge(const recnn_discrete_value_args* args, const recnn_vocab_shard* v,
                                               const float* gathered, float* terms, void* stream);
RECNN_API int recnn_discrete_value_shard_end(const recnn_discrete_value_args* args, const recnn_vocab_shard* v,
                                             const float* terms, void* stream);

/* ---- REINFORCE with Top-K correction: the behaviour policy beta ------------------------------------
 * The reference ships beta in its Top-K notebook, not in the library (examples/2. REINFORCE TopK Off Policy
 * Correction/3. TopK Reinforce Off Policy Correction.ipynb, cell 3: class Beta), and DiscreteActor.pi_beta_sample
 * (recnn/nn/models.py:113-145) calls its forward once per env step.  Beta is nn.Sequential(nn.Linear(S, num_items),
 * nn.Softmax()) trained by every forward(state, action): p = softmax(W s + b) (dim 1);
 * loss = CrossEntropyLoss(p, action.argmax(1)) -- applied to the PROBABILITIES, a softmax of a softmax, reproduced on
 * purpose; zero_grad, backward, optim.step() (torch_optimizer.RAdam(lr=1e-5, weight_decay=1e-5)); the pre-step p is
 * returned.  Parameter arena: net.0.weight [num_items, S] with row pitch pad4(S), then net.0.bias [num_items]. */
typedef struct recnn_beta_dims {
  int32_t state_dim, num_items, reserved[2];
} recnn_beta_dims;
/* out[4]: offsets of the weight and the bias, the weight's row pitch, total float count (cell 3: the Linear's layout) */
RECNN_API int recnn_beta_layout(const recnn_beta_dims* d, int64_t* out);
/* bytes of workspace of recnn_beta_step; chunk_items: num_items, or a positive multiple of 128 below it (0 when not
 * accepted).  Holds one [n_rows, chunk_items] chunk and does not grow with num_items below it. */
RECNN_API int64_t recnn_beta_workspace_bytes(const recnn_beta_dims* d, int64_t n_rows, int32_t chunk_items);

typedef struct recnn_beta_args {
  recnn_beta_dims dims;
  int64_t n_rows;
  int32_t chunk_items;
  int32_t reserved;
  recnn_net net;              /* params, grads (required), opt_m / opt_v / opt_t for the built-in optimizer */
  recnn_optim optim;          /* RECNN_OPT_EXTERNAL: stop after the gradient (left in net.grads) */
  const float* state;         /* [n_rows, state_ld] */
  int64_t state_ld;           /* >= state_dim */
  const int64_t* action;      /* [n_rows] target item ids (the notebook's action.argmax(1)) */
  float* probs_out;           /* [n_rows, num_items]: p with the weights from before the step */
  float* loss;                /* device fp32: mean cross-entropy of the call */
  int32_t* error;             /* device int32: 1 when an id was outside [0, num_items) -- then no row of that id added
                               * loss or gradient and the built-in optimizer step was skipped (t included) */
  void* workspace;
  int64_t workspace_bytes;
} recnn_beta_args;
RECNN_API int64_t recnn_sizeof_beta_args(void);
RECNN_API int64_t recnn_offsetof_beta_args(int field);
/* One Beta.forward(state, action) of the notebook's cell 3 (forward, loss, backward, optimizer step) on `stream`, no
 * allocation, no synchronisation.  The items are visited in chunks of chunk_items, twice: logits into probs_out with a
 * running max / sum, then dZ of each chunk from probs_out and that chunk's rows of dW / db.  Deterministic. */
RECNN_API int recnn_beta_step(const recnn_beta_args* args, void* stream);

/* ---- REINFORCE with Top-K correction: beta sharded over the item vocabulary, with the policy ------
 * Rank `rank` of `world` holds rows [lo, hi) of net.0.weight / net.0.bias, lo = v->item_offset and hi = lo +
 * args->dims.num_items (recnn_vocab_shard above, the policy's plan): args carries the LOCAL dims, so the arena is laid
 * out as a Beta(S, hi - lo) and args->probs_out is the rank's column block [n_rows, hi - lo].  Target ids stay global.
 * One call of recnn_beta_step becomes three phases on one stream with two exchanges (recnn_comm_allgather) between them:
 *   begin -> record (recnn_vocab_record_floats(n_rows): header {lo, hi, num_items, n_rows}, the local max and sum of
 *            exp of the block's logits, the target's logit from the rank that holds it, 0 elsewhere) -> all-gather
 *   rows  -> merges the gathered records in rank order, turns the block into its column block of p over the whole
 *            vocabulary, and writes a second record of the same size: the same header, then the block's per-row sums
 *            of expm1(p) and of p expm1(p) and a zero plane -> all-gather
 *   end   -> T = num_items + the rank-order sum of the first planes, U likewise, p_a, the loss, dW / db of the local rows
 *            (overwriting net.grads) and the built-in optimizer over the local arena (RECNN_OPT_EXTERNAL: stop after
 *            the gradient).
 * No all-reduce: the loss, T, U and p_a are the same bits on every rank.  The phases share args->workspace
 * (recnn_beta_workspace_bytes of the local dims: it does not grow with the vocabulary once chunk_items < hi - lo), which
 * must be left untouched between them; no allocation, no synchronisation.  At world 1 the three phases compute exactly
 * what recnn_beta_step does.  *error bits (written by end): 1 as for the step (an id outside [0, v->num_items), seen on
 * every rank); 2: a gathered record's header does not tile the vocabulary in rank order with this rank's block, or
 * the ranks disagree on n_rows.  With either bit set the built-in optimizer step is skipped (t included). */
RECNN_API int recnn_beta_shard_begin(const recnn_beta_args* args, const recnn_vocab_shard* v, float* record,
                                     void* stream);
RECNN_API int recnn_beta_shard_rows(const recnn_beta_args* args, const recnn_vocab_shard* v, const float* gathered,
                                    float* record, void* stream);
RECNN_API int recnn_beta_shard_end(const recnn_beta_args* args, const recnn_vocab_shard* v, const float* gathered,
                                   void* stream);

/* ---- data parallel: all-reduce over NVLink peer memory ------------------------------------------
 * BASELINE north_star: "partition the embedding gather + update across the 8 GPUs of one box with
 * an allreduce of the Actor/Critic gradients over NVLink".  The reference itself is single-process
 * (recnn/nn/update/ddpg.py:82-100 is where the gradients are complete and consumed), so these entry
 * points have no reference counterpart; they are what a torch.distributed launcher binds:
 *   every rank:  recnn_comm_create -> recnn_comm_local_handle -> (all-gather the handles with any
 *   host transport) -> recnn_comm_connect -> put the communicator in recnn_step_args.comm.
 * One process per GPU, at most 8 ranks on one node; the staging buffers are cudaMalloc memory shared
 * with cudaIpc and read by the peers' kernels directly (no NCCL call on the step's path). */
RECNN_API int recnn_comm_create(int32_t rank, int32_t world, int64_t capacity_floats, recnn_comm** out);
RECNN_API int32_t recnn_comm_handle_bytes(void);
RECNN_API int recnn_comm_local_handle(const recnn_comm* comm, void* out_handle);
/* all_handles: `world` handles of recnn_comm_handle_bytes() each, in rank order */
RECNN_API int recnn_comm_connect(recnn_comm* comm, const void* all_handles);
/* buf[i] <- sum over ranks of buf[i], in place, identical bits on every rank (n <= capacity_floats);
 * every rank must issue the same sequence of collectives on ONE stream. */
RECNN_API int recnn_comm_allreduce(const recnn_comm* comm, float* buf, int64_t n, void* stream);
/* gathered[q * n + i] <- rank q's local[i], rank-major, the same on every rank; words move as bit patterns (integer
 * payloads survive).  n * world <= capacity_floats, else refused before any launch.  Shares the epoch sequence of
 * recnn_comm_allreduce: the two may interleave on one communicator, in the same order on every rank. */
RECNN_API int recnn_comm_allgather(const recnn_comm* comm, const float* local, int64_t n, float* gathered, void* stream);
RECNN_API int recnn_comm_destroy(recnn_comm* comm);

#ifdef __cplusplus
}
#endif
#endif /* RECNN_B200_H */
