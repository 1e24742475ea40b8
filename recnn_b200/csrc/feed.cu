// Device-resident FrameEnv feed: user histories live in HBM as a CSR
//   hist_items int64[total], hist_ratings fp32[total], hist_offsets int64[n_users + 1]
// and a minibatch of sliding windows is cut out of it on the device.
//
// Restates recnn/data/utils.py:7-10 (rolling_window) + :161-181 (prepare_batch_static_size up to
// embed_batch) and the ``done`` rule of :70-71.  In the reference this runs in a DataLoader worker
// process (numpy strided views, np.concatenate, torch.tensor copy, pickling back to the parent) and
// the result crosses PCIe; here only the list of users (or window ids) of the minibatch is input.
// Pure integer/byte copies: bit-exact.
//
// One thread per output ELEMENT (row n, slot j): writes are perfectly coalesced (items: 8 B/thread,
// ratings: 4 B/thread over a dense [N, F+1] array), reads of consecutive rows of one user overlap in
// F of F+1 slots and hit L1/L2.  The owning user of a row is found by binary search over a prefix
// array (row_offsets[n_batch+1] in "users" form, win_offsets[n_users+1] in "ids" form); the F+1
// threads of a row search the same cache lines, so the search is a handful of broadcast L1 hits.
//
// Algorithmic bytes per row (F = 10): read 11*8 + 11*4 = 132 B, write 132 + 4 (done) = 136 B  => 268 B/row
// (1.6% of the 16,604 B/row of the embedding gather that consumes it).
#include "common.cuh"

namespace recnn {

// largest i in [0, n) with prefix[i] <= x   (prefix[0] <= x < prefix[n] guaranteed by the caller)
__device__ __forceinline__ long long upper_owner(const long long* __restrict__ prefix, long long n, long long x) {
  long long lo = 0, hi = n;          // invariant: prefix[lo] <= x < prefix[hi]
  while (hi - lo > 1) {
    const long long mid = (lo + hi) >> 1;
    if (__ldg(prefix + mid) <= x) lo = mid; else hi = mid;
  }
  return lo;
}

// IDS = false: rows are all windows of users batch_users[0..n_sel), in that order (the reference's minibatch).
// IDS = true : row n is global window sel[n] (windows numbered user by user in storage order).
template <bool IDS>
__global__ void __launch_bounds__(256)
window_gather_kernel(const long long* __restrict__ hist_items, const float* __restrict__ hist_ratings,
                     const long long* __restrict__ hist_offsets, long long n_users,
                     const long long* __restrict__ sel, const long long* __restrict__ prefix, long long n_sel,
                     int frame, long long n_rows,
                     long long* __restrict__ items, float* __restrict__ ratings, float* __restrict__ done,
                     long long* __restrict__ meta /* sizes[n_sel] (users form) | users[n_rows] (ids form) */,
                     int* __restrict__ err) {
  const int f1 = frame + 1;
  const long long total = n_rows * f1;
  const long long stride = (long long)gridDim.x * blockDim.x;
  for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += stride) {
    const long long n = e / f1;
    const int j = (int)(e - n * f1);
    long long user, local, want_win = -1;
    bool ok = true;
    if (IDS) {
      const long long w = __ldg(sel + n);
      ok = (w >= 0 && w < __ldg(prefix + n_users));
      user = ok ? upper_owner(prefix, n_users, w) : 0;
      local = ok ? w - __ldg(prefix + user) : 0;
    } else {
      const long long b = upper_owner(prefix, n_sel, n);
      const long long r0 = __ldg(prefix + b);
      user = __ldg(sel + b);
      local = n - r0;
      want_win = __ldg(prefix + b + 1) - r0;                    // the caller's plan for this user
      ok = (user >= 0 && user < n_users);
      if (!ok) user = 0;
    }
    const long long beg = __ldg(hist_offsets + user), end = __ldg(hist_offsets + user + 1);
    const long long n_win = end - beg - frame;                 // windows of this user (rolling_window shape[0])
    if (!IDS && n_win != want_win) ok = false;                 // row_offsets disagree with the resident histories
    if (ok) ok = (local >= 0 && local < n_win);
    if (!ok) {
      if (err) atomicOr(err, 1);
      if (items) items[e] = 0;
      if (ratings) ratings[e] = 0.f;
      if (j == 0 && done) done[n] = 0.f;
      if (IDS && j == 0 && meta) meta[n] = -1;
      continue;
    }
    const long long src = beg + local + j;
    if (items) items[e] = __ldg(hist_items + src);
    if (ratings) ratings[e] = __ldg(hist_ratings + src);
    if (j == 0) {
      if (done) done[n] = (local == n_win - 1) ? 1.0f : 0.0f;   // last window of its user (utils.py:70-71)
      if (IDS && meta) meta[n] = user;
    }
  }
  if (!IDS && meta) {                                           // sizes[b] = history length (utils.py:171,179)
    for (long long b = (long long)blockIdx.x * blockDim.x + threadIdx.x; b < n_sel; b += stride) {
      const long long u = __ldg(sel + b);
      meta[b] = (u >= 0 && u < n_users) ? __ldg(hist_offsets + u + 1) - __ldg(hist_offsets + u) : 0;
    }
  }
}

static int launch_window_gather(bool ids, const int64_t* hist_items, const float* hist_ratings,
                                const int64_t* hist_offsets, int64_t n_users, const int64_t* sel,
                                const int64_t* prefix, int64_t n_sel, int frame, int64_t n_rows, int64_t* items,
                                float* ratings, float* done, int64_t* meta, int* err, cudaStream_t st) {
  RECNN_REQUIRE(hist_items && hist_ratings && hist_offsets, "history arrays must be non-null");
  RECNN_REQUIRE(sel && prefix, "selection / prefix arrays must be non-null");
  RECNN_REQUIRE(n_users > 0 && frame > 0 && n_rows >= 0 && n_sel >= 0, "sizes must be positive");
  if (n_rows == 0 && (ids || n_sel == 0)) return RECNN_OK;
  const int64_t work = n_rows * (frame + 1) > n_sel ? n_rows * (frame + 1) : n_sel;
  const int64_t blocks = ceil_div(work, 256);
  const int grid = (int)(blocks < (int64_t)kNumSMs * 8 ? blocks : (int64_t)kNumSMs * 8);
  if (ids)
    window_gather_kernel<true><<<grid, 256, 0, st>>>((const long long*)hist_items, hist_ratings,
                                                     (const long long*)hist_offsets, n_users, (const long long*)sel,
                                                     (const long long*)prefix, n_sel, frame, n_rows,
                                                     (long long*)items, ratings, done, (long long*)meta, err);
  else
    window_gather_kernel<false><<<grid, 256, 0, st>>>((const long long*)hist_items, hist_ratings,
                                                      (const long long*)hist_offsets, n_users, (const long long*)sel,
                                                      (const long long*)prefix, n_sel, frame, n_rows,
                                                      (long long*)items, ratings, done, (long long*)meta, err);
  RECNN_CHECK_LAUNCH("window_gather_kernel");
  return RECNN_OK;
}

}  // namespace recnn

extern "C" int recnn_window_gather_users(const int64_t* hist_items, const float* hist_ratings,
                                         const int64_t* hist_offsets, int64_t n_users, const int64_t* batch_users,
                                         const int64_t* row_offsets, int64_t n_batch, int frame, int64_t n_rows,
                                         int64_t* items, float* ratings, float* done, int64_t* sizes,
                                         int* err_flag, void* stream) {
  RECNN_REQUIRE(n_batch > 0 || n_rows == 0, "a non-empty minibatch needs at least one user");
  if (n_batch == 0) return RECNN_OK;            // nothing to cut
  return recnn::launch_window_gather(false, hist_items, hist_ratings, hist_offsets, n_users, batch_users,
                                     row_offsets, n_batch, frame, n_rows, items, ratings, done, sizes, err_flag,
                                     static_cast<cudaStream_t>(stream));
}

extern "C" int recnn_window_gather_ids(const int64_t* hist_items, const float* hist_ratings,
                                       const int64_t* hist_offsets, const int64_t* win_offsets, int64_t n_users,
                                       const int64_t* window_ids, int frame, int64_t n_rows, int64_t* items,
                                       float* ratings, float* done, int64_t* users, int* err_flag, void* stream) {
  return recnn::launch_window_gather(true, hist_items, hist_ratings, hist_offsets, n_users, window_ids, win_offsets,
                                     n_rows, frame, n_rows, items, ratings, done, users, err_flag,
                                     static_cast<cudaStream_t>(stream));
}

// ---- Serving state: the state after each user's whole history ------------------------------------------------------
// Row u of out [n, F*D + F] is the next_state of user users[u]'s last window, in batch_tensor_embeddings' column order
// (F embedding rows, then F ratings) -- the history's last F items and ratings.  A user with exactly F interactions has
// no window but has this state.  One warp per (row, slot): pure copies, bit-exact.  *err |= 1 for a user position
// outside [0, n_users), 2 for a history shorter than F, 4 for an item outside the table (the row is then zero-filled
// where it could not be read).
namespace recnn {
__global__ void __launch_bounds__(256)
user_state_kernel(const float* __restrict__ table, long long n_items, int dim, const long long* __restrict__ hist_items,
                  const float* __restrict__ hist_ratings, const long long* __restrict__ hist_offsets,
                  long long n_users, const long long* __restrict__ users, long long n, int frame,
                  float* __restrict__ out, int* __restrict__ err) {
  const long long warp = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  const long long units = n * (frame + 1);               // F embedding rows and one ratings tail per row
  if (warp >= units) return;
  const long long r = warp / (frame + 1);
  const int j = (int)(warp - r * (frame + 1));
  const long long ld = (long long)frame * dim + frame;
  float* row = out + r * ld;
  const long long u = users[r];
  int bad = 0;
  long long src = 0;
  if (u < 0 || u >= n_users) bad = 1;
  else {
    const long long end = hist_offsets[u + 1];
    if (end - hist_offsets[u] < frame) bad = 2;
    src = end - frame;
  }
  if (j == frame) {                                      // the ratings tail
    for (int t = lane; t < frame; t += 32) row[(long long)frame * dim + t] = bad ? 0.f : hist_ratings[src + t];
    if (bad && lane == 0) atomicOr(err, bad);
    return;
  }
  long long id = bad ? -1 : hist_items[src + j];
  if (!bad && (id < 0 || id >= n_items)) {
    if (lane == 0) atomicOr(err, 4);
    id = -1;
  }
  float* dst = row + (long long)j * dim;
  for (int c = lane; c < dim; c += 32) dst[c] = id < 0 ? 0.f : __ldg(table + id * dim + c);
}
}  // namespace recnn

extern "C" int recnn_user_states(const float* table, int64_t n_items, int32_t dim, const int64_t* hist_items,
                                 const float* hist_ratings, const int64_t* hist_offsets, int64_t n_users,
                                 const int64_t* users, int64_t n, int32_t frame, float* out, int32_t* err_flag,
                                 void* stream) {
  RECNN_REQUIRE(table && hist_items && hist_ratings && hist_offsets && out && err_flag && (users || n == 0),
                "null pointer");
  RECNN_REQUIRE(n_items > 0 && dim > 0 && n_users > 0 && n >= 0 && frame > 0, "sizes");
  if (n == 0) return RECNN_OK;
  const int64_t blocks = recnn::ceil_div(n * (frame + 1), 8);
  recnn::user_state_kernel<<<(unsigned)blocks, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      table, n_items, dim, (const long long*)hist_items, hist_ratings, (const long long*)hist_offsets, n_users,
      (const long long*)users, n, frame, out, err_flag);
  RECNN_CHECK_LAUNCH("user_state_kernel");
  return RECNN_OK;
}
