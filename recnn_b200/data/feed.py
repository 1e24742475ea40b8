"""Device-resident FrameEnv feed (SURVEY.md 8f rank 1).

The reference produces every minibatch on the host: ``DataLoader(UserDataset, shuffle=True,
collate_fn=prepare_batch_static_size)`` (recnn/data/env.py:225-248) runs ``rolling_window`` +
``np.concatenate`` + ``torch.tensor`` in a worker process (recnn/data/utils.py:7-10, :161-181), pickles
the batch back to the parent and copies it to the GPU.  Here the user histories are uploaded ONCE as a
CSR (``HistoryCSR`` -> ``DeviceFrameFeed``) and a minibatch is cut out of it by one kernel
(``recnn_window_gather_users`` / ``recnn_window_gather_ids``, csrc/feed.cu); its output is exactly what
the collate hands to ``embed_batch`` -- ``items int64[N, F+1]``, ``ratings fp32[N, F+1]``, ``sizes``,
``users`` -- plus ``done``, i.e. the *frame form* that ``ddpg_update`` / ``td3_update`` of this package
gather from inside the step.  Per minibatch nothing but the user list crosses PCIe, and with ``epoch()``
not even that (permutation and row plan are uploaded once per epoch).

Two samplers:
  * ``batch(user_positions)`` / ``epoch(batch_size)``: the reference's minibatch -- ALL windows of
    ``batch_size`` shuffled users (variable row count N = sum(len_u - F));
  * ``sample(n_rows)``: a constant number of uniformly drawn windows per step (replay-buffer style;
    constant shapes keep the update step a single CUDA graph).  Row n equals row ``window_ids[n]`` of the
    reference collate over all users.

``HistoryCSR`` is plain numpy (host) so the planning logic is testable without a GPU; everything that
touches the device lives in ``DeviceFrameFeed``, which raises without CUDA (no CPU fallback).
"""
from __future__ import annotations

import numpy as np
import torch

from .. import _lib


class HistoryCSR:
    """Host-side CSR of a ``UserDataset``: users in dataset order, each with its time-ordered item rows
    and ratings (recnn/data/env.py:23-64).  Ratings are stored as fp32 -- the collate's ``.float()``
    (recnn/data/utils.py:178) applied once instead of per batch (same IEEE rounding, element-wise)."""

    def __init__(self, user_ids, items_per_user, ratings_per_user, frame_size):
        if len(user_ids) == 0:
            raise ValueError("HistoryCSR needs at least one user")
        self.frame_size = int(frame_size)
        self.user_ids = np.asarray(user_ids, dtype=np.int64)
        lengths = np.asarray([len(x) for x in items_per_user], dtype=np.int64)
        if any(len(r) != n for r, n in zip(ratings_per_user, lengths)):
            raise ValueError("items and ratings of a user must have the same length")
        self.lengths = lengths
        self.offsets = np.zeros(len(lengths) + 1, dtype=np.int64)
        np.cumsum(lengths, out=self.offsets[1:])
        self.items = np.concatenate([np.asarray(x, dtype=np.int64) for x in items_per_user])
        self.ratings = np.concatenate([np.asarray(r).astype(np.float32) for r in ratings_per_user])
        self.win_counts = np.maximum(lengths - self.frame_size, 0)          # rolling_window(...).shape[0]
        self.win_offsets = np.zeros(len(lengths) + 1, dtype=np.int64)
        np.cumsum(self.win_counts, out=self.win_offsets[1:])

    @classmethod
    def from_dataset(cls, dataset, frame_size):
        """From a ``UserDataset`` (``users`` list + ``user_dict``), in ``dataset.users`` order."""
        recs = [dataset.user_dict[u] for u in dataset.users]
        return cls(list(dataset.users), [r["items"] for r in recs], [r["ratings"] for r in recs], frame_size)

    @property
    def n_users(self):
        return int(self.lengths.shape[0])

    @property
    def n_windows(self):
        return int(self.win_offsets[-1])

    def check_positions(self, pos):
        pos = np.asarray(pos, dtype=np.int64).reshape(-1)
        if pos.size and (pos.min() < 0 or pos.max() >= self.n_users):
            raise IndexError("user position out of range [0, %d)" % self.n_users)
        short = self.lengths[pos] < self.frame_size       # rolling_window raises on a negative shape
        if short.any():
            raise ValueError("user(s) with fewer than frame_size=%d interactions cannot be windowed"
                             % self.frame_size)
        return pos

    def holdout_windows(self, pos):
        """int64 [U]: the id of each user's last window (the leave-last-out row: its action is the user's last item),
        in the collate's window order over all users.  A user without a window (fewer than F + 1 items) raises
        ValueError."""
        pos = self.check_positions(pos)
        if (self.win_counts[pos] == 0).any():
            raise ValueError("user(s) with fewer than frame_size + 1 = %d interactions have no held-out item"
                             % (self.frame_size + 1))
        return self.win_offsets[pos + 1] - 1

    def plan_users(self, pos):
        """row_offsets int64[B+1] (exclusive prefix sum of len - F over the batch's users) and N."""
        pos = self.check_positions(pos)
        row_offsets = np.zeros(pos.size + 1, dtype=np.int64)
        np.cumsum(self.lengths[pos] - self.frame_size, out=row_offsets[1:])
        return row_offsets, int(row_offsets[-1])

    def plan_epoch(self, perm, batch_size, drop_last=False):
        """Cut a user permutation into minibatches as ``DataLoader(batch_size=...)`` does.
        Returns (starts, counts, row_offsets_flat, row_starts, n_rows): batch b covers
        ``perm[starts[b] : starts[b]+counts[b]]`` and its row plan is
        ``row_offsets_flat[row_starts[b] : row_starts[b]+counts[b]+1]``."""
        perm = self.check_positions(perm)
        n = perm.size
        starts = np.arange(0, n, batch_size, dtype=np.int64)
        counts = np.minimum(batch_size, n - starts)
        if drop_last and counts.size and counts[-1] < batch_size:
            starts, counts = starts[:-1], counts[:-1]
        wins = self.lengths[perm] - self.frame_size
        flat = np.zeros(int(counts.sum() + counts.size), dtype=np.int64)
        row_starts = np.zeros(counts.size, dtype=np.int64)
        n_rows = np.zeros(counts.size, dtype=np.int64)
        at = 0
        for b, (s, c) in enumerate(zip(starts, counts)):
            row_starts[b] = at
            np.cumsum(wins[s:s + c], out=flat[at + 1:at + 1 + c])
            n_rows[b] = flat[at + c]
            at += c + 1
        return starts, counts, flat, row_starts, n_rows


class DeviceFrameFeed:
    """User histories + embedding table resident in HBM; minibatches are produced by one kernel."""

    def __init__(self, csr: HistoryCSR, table, device=None):
        if device is None:
            device = table.device if torch.is_tensor(table) and table.device.type == "cuda" else torch.device("cuda")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.RecnnError("DeviceFrameFeed lives on a CUDA device (got %s); there is no CPU feed here -- "
                                  "use FrameEnv's DataLoader for host-side batches" % self.device)
        if not torch.cuda.is_available():
            raise _lib.RecnnError("DeviceFrameFeed needs a CUDA device and none is available")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.csr = csr
        self.frame_size = csr.frame_size
        table = torch.as_tensor(table)
        if table.dtype != torch.float32:
            raise ValueError("embedding table must be fp32")
        self.table = table.to(self.device).contiguous()
        if csr.items.size and (csr.items.min() < 0 or csr.items.max() >= self.table.shape[0]):
            raise IndexError("a history holds an item row outside the embedding table")
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)
        self.hist_items = up(csr.items)
        self.hist_ratings = up(csr.ratings)
        self.hist_offsets = up(csr.offsets)
        self.win_offsets = up(csr.win_offsets)
        self._err = torch.zeros(1, dtype=torch.int32, device=self.device)
        self._seen = None
        self._popularity = None
        self.kernels = 0

    # ------------------------------------------------------------------ helpers
    def _outputs(self, n_rows):
        f1 = self.frame_size + 1
        return (torch.empty(n_rows, f1, dtype=torch.int64, device=self.device),
                torch.empty(n_rows, f1, dtype=torch.float32, device=self.device),
                torch.empty(n_rows, dtype=torch.float32, device=self.device))

    def _raise_on_error(self):
        if int(self._err.item()) != 0:
            self._err.zero_()
            raise IndexError("window gather: user / window index outside the resident histories")

    def _gather_users(self, users_d, row_off_d, n_batch, n_rows):
        items, ratings, done = self._outputs(n_rows)
        sizes = torch.empty(n_batch, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            L = _lib.lib()
            before = L.recnn_b200_launch_count()
            _lib.check(L.recnn_window_gather_users(
                self.hist_items.data_ptr(), self.hist_ratings.data_ptr(), self.hist_offsets.data_ptr(),
                self.csr.n_users, users_d.data_ptr(), row_off_d.data_ptr(), n_batch, self.frame_size, n_rows,
                items.data_ptr(), ratings.data_ptr(), done.data_ptr(), sizes.data_ptr(), self._err.data_ptr(),
                _lib.stream_ptr(self.device)))
            self.kernels += L.recnn_b200_launch_count() - before
        return items, ratings, done, sizes

    def _frame_batch(self, items, ratings, done, sizes, user_pos_host):
        ids = torch.from_numpy(self.csr.user_ids[user_pos_host])
        sizes_h = torch.from_numpy(self.csr.lengths[user_pos_host])
        return {"items": items, "ratings": ratings, "done": done, "sizes": sizes, "users": ids,
                "table": self.table, "meta": {"users": ids, "sizes": sizes_h}}

    # ------------------------------------------------------------------ the reference's minibatch
    def batch(self, user_positions, check=False):
        """All windows of the given users (positions in the CSR = indices into ``dataset.users``), in
        that order: what ``prepare_batch_static_size`` hands to ``embed_batch`` for the same users."""
        row_offsets, n_rows = self.csr.plan_users(user_positions)
        pos = np.asarray(user_positions, dtype=np.int64).reshape(-1)
        if pos.size == 0:
            raise ValueError("empty minibatch: need at least one user")    # np.concatenate([]) raises in the reference too
        plan = torch.from_numpy(np.concatenate([pos, row_offsets])).to(self.device)      # one small H2D
        items, ratings, done, sizes = self._gather_users(plan[:pos.size], plan[pos.size:], pos.size, n_rows)
        if check:
            self._raise_on_error()
        return self._frame_batch(items, ratings, done, sizes, pos)

    def epoch(self, batch_size=25, generator=None, drop_last=False, shuffle=True):
        """One pass over all users in minibatches of ``batch_size`` users, like the reference's
        ``DataLoader(..., shuffle=True)`` (recnn/data/env.py:225-231): a ``torch.randperm`` of the users
        drawn from ``generator`` (the sampler RandomSampler uses).  The permutation and the row plan of
        the whole epoch are uploaded once; each minibatch is then a single kernel launch."""
        n = self.csr.n_users
        perm = (torch.randperm(n, generator=generator) if shuffle else torch.arange(n)).numpy().astype(np.int64)
        starts, counts, flat, row_starts, n_rows = self.csr.plan_epoch(perm, batch_size, drop_last)
        plan = torch.from_numpy(np.concatenate([perm, flat])).to(self.device)
        perm_d, flat_d = plan[:n], plan[n:]
        for s, c, rs, nr in zip(starts.tolist(), counts.tolist(), row_starts.tolist(), n_rows.tolist()):
            items, ratings, done, sizes = self._gather_users(perm_d[s:s + c], flat_d[rs:rs + c + 1], c, nr)
            yield self._frame_batch(items, ratings, done, sizes, perm[s:s + c])

    # ------------------------------------------------------------------ constant-size minibatch
    def windows(self, window_ids, check=False):
        """Rows ``window_ids`` (int64 tensor, device or host) of the collate over ALL users."""
        w = torch.as_tensor(window_ids, dtype=torch.int64).to(self.device).contiguous().reshape(-1)
        n_rows = int(w.numel())
        items, ratings, done = self._outputs(n_rows)
        users = torch.empty(n_rows, dtype=torch.int64, device=self.device)
        with torch.cuda.device(self.device):
            L = _lib.lib()
            before = L.recnn_b200_launch_count()
            _lib.check(L.recnn_window_gather_ids(
                self.hist_items.data_ptr(), self.hist_ratings.data_ptr(), self.hist_offsets.data_ptr(),
                self.win_offsets.data_ptr(), self.csr.n_users, w.data_ptr(), self.frame_size, n_rows,
                items.data_ptr(), ratings.data_ptr(), done.data_ptr(), users.data_ptr(), self._err.data_ptr(),
                _lib.stream_ptr(self.device)))
            self.kernels += L.recnn_b200_launch_count() - before
        if check:
            self._raise_on_error()
        return {"items": items, "ratings": ratings, "done": done, "table": self.table, "window_ids": w,
                "user_positions": users, "meta": {"user_positions": users}}

    def sample(self, n_rows, generator=None):
        """``n_rows`` windows drawn uniformly (with replacement) over all windows of all users; the draw
        happens on the device (``generator``: a CUDA ``torch.Generator`` for reproducibility)."""
        if self.csr.n_windows <= 0:
            raise ValueError("no user has more than frame_size interactions")
        w = torch.randint(0, self.csr.n_windows, (int(n_rows),), device=self.device, dtype=torch.int64,
                          generator=generator)
        return self.windows(w)

    # ------------------------------------------------------------------ reference-shaped batch
    def embed(self, frame_batch):
        """state / action / reward / next_state / done dict of the reference (batch_tensor_embeddings,
        recnn/data/utils.py:51-81) from a frame-form batch of this feed."""
        n = frame_batch["items"].shape[0]
        dim = self.table.shape[1]
        s_dim = self.frame_size * dim + self.frame_size
        state = torch.empty(n, s_dim, device=self.device)
        next_state = torch.empty(n, s_dim, device=self.device)
        action = torch.empty(n, dim, device=self.device)
        reward = torch.empty(n, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().recnn_frame_gather(
                self.table.data_ptr(), self.table.shape[0], dim, frame_batch["items"].data_ptr(),
                frame_batch["ratings"].data_ptr(), n, self.frame_size, state.data_ptr(), next_state.data_ptr(),
                action.data_ptr(), reward.data_ptr(), None, _lib.stream_ptr(self.device)))
        return {"state": state, "action": action, "reward": reward, "next_state": next_state,
                "done": frame_batch["done"], "meta": frame_batch.get("meta", {})}

    # ------------------------------------------------------------------ serving
    def user_states(self, user_positions):
        """fp32 [U, F*D + F]: the state after each user's whole history (its last F items and ratings), the state a
        recommendation for that user is served from -- bit for bit the ``next_state`` of the user's last window, in
        ``batch_tensor_embeddings``' column order.  A user with exactly F interactions has no window but has this
        state; fewer than F raises ValueError.  One kernel (recnn_user_states)."""
        pos = self.csr.check_positions(user_positions)
        n = int(pos.size)
        dim = self.table.shape[1]
        out = torch.empty(n, self.frame_size * dim + self.frame_size, device=self.device)
        if n == 0:
            return out
        users = torch.from_numpy(pos).to(self.device)
        err = torch.zeros(1, dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().recnn_user_states(
                self.table.data_ptr(), self.table.shape[0], dim, self.hist_items.data_ptr(),
                self.hist_ratings.data_ptr(), self.hist_offsets.data_ptr(), self.csr.n_users, users.data_ptr(), n,
                self.frame_size, out.data_ptr(), err.data_ptr(), _lib.stream_ptr(self.device)))
        if int(err.item()) != 0:
            raise IndexError("user_states: a user position or history item outside the resident histories")
        return out

    def holdout(self, user_positions):
        """The leave-last-out evaluation rows of the given users: ``state`` fp32 [U, F*D + F], the state of each
        user's last window (bit for bit ``embed(windows(last))["state"]``); ``target`` int64 [U], that window's last
        item (the user's last rated item); ``exclude_rows`` int64 [U], the user positions, the rows of
        ``seen_items()``.  ``policy.rank(h["state"], h["target"], exclude=feed.seen_items(),
        exclude_rows=h["exclude_rows"])`` ranks each held-out item among the items the user has not rated before (the
        target itself is never excluded).  ``reward`` fp32 [U] is the held-out item's rating (bit for bit
        ``embed(windows(last))["reward"]``): with ``target`` as the logged action, the logged data of an off-policy
        estimate (``recnn_b200.utils.metrics.off_policy_estimates``).  A user with fewer than F + 1 items raises
        ValueError."""
        last = self.csr.holdout_windows(user_positions)
        pos = np.array(user_positions, dtype=np.int64).reshape(-1)
        batch = self.windows(torch.from_numpy(last))
        emb = self.embed(batch)
        return {"state": emb["state"], "target": batch["items"][:, self.frame_size].contiguous(),
                "reward": emb["reward"], "exclude_rows": torch.from_numpy(pos).to(self.device),
                "window_ids": batch["window_ids"]}

    def seen_items(self):
        """``ItemSets`` with one set per user position of the CSR: the distinct items of that user's history,
        ascending.  Built on the device once and cached.  ``policy.topk(feed.user_states(pos), k,
        exclude=feed.seen_items(), exclude_rows=pos)`` recommends only items the users have not rated."""
        if self._seen is None:
            from .item_sets import ItemSets
            self._seen = ItemSets(self.hist_items, self.hist_offsets, unique=True)
        return self._seen

    def item_popularity(self):
        """int64 [n_items] on the feed's device: the number of resident users whose history holds each item (the
        bincount of ``seen_items()``' ids).  Built once and cached.  With ``n_users = feed.csr.n_users`` it is the
        popularity that ``recnn_b200.utils.metrics.slate_metrics`` scores novelty against."""
        if self._popularity is None:
            self._popularity = torch.bincount(self.seen_items().ids, minlength=self.table.shape[0])
        return self._popularity
