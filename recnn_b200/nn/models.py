"""Actor / Critic / DiscreteActor with the reference's constructor, attributes and state_dict
layout (recnn/nn/models.py:41-73, :76-184, :187-213), evaluated by the sm_90a kernels.

``forward`` is the inference / evaluation entry (no autograd graph): training
goes through recnn_b200.nn.update.*, which runs forward+backward+optimizer as
one fused device step.  There is no CPU implementation behind ``forward`` --
calling it on CPU tensors raises.
"""
from __future__ import annotations

import types

import torch
import torch.nn as nn

from .. import _lib
from .arena import param_arena, discrete_dims


def _dims(state_dim, action_dim, hidden):
    return _lib.Dims(int(state_dim), int(action_dim), int(hidden), 0)


def _device_check(module, *tensors):
    dev = module.linear1.weight.device
    if dev.type != "cuda":
        raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
    out = []
    for t in tensors:
        out.append(t.detach().to(device=dev, dtype=torch.float32).contiguous())
    return dev, out


def _check_row_ids(ids, n, name):
    """ValueError unless ``ids`` is an integer tensor [n] (one item id per row)."""
    if (not torch.is_tensor(ids) or ids.dim() != 1 or ids.shape[0] != n
            or ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool):
        raise ValueError("%s must be an integer tensor [N] with N = %d rows (got %s)"
                         % (name, n, "%s %s" % (tuple(ids.shape), ids.dtype) if torch.is_tensor(ids)
                            else type(ids).__name__))


def _log_prob_errors(bits, items):
    """Raise what the error bits of a log-prob call (unsharded, or recnn_vocab_log_prob_finish) report."""
    if bits & 2:
        raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
    if bits & 1:
        raise IndexError("an item id is out of range for the net's %d items" % items)


def _train_masks(module, n_rows, hidden, device):
    """Dropout(p=0.5) keep-masks for the two hidden layers (train mode only)."""
    if not module.training:
        return None, None
    keep = torch.rand(2, n_rows, hidden, device=device) >= 0.5
    keep = keep.to(torch.uint8)
    return keep[0], keep[1]


class Actor(nn.Module):
    """Vanilla actor: state -> action.  Same signature as recnn.nn.Actor."""

    def __init__(self, input_dim, action_dim, hidden_size, init_w=2e-1):
        super().__init__()
        self.drop_layer = nn.Dropout(p=0.5)       # kept for attribute parity; p is fixed at 0.5 in the kernels
        self.linear1 = nn.Linear(input_dim, hidden_size)
        self.linear2 = nn.Linear(hidden_size, hidden_size)
        self.linear3 = nn.Linear(hidden_size, action_dim)
        self.linear3.weight.data.uniform_(-init_w, init_w)
        self.linear3.bias.data.uniform_(-init_w, init_w)

    @property
    def dims(self):
        return _dims(self.linear1.in_features, self.linear3.out_features, self.linear1.out_features)

    def forward(self, state, tanh=False, masks=None):
        dev, (state,) = _device_check(self, state)
        n = state.shape[0]
        d = self.dims
        flat = param_arena(self)
        m1, m2 = masks if masks is not None else _train_masks(self, n, d.hidden, dev)
        out = torch.empty(n, d.action_dim, device=dev, dtype=torch.float32)
        scratch = torch.empty(_lib.lib().recnn_forward_scratch_floats(d, n, 0), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().recnn_actor_forward(
                d, flat.data_ptr(), state.data_ptr(), n, _lib.ptr(m1), _lib.ptr(m2), int(bool(tanh)),
                out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
        return out


class Critic(nn.Module):
    """Vanilla critic: (state, action) -> value [N,1].  Same signature as recnn.nn.Critic."""

    def __init__(self, input_dim, action_dim, hidden_size, init_w=3e-5):
        super().__init__()
        self.drop_layer = nn.Dropout(p=0.5)
        self.linear1 = nn.Linear(input_dim + action_dim, hidden_size)
        self.linear2 = nn.Linear(hidden_size, hidden_size)
        self.linear3 = nn.Linear(hidden_size, 1)
        self.linear3.weight.data.uniform_(-init_w, init_w)
        self.linear3.bias.data.uniform_(-init_w, init_w)
        self._action_dim = int(action_dim)

    @property
    def dims(self):
        a = self._action_dim
        return _dims(self.linear1.in_features - a, a, self.linear1.out_features)

    def forward(self, state, action, masks=None):
        dev, (state, action) = _device_check(self, state, action)
        n = state.shape[0]
        d = self.dims
        flat = param_arena(self)
        m1, m2 = masks if masks is not None else _train_masks(self, n, d.hidden, dev)
        out = torch.empty(n, 1, device=dev, dtype=torch.float32)
        scratch = torch.empty(_lib.lib().recnn_forward_scratch_floats(d, n, 1), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().recnn_critic_forward(
                d, flat.data_ptr(), state.data_ptr(), action.data_ptr(), n, _lib.ptr(m1), _lib.ptr(m2),
                out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
        return out

    # -- serving: items scored by Q (the Wolpertinger policy) --------------------------------------------------------
    def _serve_args(self, state, items, candidates, exclude, exclude_rows, chunk, target=None):
        """The argument handling of ``topk`` and ``rank``: every refusal before any device work, then the device
        forms.  A namespace of d, n, dev, state, items, cand / m (m = 0: every item), table (the C arguments of the
        exclusion: five values, offsets None for none), target, chunk."""
        from ..data.item_sets import ItemSets, row_map
        d = self.dims
        if not torch.is_tensor(state) or state.dim() != 2 or state.shape[1] != d.state_dim \
                or not state.dtype.is_floating_point:
            raise ValueError("state must be a floating-point tensor [N, %d]" % d.state_dim)
        n = state.shape[0]
        if not torch.is_tensor(items) or items.dim() != 2 or items.dtype != torch.float32 or items.shape[0] < 1:
            raise ValueError("items must be the fp32 embedding table [n_items, %d] (got %s)"
                             % (d.action_dim, "%s %s" % (tuple(items.shape), items.dtype) if torch.is_tensor(items)
                                else type(items).__name__))
        if items.shape[1] != d.action_dim:
            raise ValueError("items has %d columns but the critic's action_dim is %d" % (items.shape[1], d.action_dim))
        if candidates is not None:
            if (not torch.is_tensor(candidates) or candidates.dim() != 2 or candidates.shape[0] != n
                    or candidates.shape[1] < 1 or candidates.dtype.is_floating_point or candidates.dtype.is_complex
                    or candidates.dtype == torch.bool):
                raise ValueError("candidates must be an integer tensor [N, M] with N = %d rows and M >= 1 (got %s)"
                                 % (n, "%s %s" % (tuple(candidates.shape), candidates.dtype)
                                    if torch.is_tensor(candidates) else type(candidates).__name__))
        sets = rows = None
        if isinstance(exclude, ItemSets):
            sets, rows = row_map(exclude, exclude_rows, n)
        elif exclude is not None:
            raise ValueError("exclude must be a recnn_b200.data.ItemSets (got %s)" % type(exclude).__name__)
        elif exclude_rows is not None:
            raise ValueError("exclude_rows maps rows to the sets of an ItemSets exclude")
        if target is not None:
            _check_row_ids(target, n, "target")
        if chunk is None:
            chunk = 0
        if isinstance(chunk, bool) or not isinstance(chunk, int) or not 0 <= chunk < 2 ** 31:
            raise ValueError("chunk must be None (auto) or an int in [1, 2^31), got %r" % (chunk,))
        dev = self.linear1.weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
        if items.device != dev:
            raise ValueError("items must be on the critic's device %s (got %s)" % (dev, items.device))
        a = types.SimpleNamespace(d=d, n=n, dev=dev, chunk=chunk, n_items=int(items.shape[0]), cand=None, m=0,
                                  table=(None, 0, None, 0, None), target=None, sets=sets)
        if n == 0:
            return a
        _, (a.state,) = _device_check(self, state)
        a.items = items.contiguous()
        if candidates is not None:
            a.cand = candidates.detach().to(device=dev, dtype=torch.int64).contiguous()
            a.m = int(candidates.shape[1])
        if target is not None:
            a.target = target.detach().to(device=dev, dtype=torch.int64).contiguous()
        if sets is not None:
            a.sets = sets = sets.to(dev)
            rows = None if rows is None else rows.to(dev).contiguous()
            a.rows = rows                       # keeps the device copy alive: the table holds its pointer
            a.table = (sets.ids.data_ptr() if sets.ids.numel() else None, sets.ids.numel(), sets.offsets.data_ptr(),
                       len(sets), _lib.ptr(rows))
        return a

    @staticmethod
    def _serve_errors(flag, a):
        bits = int(flag.item())
        if bits & 1:
            raise IndexError("a candidate, target or excluded item id is out of range for the table's %d items"
                             % a.n_items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % len(a.sets))
        if bits & 8:
            raise ValueError("an item id is repeated within a row's candidates")

    def topk(self, state, k, items, candidates=None, exclude=None, exclude_rows=None, chunk=None):
        """``(values, ids)``: the k items of highest Q(state[r], items[j]) per row, best first (equal Q: the smaller
        id first) -- the Wolpertinger policy's choice when ``candidates`` holds the actor's nearest items.

        ``items``: the fp32 embedding table [n_items, action_dim] on the critic's device (e.g. ``ItemIndex.table``).
        ``candidates``: int [N, M] item ids per row, -1 padding (e.g. ``index.search(actor(state), 64).id()``, or
        several such lists concatenated); None scores every item of the table.  ``exclude`` / ``exclude_rows``: an
        ``ItemSets`` of ids never returned (e.g. ``DeviceFrameFeed.seen_items()``), as in ``ItemIndex.search``.
        values fp32 [N, k] are the Q values, ids int64 [N, k]; a row with fewer than k eligible items ends in id -1,
        value -FLT_MAX.  A NaN or -inf Q ranks after every finite one (ties by id, value -FLT_MAX), before any -1.  1 <= k <= 64.  ``chunk``: columns per chunk (None: auto); it does not change a bit.

        Scores are the eval-mode forward whatever ``self.training`` says; nothing of the critic is changed.  A repeated
        id within a row's candidates or a malformed table raises ValueError, an id out of range IndexError.  Nothing of
        size [N, n_items] is formed: layer 1 is split into a per-row and a per-item term, and each pair costs one
        H x H layer on the tensor cores."""
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= 64:
            raise ValueError("k must be an int in [1, 64], got %r" % (k,))
        a = self._serve_args(state, items, candidates, exclude, exclude_rows, chunk)
        values = torch.empty(a.n, k, device=a.dev, dtype=torch.float32)
        ids = torch.empty(a.n, k, device=a.dev, dtype=torch.int64)
        if a.n == 0:
            return values, ids
        L = _lib.lib()
        flat = param_arena(self)
        nbytes = L.recnn_critic_serve_workspace_bytes(a.d, a.n, a.m, a.n_items, k, a.chunk)
        ws = torch.empty(nbytes, device=a.dev, dtype=torch.uint8)
        flag = torch.zeros(1, dtype=torch.int32, device=a.dev)
        with torch.cuda.device(a.dev):
            _lib.check(L.recnn_critic_topk(a.d, flat.data_ptr(), a.state.data_ptr(), a.n, a.items.data_ptr(),
                                           a.n_items, _lib.ptr(a.cand), a.m, k, *a.table, a.chunk,
                                           values.data_ptr(), ids.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                           _lib.stream_ptr(a.dev)))
        self._serve_errors(flag, a)
        return values, ids

    def rank(self, state, target, items, candidates=None, exclude=None, exclude_rows=None, chunk=None):
        """int64 [N]: for offline evaluation, the number of eligible items that beat ``target[r]`` under Q (a higher
        Q, or an equal Q and a smaller id), i.e. the target's position in ``topk`` on the same inputs when below k, at
        any k.  Arguments as in ``topk``; a row's target is never excluded.  With ``candidates``, a target missing from
        its row's candidates gets the row's count of eligible candidates (it is absent from every list, so
        ``ranking_metrics`` at k <= M stays exact).  A target out of range raises IndexError."""
        a = self._serve_args(state, items, candidates, exclude, exclude_rows, chunk, target=target)
        rank = torch.empty(a.n, device=a.dev, dtype=torch.int64)
        if a.n == 0:
            return rank
        L = _lib.lib()
        flat = param_arena(self)
        nbytes = L.recnn_critic_serve_workspace_bytes(a.d, a.n, a.m, a.n_items, 0, a.chunk)
        ws = torch.empty(nbytes, device=a.dev, dtype=torch.uint8)
        flag = torch.zeros(1, dtype=torch.int32, device=a.dev)
        with torch.cuda.device(a.dev):
            _lib.check(L.recnn_critic_rank(a.d, flat.data_ptr(), a.state.data_ptr(), a.n, a.items.data_ptr(),
                                           a.n_items, _lib.ptr(a.cand), a.m, a.target.data_ptr(), *a.table, a.chunk,
                                           rank.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                           _lib.stream_ptr(a.dev)))
        self._serve_errors(flag, a)
        return rank


class DiscreteActor(nn.Module):
    """REINFORCE policy over a discrete item set: state -> probabilities [N, action_dim]
    (recnn/nn/models.py:76-184; same constructor, attributes and methods).

    Differences from the reference, all forced by running without an autograd graph:

    * ``saved_log_probs`` / ``correction`` / ``lambda_k`` hold the same VALUES (device tensors) but carry no graph; the
      policy update recomputes the forward over the rows saved here (``_saved``: state, drawn action, beta log-prob per
      env step) inside one fused backward (recnn_reinforce_policy_grad) -- valid because the policy's weights do not
      change between two policy updates.  ``gc()`` drops both.
    * Categorical draws are inverse-CDF draws on a counter-based Philox stream keyed by ``torch.initial_seed()`` (or on
      ``uniform_source(n_rows) -> tensor[n_rows]`` when set: replayable draws for tests), not torch's global generator.
    * After ``recnn_b200.dist.enable_vocab_parallel`` each rank holds a block of linear2's rows, and ``forward`` /
      ``select_action`` return the rank's column block of the probabilities; draws and log-probs stay global.
    * After ``recnn_b200.dist.enable_data_parallel`` each rank holds a full replica and its own rows: ``select_action``
      / ``pi_beta_sample`` draw row r of the rank at the Philox counter of its global row; ``forward`` and ``topk``
      stay local, with no exchange; ``sample_topk`` keys row r by its global row (one all-gather of row counts).
    """

    def __init__(self, input_dim, action_dim, hidden_size, init_w=0):
        super().__init__()
        self.linear1 = nn.Linear(input_dim, hidden_size)
        self.linear2 = nn.Linear(hidden_size, action_dim)
        self.saved_log_probs = []
        self.rewards = []
        self.correction = []
        self.lambda_k = []
        # {pi: pi, beta: beta} by default; {pi: beta, beta: beta} is the variant of awarebayes/RecNN issue 7
        self.action_source = {"pi": "pi", "beta": "beta"}
        self.select_action = self._select_action
        self.uniform_source = None
        self._saved = []
        self._draws = 0

    @property
    def dims(self):
        return discrete_dims(self)

    def forward(self, inputs):
        """probabilities [N, num_items]; on a vocabulary-parallel policy (recnn_b200.dist.enable_vocab_parallel) the
        rank's column block [N, hi - lo] of them."""
        return self._pi(inputs)[0]

    def _pi(self, inputs):
        """(probs, gathered records): the records of the rank-order all-gather when the policy is sharded, else None."""
        dev, (state,) = _device_check(self, inputs)
        n = state.shape[0]
        d = self.dims
        flat = param_arena(self)
        out = torch.empty(n, d.num_items, device=dev, dtype=torch.float32)
        if n == 0:
            return out, None
        L = _lib.lib()
        vp = self.__dict__.get("_recnn_vp")
        scratch = torch.empty(L.recnn_discrete_scratch_floats(d, n, 0), device=dev, dtype=torch.float32)
        with torch.cuda.device(dev):
            if vp is None:
                _lib.check(L.recnn_discrete_forward(d, flat.data_ptr(), state.data_ptr(), n, out.data_ptr(),
                                                    scratch.data_ptr(), _lib.stream_ptr(dev)))
                return out, None
            shard = vp.shard()
            rec = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
            _lib.check(L.recnn_discrete_shard_forward(d, shard, flat.data_ptr(), state.data_ptr(), n, out.data_ptr(),
                                                      rec.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
            gathered = vp.all_gather(rec)
            flag = torch.zeros(1, dtype=torch.int32, device=dev)
            _lib.check(L.recnn_discrete_shard_finish(d, shard, gathered.data_ptr(), n, out.data_ptr(), flag.data_ptr(),
                                                     _lib.stream_ptr(dev)))
        if int(flag.item()) != 0:
            raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
        return out, gathered

    def _slate_args(self, state, k, exclude, exclude_rows):
        """The argument handling of ``topk`` and ``sample_topk``: every refusal before any device work, then the
        outputs and the device forms of the state and the exclusion.  A namespace of vp, d, items, n, dev, state,
        values, ids, ex / n_ex (the dense form), sets / table (an ItemSets form, table: its C arguments)."""
        from ..data.item_sets import ItemSets, row_map
        vp = self.__dict__.get("_recnn_vp")
        d = self.dims
        items = d.num_items if vp is None else vp.num_items
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(64, items):
            raise ValueError("k must be an int in [1, min(64, num_items)] = [1, %d], got %r" % (min(64, items), k))
        if not torch.is_tensor(state) or state.dim() != 2 or state.shape[1] != d.state_dim:
            raise ValueError("state must be a [N, %d] tensor" % d.state_dim)
        n = state.shape[0]
        n_ex = 0
        sets = rows = None
        if isinstance(exclude, ItemSets):
            sets, rows = row_map(exclude, exclude_rows, n)
        elif exclude_rows is not None:
            raise ValueError("exclude_rows maps rows to the sets of an ItemSets exclude")
        elif exclude is not None:
            if (not torch.is_tensor(exclude) or exclude.dim() != 2 or exclude.shape[0] != n
                    or exclude.shape[1] > 256 or exclude.dtype.is_floating_point or exclude.dtype == torch.bool):
                raise ValueError("exclude must be an ItemSets or an integer tensor [N, E] with N = %d rows and E <= 256 "
                                 "(got %s)" % (n, tuple(exclude.shape) if torch.is_tensor(exclude)
                                               else type(exclude).__name__))
            n_ex = exclude.shape[1]
        dev = self.linear1.weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
        a = types.SimpleNamespace(vp=vp, d=d, items=items, n=n, dev=dev, n_ex=n_ex, ex=None, sets=None, table=None,
                                  values=torch.empty(n, k, device=dev, dtype=torch.float32),
                                  ids=torch.empty(n, k, device=dev, dtype=torch.int64))
        if n == 0:
            return a
        _, (a.state,) = _device_check(self, state)
        a.ex = None if n_ex == 0 else exclude.detach().to(device=dev, dtype=torch.int64).contiguous()
        if sets is not None:
            a.sets = sets = sets.to(dev)
            rows = None if rows is None else rows.to(dev).contiguous()
            a.table = (sets.ids.data_ptr() if sets.ids.numel() else None, sets.ids.numel(), sets.offsets.data_ptr(),
                       len(sets), _lib.ptr(rows))
        return a

    @staticmethod
    def _slate_errors(flag, a):
        """Raise what the error bits of a topk / sample_topk call (the call's word, the table check's) report."""
        f = flag.tolist()
        bits = f[0] | f[1]
        if bits & 2:
            raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
        if bits & 1:
            raise IndexError("an excluded item id is out of range for the policy's %d items" % a.items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % len(a.sets))

    def topk(self, state, k, exclude=None, exclude_rows=None):
        """``(values, indices)`` as ``torch.topk(self(state), k)`` without forming the [N, num_items] probabilities:
        the k items of highest logit per row (equal logits: the smaller id first), values fp32 [N, k] = pi(a|s),
        indices int64 [N, k] global item ids, on a vocabulary-parallel policy too (one all-gather of k candidates per
        row and rank).  ``exclude``: ids never returned, which stay in the softmax's normaliser (values are not
        renormalised) -- either an integer tensor [N, E] (E <= 256, e.g. the frame's items; negative ids are padding)
        or a ``recnn_b200.data.ItemSets`` table of any length (e.g. ``DeviceFrameFeed.seen_items()``: everything the
        user has rated), with ``exclude_rows`` int64 [N] naming each row's set (-1: none; default row r -> set r).
        An excluded id outside [0, num_items) raises IndexError, a malformed table ValueError.  A row with fewer than
        k eligible items ends in id -1, value 0.  1 <= k <= min(64, num_items).  Inference only: nothing saved for
        the policy update is touched."""
        from .update.reinforce import _chunk_items
        a = self._slate_args(state, k, exclude, exclude_rows)
        if a.n == 0:
            return a.values, a.ids
        vp, d, n, dev, ex, n_ex = a.vp, a.d, a.n, a.dev, a.ex, a.n_ex
        values, ids, table = a.values, a.ids, a.table
        L = _lib.lib()
        flat = param_arena(self)
        chunk = _chunk_items(n, d.num_items)
        nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        flag = torch.zeros(2, dtype=torch.int32, device=dev)       # the call's bits, the table check's (sharded)
        with torch.cuda.device(dev):
            if vp is None and table is None:
                _lib.check(L.recnn_discrete_topk(d, flat.data_ptr(), a.state.data_ptr(), n, k, _lib.ptr(ex), n_ex,
                                                 chunk, values.data_ptr(), ids.data_ptr(), flag.data_ptr(),
                                                 ws.data_ptr(), nbytes, _lib.stream_ptr(dev)))
            elif vp is None:
                _lib.check(L.recnn_discrete_topk_sets(d, flat.data_ptr(), a.state.data_ptr(), n, k, *table, chunk,
                                                      values.data_ptr(), ids.data_ptr(), flag.data_ptr(),
                                                      ws.data_ptr(), nbytes, _lib.stream_ptr(dev)))
            else:
                shard = vp.shard()
                rec = torch.empty(L.recnn_vocab_topk_record_floats(n, k), device=dev, dtype=torch.float32)
                if table is None:
                    _lib.check(L.recnn_discrete_shard_topk(d, shard, flat.data_ptr(), a.state.data_ptr(), n, k,
                                                           _lib.ptr(ex), n_ex, chunk, rec.data_ptr(), ws.data_ptr(),
                                                           nbytes, _lib.stream_ptr(dev)))
                else:
                    _lib.check(L.recnn_discrete_shard_topk_sets(d, shard, flat.data_ptr(), a.state.data_ptr(), n, k,
                                                                *table, chunk, rec.data_ptr(), flag[1:].data_ptr(),
                                                                ws.data_ptr(), nbytes, _lib.stream_ptr(dev)))
                del ws
                gathered = vp.all_gather(rec)
                _lib.check(L.recnn_discrete_shard_topk_finish(d, shard, gathered.data_ptr(), n, k, _lib.ptr(ex), n_ex,
                                                              values.data_ptr(), ids.data_ptr(), flag.data_ptr(),
                                                              _lib.stream_ptr(dev)))
        self._slate_errors(flag, a)
        return values, ids

    def sample_topk(self, state, k, exclude=None, exclude_rows=None, seed=None):
        """``(values, indices)`` of a slate of k items per row drawn from the policy without replacement: the
        distribution of ``torch.multinomial(self(state), k, replacement=False)`` with the excluded items'
        probabilities set to 0, position 0 the first draw, every row independent -- without forming the
        [N, num_items] probabilities.  The draw is the top-k of logit + Gumbel noise (Gumbel-top-k), so it runs
        ``topk``'s pass with another key; ``exclude`` / ``exclude_rows``, k, the errors and the -1 / 0 padding of
        short rows are ``topk``'s.  values fp32 [N, k] = pi(a|s) under the full softmax (excluded items stay in the
        normaliser), indices int64 [N, k] global item ids.

        ``seed``: None draws a 63-bit seed from torch's default CPU generator (so ``torch.manual_seed`` makes a call
        reproducible and successive calls differ); an int in [0, 2^64) keys the noise, which is then a pure function
        of (seed, global row, item id): the ids do not depend on the chunking, the GEMM back end (beyond the logits'
        rounding), the world size or the batching.  On a vocabulary-parallel policy the slate is over the whole
        vocabulary (one all-gather of k candidates per row and rank) and every rank returns the same bits; ranks
        passing different seeds raise RuntimeError on every rank.  On a data-parallel replica row r is keyed by its
        global row, so the ranks' rows are the single-GPU call's over the whole batch.  Inference only: nothing saved
        for the policy update is touched."""
        from .update.reinforce import _chunk_items
        if seed is not None and (isinstance(seed, bool) or not isinstance(seed, int) or not 0 <= seed < 2 ** 64):
            raise ValueError("seed must be None or an int in [0, 2^64), got %r" % (seed,))
        a = self._slate_args(state, k, exclude, exclude_rows)
        row0 = self._row_offset(a.n) or 0            # a collective on a data-parallel replica, before any return
        if seed is None:
            seed = int(torch.randint(0, 2 ** 63 - 1, (1,), dtype=torch.int64).item())
        if a.n == 0:
            return a.values, a.ids
        vp, d, n, dev, ex, n_ex = a.vp, a.d, a.n, a.dev, a.ex, a.n_ex
        values, ids, table = a.values, a.ids, a.table
        L = _lib.lib()
        flat = param_arena(self)
        chunk = _chunk_items(n, d.num_items)
        nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        flag = torch.zeros(2, dtype=torch.int32, device=dev)       # the call's bits, the table check's (sharded)
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            if vp is None and table is None:
                _lib.check(L.recnn_discrete_sample_topk(d, flat.data_ptr(), a.state.data_ptr(), n, k, _lib.ptr(ex),
                                                        n_ex, seed, row0, chunk, values.data_ptr(), ids.data_ptr(),
                                                        flag.data_ptr(), ws.data_ptr(), nbytes, st))
            elif vp is None:
                _lib.check(L.recnn_discrete_sample_topk_sets(d, flat.data_ptr(), a.state.data_ptr(), n, k, *table,
                                                             seed, row0, chunk, values.data_ptr(), ids.data_ptr(),
                                                             flag.data_ptr(), ws.data_ptr(), nbytes, st))
            else:
                shard = vp.shard()
                rec = torch.empty(L.recnn_vocab_sample_topk_record_floats(n, k), device=dev, dtype=torch.float32)
                if table is None:
                    _lib.check(L.recnn_discrete_shard_sample_topk(d, shard, flat.data_ptr(), a.state.data_ptr(), n, k,
                                                                  _lib.ptr(ex), n_ex, seed, row0, chunk,
                                                                  rec.data_ptr(), ws.data_ptr(), nbytes, st))
                else:
                    _lib.check(L.recnn_discrete_shard_sample_topk_sets(d, shard, flat.data_ptr(), a.state.data_ptr(),
                                                                       n, k, *table, seed, row0, chunk,
                                                                       rec.data_ptr(), flag[1:].data_ptr(),
                                                                       ws.data_ptr(), nbytes, st))
                del ws
                gathered = vp.all_gather(rec)
                _lib.check(L.recnn_discrete_shard_sample_topk_finish(d, shard, gathered.data_ptr(), n, k, _lib.ptr(ex),
                                                                     n_ex, seed, values.data_ptr(), ids.data_ptr(),
                                                                     flag.data_ptr(), st))
        if vp is not None and flag.tolist()[0] & 2:
            raise RuntimeError("the ranks disagree on the vocabulary shard plan, the number of rows or the seed: pass "
                               "every rank the same seed (or seed every rank's generator the same)")
        self._slate_errors(flag, a)
        return values, ids

    def rank(self, state, target, exclude=None, exclude_rows=None):
        """``(rank, log_prob)`` of each row's target item, for offline evaluation: ``rank`` int64 [N] is the number of
        items ``topk`` on the same rows would put before ``target[r]`` (higher logit, equal logits the smaller id), so
        it is ``target``'s position in ``topk(state, k)`` when below k and the target is absent otherwise, at any k;
        ``log_prob`` fp32 [N] is log pi(target | state).  ``exclude``: a ``recnn_b200.data.ItemSets`` of ids that do
        not count (e.g. ``DeviceFrameFeed.seen_items()``), with ``exclude_rows`` as in ``topk``; a row's target is
        never excluded.  A target or excluded id outside [0, num_items) raises IndexError, a malformed table
        ValueError.  Never forms the [N, num_items] probabilities; on a vocabulary-parallel policy it ranks over the
        whole vocabulary (two all-gathers of O(N) records), on a data-parallel replica it stays local.  Inference
        only: nothing saved for the policy update is touched."""
        from .update.reinforce import _chunk_items
        from ..data.item_sets import ItemSets, row_map
        vp = self.__dict__.get("_recnn_vp")
        d = self.dims
        items = d.num_items if vp is None else vp.num_items
        if not torch.is_tensor(state) or state.dim() != 2 or state.shape[1] != d.state_dim:
            raise ValueError("state must be a [N, %d] tensor" % d.state_dim)
        n = state.shape[0]
        _check_row_ids(target, n, "target")
        sets = rows = None
        if isinstance(exclude, ItemSets):
            sets, rows = row_map(exclude, exclude_rows, n)
        elif exclude is not None:
            raise ValueError("exclude must be a recnn_b200.data.ItemSets (got %s)" % type(exclude).__name__)
        elif exclude_rows is not None:
            raise ValueError("exclude_rows maps rows to the sets of an ItemSets exclude")
        dev = self.linear1.weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
        rank = torch.empty(n, device=dev, dtype=torch.int64)
        logp = torch.empty(n, device=dev, dtype=torch.float32)
        if n == 0:
            return rank, logp
        _, (state,) = _device_check(self, state)
        target = target.detach().to(device=dev, dtype=torch.int64).contiguous()
        table = ()
        if sets is not None:
            sets = sets.to(dev)
            rows = None if rows is None else rows.to(dev).contiguous()
            table = (sets.ids.data_ptr() if sets.ids.numel() else None, sets.ids.numel(), sets.offsets.data_ptr(),
                     len(sets), _lib.ptr(rows))
        L = _lib.lib()
        flat = param_arena(self)
        chunk = _chunk_items(n, d.num_items)
        nbytes = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        flag = torch.zeros(2, dtype=torch.int32, device=dev)       # the call's bits, the table check's (sharded)
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            if vp is None and sets is None:
                _lib.check(L.recnn_discrete_rank(d, flat.data_ptr(), state.data_ptr(), target.data_ptr(), n, chunk,
                                                 rank.data_ptr(), logp.data_ptr(), flag.data_ptr(), ws.data_ptr(),
                                                 nbytes, st))
            elif vp is None:
                _lib.check(L.recnn_discrete_rank_sets(d, flat.data_ptr(), state.data_ptr(), target.data_ptr(), n,
                                                      *table, chunk, rank.data_ptr(), logp.data_ptr(),
                                                      flag.data_ptr(), ws.data_ptr(), nbytes, st))
            else:
                shard = vp.shard()
                stats = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
                _lib.check(L.recnn_discrete_shard_rank_stats(d, shard, flat.data_ptr(), state.data_ptr(),
                                                             target.data_ptr(), n, chunk, stats.data_ptr(),
                                                             ws.data_ptr(), nbytes, st))
                g_stats = vp.all_gather(stats)
                counts = torch.empty(L.recnn_vocab_rank_record_floats(n), device=dev, dtype=torch.float32)
                if sets is None:
                    _lib.check(L.recnn_discrete_shard_rank(d, shard, flat.data_ptr(), target.data_ptr(), n, chunk,
                                                           g_stats.data_ptr(), counts.data_ptr(), ws.data_ptr(),
                                                           nbytes, st))
                else:
                    _lib.check(L.recnn_discrete_shard_rank_sets(d, shard, flat.data_ptr(), target.data_ptr(), n,
                                                                *table, chunk, g_stats.data_ptr(), counts.data_ptr(),
                                                                flag[1:].data_ptr(), ws.data_ptr(), nbytes, st))
                del ws
                g_counts = vp.all_gather(counts)
                _lib.check(L.recnn_discrete_shard_rank_finish(d, shard, g_stats.data_ptr(), g_counts.data_ptr(),
                                                              target.data_ptr(), n, rank.data_ptr(), logp.data_ptr(),
                                                              flag.data_ptr(), st))
        f = flag.tolist()
        bits = f[0] | f[1]
        if bits & 2:
            raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
        if bits & 1:
            raise IndexError("a target or excluded item id is out of range for the policy's %d items" % items)
        if bits & 4:
            raise ValueError("malformed exclusion table: a set is not ascending, its offsets are out of range or "
                             "decreasing, or an exclude_rows entry is outside [-1, %d)" % len(sets))
        return rank, logp

    def log_prob(self, state, action):
        """fp32 [N]: log pi(action | state) of given (e.g. logged) item ids, the exact log-softmax z_a - M - log S --
        not the Categorical's clamped value -- for off-policy estimation
        (``recnn_b200.utils.metrics.off_policy_estimates``).  It is ``rank``'s pass 1 alone, so it equals ``rank``'s
        ``log_prob`` bit for bit at a lower cost, and never forms the [N, num_items] probabilities.  On a
        vocabulary-parallel policy it covers the whole vocabulary (one all-gather of O(N) records) and every rank
        returns the same bits; on a data-parallel replica it stays local.  A bad shape raises ValueError, an id
        outside [0, num_items) IndexError.  Inference only: nothing saved for the policy update is touched."""
        from .update.reinforce import _chunk_items
        vp = self.__dict__.get("_recnn_vp")
        d = self.dims
        items = d.num_items if vp is None else vp.num_items
        if not torch.is_tensor(state) or state.dim() != 2 or state.shape[1] != d.state_dim:
            raise ValueError("state must be a [N, %d] tensor" % d.state_dim)
        n = state.shape[0]
        _check_row_ids(action, n, "action")
        dev = self.linear1.weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
        logp = torch.empty(n, device=dev, dtype=torch.float32)
        if n == 0:
            return logp
        _, (state,) = _device_check(self, state)
        action = action.detach().to(device=dev, dtype=torch.int64).contiguous()
        L = _lib.lib()
        flat = param_arena(self)
        chunk = _chunk_items(n, d.num_items)
        nbytes = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            if vp is None:
                _lib.check(L.recnn_discrete_log_prob(d, flat.data_ptr(), state.data_ptr(), action.data_ptr(), n, chunk,
                                                     logp.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes, st))
            else:
                shard = vp.shard()
                stats = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
                _lib.check(L.recnn_discrete_shard_rank_stats(d, shard, flat.data_ptr(), state.data_ptr(),
                                                             action.data_ptr(), n, chunk, stats.data_ptr(),
                                                             ws.data_ptr(), nbytes, st))
                del ws
                gathered = vp.all_gather(stats)
                _lib.check(L.recnn_vocab_log_prob_finish(shard, gathered.data_ptr(), action.data_ptr(), n,
                                                         logp.data_ptr(), flag.data_ptr(), st))
        _log_prob_errors(int(flag.item()), items)
        return logp

    def gc(self):
        del self.rewards[:]
        del self.saved_log_probs[:]
        del self.correction[:]
        del self.lambda_k[:]
        del self._saved[:]

    # -- Categorical(probs).sample() / .log_prob() on the device ----------------------------------------------------
    def _row_offset(self, n):
        """On a data-parallel policy (recnn_b200.dist.enable_data_parallel) the global row of this call's first row,
        from the ranks' row counts (a collective); else None."""
        plan = self.__dict__.get("_recnn_rows")
        return None if plan is None else plan.rows(n)[0]

    def _sample(self, probs, gathered=None, row_offset=None):
        """(action int64 [N], log_prob fp32 [N]) of one draw per row.  ``gathered``: the records of the sharded
        forward that made ``probs`` (the rank's column block); the draw is then over the whole vocabulary.
        ``row_offset``: the global row of the first row (data parallel): row r draws the uniform of global row
        row_offset + r, what the single-GPU call over the whole batch draws for it."""
        n, items = probs.shape
        dev = probs.device
        action = torch.empty(n, dtype=torch.int64, device=dev)
        logp = torch.empty(n, dtype=torch.float32, device=dev)
        u = None
        if self.uniform_source is not None:
            u = torch.as_tensor(self.uniform_source(n)).to(device=dev, dtype=torch.float32).contiguous()
            if u.shape != (n,):
                raise ValueError("uniform_source must return %d values" % n)
        self._draws += 1
        seed = int(torch.initial_seed()) & (2 ** 64 - 1)
        with torch.cuda.device(dev):
            if gathered is None and row_offset is not None:
                _lib.check(_lib.lib().recnn_categorical_sample_at(
                    probs.data_ptr(), n, items, probs.stride(0), _lib.ptr(u), seed, self._draws, row_offset,
                    action.data_ptr(), logp.data_ptr(), _lib.stream_ptr(dev)))
                return action, logp
            if gathered is None:
                _lib.check(_lib.lib().recnn_categorical_sample(
                    probs.data_ptr(), n, items, probs.stride(0), _lib.ptr(u), seed, self._draws, action.data_ptr(),
                    logp.data_ptr(), _lib.stream_ptr(dev)))
                return action, logp
            draw = torch.empty(2 * n, dtype=torch.float32, device=dev)
            _lib.check(_lib.lib().recnn_discrete_shard_sample(
                self.dims, self._recnn_vp.shard(), gathered.data_ptr(), probs.data_ptr(), n, _lib.ptr(u), seed,
                self._draws, draw.data_ptr(), _lib.stream_ptr(dev)))
        self._shard_pick(draw, n, action, logp, None)
        return action, logp

    def _shard_pick(self, draw, n, action, logp, oob):
        """The owners' (id, log-prob) of every row from the ranks' draw records (the second all-gather)."""
        dev = draw.device
        gathered = self._recnn_vp.all_gather(draw)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().recnn_discrete_shard_pick(self._recnn_vp.world, gathered.data_ptr(), n,
                                                            action.data_ptr(), logp.data_ptr(), flag.data_ptr(),
                                                            _lib.stream_ptr(dev)))
        if oob is not None and int(oob.item()) != 0:
            raise IndexError("action index out of range for the policy's output layer")
        if int(flag.item()) != 0:
            raise RuntimeError("the ranks of a vocabulary-parallel policy drew different uniforms: seed every rank "
                               "the same (torch.manual_seed) or give each the same uniform_source")

    def _shard_log_prob(self, probs, action):
        """_log_prob of global ids on a sharded policy: from the owner's column block, through the second exchange."""
        n = probs.shape[0]
        dev = probs.device
        action = action.to(device=dev, dtype=torch.int64).contiguous()
        draw = torch.empty(2 * n, dtype=torch.float32, device=dev)
        oob = torch.zeros(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().recnn_discrete_shard_log_prob(self.dims, self._recnn_vp.shard(), probs.data_ptr(), n,
                                                                action.data_ptr(), draw.data_ptr(), oob.data_ptr(),
                                                                _lib.stream_ptr(dev)))
        logp = torch.empty(n, dtype=torch.float32, device=dev)
        self._shard_pick(draw, n, torch.empty(n, dtype=torch.int64, device=dev), logp, oob)
        return logp

    @staticmethod
    def _log_prob(probs, action):
        n, items = probs.shape
        dev = probs.device
        logp = torch.empty(n, dtype=torch.float32, device=dev)
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        action = action.to(device=dev, dtype=torch.int64).contiguous()
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().recnn_categorical_log_prob(probs.data_ptr(), n, items, probs.stride(0),
                                                             action.data_ptr(), logp.data_ptr(), flag.data_ptr(),
                                                             _lib.stream_ptr(dev)))
        if int(flag.item()) != 0:
            raise IndexError("action index out of range for the policy's output layer")
        return logp

    @staticmethod
    def _as_probs(t, dev):
        t = t.detach().to(device=dev, dtype=torch.float32)
        return t if t.stride(1) == 1 else t.contiguous()

    def _select_action(self, state, **kwargs):
        # REINFORCE without correction: only pi is available, the action source is ignored (models.py:102-111)
        dev, (state,) = _device_check(self, state)
        pi_probs, gathered = self._pi(state)
        pi_action, pi_log_prob = self._sample(pi_probs, gathered, self._row_offset(state.shape[0]))
        self.saved_log_probs.append(pi_log_prob)
        self._saved.append({"state": state.clone(), "action": pi_action, "beta_log_prob": None})
        return pi_probs

    def _beta_records(self, beta_out):
        """The gathered records of a sharded Beta's column block ``beta_out`` (None for full probabilities); refuses
        a beta output this policy cannot draw from."""
        from .beta import block_records
        vp = self.__dict__.get("_recnn_vp")
        found = block_records(beta_out)
        if found is not None:
            if vp is None:
                raise ValueError("beta returned the column block of a vocabulary-parallel Beta, but the policy is not "
                                 "vocabulary-parallel: shard both with enable_vocab_parallel(..., beta=)")
            bvp = found[1]
            if (bvp.lo, bvp.hi, bvp.num_items, bvp.rank, bvp.world) != (vp.lo, vp.hi, vp.num_items, vp.rank, vp.world):
                raise ValueError("beta is sharded on items [%d, %d) of %d, the policy on [%d, %d) of %d: shard them in "
                                 "one enable_vocab_parallel(..., beta=) call"
                                 % (bvp.lo, bvp.hi, bvp.num_items, vp.lo, vp.hi, vp.num_items))
            return found[0]
        if vp is not None and (beta_out.dim() != 2 or beta_out.shape[1] != vp.num_items):
            block = beta_out.dim() == 2 and beta_out.shape[1] == vp.hi - vp.lo
            raise ValueError("beta must return probabilities [N, %d] or the column block of a Beta sharded with the "
                             "policy (got shape %s)%s"
                             % (vp.num_items, tuple(beta_out.shape),
                                ": a column block without its records (a copy, or not the Beta's latest output)"
                                if block else ""))
        return None

    def pi_beta_sample(self, state, beta, action, **kwargs):
        """models.py:113-145.  ``beta`` is any callable (state, action=...) -> probabilities [N, action_dim]; on a
        vocabulary-parallel policy also the rank's column block a Beta sharded with it returned (its latest output,
        as returned: the block's draw needs the records of the Beta's call)."""
        dev, (state,) = _device_check(self, state)
        beta_out = beta(state.detach(), action=action)
        beta_gathered = self._beta_records(beta_out) if torch.is_tensor(beta_out) else None
        beta_probs = self._as_probs(beta_out, dev)
        pi_probs, gathered = self._pi(state)
        row_offset = self._row_offset(state.shape[0])
        # the pi draw is made first, then the beta draw (models.py:133-136)
        pi_draw = self._sample(pi_probs, gathered, row_offset)
        beta_draw = self._sample(beta_probs, beta_gathered, row_offset)
        available = {"pi": (pi_draw, pi_probs), "beta": (beta_draw, beta_probs)}
        (pi_action, pi_lp), src_pi = available[self.action_source["pi"]]
        (beta_action, beta_lp), src_beta = available[self.action_source["beta"]]
        if src_pi is pi_probs:
            pi_log_prob = pi_lp
        elif gathered is None:
            pi_log_prob = self._log_prob(pi_probs, pi_action)
        else:
            pi_log_prob = self._shard_log_prob(pi_probs, pi_action)
        if src_beta is beta_probs:
            beta_log_prob = beta_lp
        elif beta_gathered is None:
            beta_log_prob = self._log_prob(beta_probs, beta_action)
        else:
            beta_log_prob = self._shard_log_prob(beta_probs, beta_action)
        self._last_sample = {"state": state, "action": pi_action, "beta_log_prob": beta_log_prob}
        return pi_log_prob, beta_log_prob, pi_probs

    def _select_action_with_correction(self, state, beta, action, writer, step, **kwargs):
        pi_log_prob, beta_log_prob, pi_probs = self.pi_beta_sample(state, beta, action)
        corr = torch.exp(pi_log_prob) / torch.exp(beta_log_prob)
        writer.add_histogram("correction", corr, step)
        writer.add_histogram("pi_log_prob", pi_log_prob, step)
        writer.add_histogram("beta_log_prob", beta_log_prob, step)
        self.correction.append(corr)
        self.saved_log_probs.append(pi_log_prob)
        rec = self._last_sample
        self._saved.append({"state": rec["state"].clone(), "action": rec["action"], "beta_log_prob": rec["beta_log_prob"]})
        return pi_probs

    def _select_action_with_TopK_correction(self, state, beta, action, K, writer, step, **kwargs):
        pi_log_prob, beta_log_prob, pi_probs = self.pi_beta_sample(state, beta, action)
        corr = torch.exp(pi_log_prob) / torch.exp(beta_log_prob)
        l_k = K * (1 - torch.exp(pi_log_prob)) ** (K - 1)
        writer.add_histogram("correction", corr, step)
        writer.add_histogram("l_k", l_k, step)
        writer.add_histogram("pi_log_prob", pi_log_prob, step)
        writer.add_histogram("beta_log_prob", beta_log_prob, step)
        self.correction.append(corr)
        self.lambda_k.append(l_k)
        self.saved_log_probs.append(pi_log_prob)
        rec = self._last_sample
        self._saved.append({"state": rec["state"].clone(), "action": rec["action"], "beta_log_prob": rec["beta_log_prob"],
                            "K": int(K)})
        return pi_probs
