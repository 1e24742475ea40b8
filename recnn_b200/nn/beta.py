"""The behaviour policy beta of REINFORCE with Top-K off-policy correction.

The reference does not ship it in its library: the Top-K notebook defines it (examples/2. REINFORCE TopK Off Policy
Correction/3. TopK Reinforce Off Policy Correction.ipynb, cell 3) and passes ``beta_net.forward`` to
``DiscreteActor._select_action_with_TopK_correction``.  ``Beta`` here has that class's attributes (``net``, ``optim``,
``criterion``), state_dict keys and call contract -- every ``forward(state, action)`` trains once and returns the
probabilities from before the step -- and runs the whole call as one device step (recnn_beta_step): the items are
visited in chunks, so besides the dense output nothing of size [N, num_items] is allocated, and the optimizer is the
built-in RAdam (torch_optimizer is not installable next to the notebook's code here).

``recnn_b200.dist.enable_vocab_parallel(policy_or_agent, beta=beta_net)`` shards a Beta over the item vocabulary with
the policy: each rank keeps rows [lo, hi) of ``net.0`` and ``forward`` returns the rank's column block [N, hi - lo] of
the probabilities (recnn_beta_shard_* in include/recnn_b200.h).  ``recnn_b200.dist.enable_data_parallel(agent,
beta=beta_net)`` keeps a full replica on every rank instead: a call on the rank's rows steps on the cross-entropy mean
over every rank's rows (the gradient all-reduced), so the replicas stay identical.
"""
from __future__ import annotations

import weakref

import torch
import torch.nn as nn

from .. import _lib
from .. import optim as _optim
from .arena import param_arena, grad_arena
from .update import _ids
from .update.reinforce import _chunk_items


# The sharded Betas, held weakly: block_records() finds the one that returned a given block.
_SHARDED = weakref.WeakSet()


def block_records(t):
    """(gathered records of exchange 1, VocabParallel) of the column block ``t`` a sharded Beta's last call returned,
    or None (``t`` is not such a block: a replicated Beta's output, a copy, or an older block)."""
    for beta in list(_SHARDED):
        held = beta.__dict__.get("_recnn_block")
        if held is not None and held[0]() is t:
            return held[1], beta.__dict__["_recnn_vp"]
    return None


class Beta(nn.Module):
    """``Beta(input_dim, num_items)``: the notebook's cell 3 with its hard-wired 1290 and ``num_items`` as arguments.

    As in the notebook, the loss is ``CrossEntropyLoss`` applied to the softmax *probabilities* (a softmax of a
    softmax), and ``action`` is a one-hot [N, num_items] float matrix whose ``argmax(1)`` is the target.  Item ids
    (an integer tensor [N], as ``batch_contstate_discaction(..., one_hot=False)`` gives) are accepted too.  The loss
    of the last call stays on the device in ``last_loss``.  Replacing ``optim`` by a torch optimizer makes the call
    stop after the gradient (left in ``.grad``) and call its ``step()``.

    Sharded over the item vocabulary (``recnn_b200.dist.enable_vocab_parallel(..., beta=)``), a call returns the rank's
    column block [N, hi - lo] of the probabilities; ``action`` stays a one-hot [N, num_items] row or global item ids, and
    ``last_loss`` is the loss over the whole vocabulary, the same on every rank.  Every rank must make the same calls
    with the same states and actions."""

    _recnn_beta = True

    def __init__(self, input_dim, num_items, lr=1e-5, weight_decay=1e-5):
        super().__init__()
        self.net = nn.Sequential(nn.Linear(input_dim, num_items), nn.Softmax(dim=1))
        self.optim = _optim.RAdam(self.net.parameters(), lr=lr, weight_decay=weight_decay)
        self.criterion = nn.CrossEntropyLoss()
        self.last_loss = None
        self._workspace = None

    @property
    def dims(self):
        lin = self.net[0]
        return _lib.BetaDims(lin.in_features, lin.out_features, (0, 0))

    def _targets(self, action, n, num_items):
        """int64 target ids [n] from a one-hot [n, num_items] action (argmax(1): the first maximum) or from ids [n]."""
        if not torch.is_tensor(action):
            action = torch.as_tensor(action)
        if _ids.is_item_ids(action):
            if action.shape[0] != n:
                raise ValueError("%d item ids for %d state rows" % (action.shape[0], n))
            return action
        if tuple(action.shape) != (n, num_items):
            raise ValueError("action must be one-hot [%d, %d] or item ids [%d] (got shape %s)"
                             % (n, num_items, n, tuple(action.shape)))
        return action.argmax(1)

    def _states(self, state):
        """``state`` as a tensor [N, state_dim] (ValueError otherwise)."""
        d = self.dims
        if not torch.is_tensor(state):
            state = torch.as_tensor(state)
        if state.dim() != 2 or state.shape[1] != d.state_dim:
            raise ValueError("state must be [N, %d] (got shape %s)" % (d.state_dim, tuple(state.shape)))
        return state

    def forward(self, state, action):
        d = self.dims
        state = self._states(state)
        n = int(state.shape[0])
        vp = self.__dict__.get("_recnn_vp")
        self.__dict__.pop("_recnn_block", None)
        target = self._targets(action, n, d.num_items if vp is None else vp.num_items)
        dev = self.net[0].weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (Beta is on %s); call .cuda() first" % dev)
        if n == 0:
            raise ValueError("an empty batch has no cross-entropy mean")
        with torch.cuda.device(dev):
            state = state.detach().to(device=dev, dtype=torch.float32)
            if state.stride(1) != 1:
                state = state.contiguous()
            target = target.detach().to(device=dev, dtype=torch.int64).contiguous()
            opt = self.optim
            builtin = isinstance(opt, _optim._ArenaOptimizer)
            if builtin:
                # not bind(): the Beta holds its optimizer, so a back reference would make a cycle that keeps the
                # [num_items, S] arenas on the device until the garbage collector runs
                if [id(p) for p in opt.param_groups[0]["params"]] != [id(p) for p in self.net.parameters()]:
                    raise ValueError("Beta.optim must own exactly this Beta's parameters (net.0.weight, net.0.bias)")
                net = opt.c_net(self)
                c_opt = opt.c_optim()
            else:
                net = _lib.Net(param_arena(self).data_ptr(), grad_arena(self).data_ptr(), None, None, None, None)
                c_opt = _lib.Optim(_lib.OPT_EXTERNAL, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
            probs = torch.empty(n, d.num_items, device=dev, dtype=torch.float32)
            loss = torch.empty((), device=dev, dtype=torch.float32)
            error = torch.zeros(1, device=dev, dtype=torch.int32)
            L = _lib.lib()
            a = _lib.BetaArgs()
            a.dims = d
            a.n_rows = n
            a.chunk_items = _chunk_items(n, d.num_items)
            a.net, a.optim = net, c_opt
            a.state, a.state_ld = state.data_ptr(), state.stride(0)
            a.action, a.probs_out = target.data_ptr(), probs.data_ptr()
            a.loss, a.error = loss.data_ptr(), error.data_ptr()
            nbytes = L.recnn_beta_workspace_bytes(d, n, a.chunk_items)
            if self._workspace is None or self._workspace.device != dev or self._workspace.numel() < nbytes:
                self._workspace = None
                self._workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            a.workspace, a.workspace_bytes = self._workspace.data_ptr(), self._workspace.numel()
            rows = self.__dict__.get("_recnn_rows")
            if rows is not None:
                loss, error = self._row_parallel_grad(a, rows, n, dev, loss, error)
            elif vp is None:
                _lib.check(L.recnn_beta_step(a, _lib.stream_ptr(dev)))
            else:
                gathered = self._sharded_step(a, vp, n, dev)
            self.last_loss = loss
            err = int(error.item())            # the call's one synchronisation
            if err & 2:
                raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows: no "
                                   "optimizer step was taken")
            if err != 0:
                raise IndexError("action holds an item id outside [0, num_items): no optimizer step was taken")
            if rows is not None and builtin:
                _lib.check(L.recnn_optimizer_step(c_opt, net, param_arena(self).numel(), None, _lib.stream_ptr(dev)))
            if not builtin:
                grad_arena(self)               # re-attach p.grad views if zero_grad(set_to_none) dropped them
                opt.step()
        if vp is not None:
            self.__dict__["_recnn_block"] = (weakref.ref(probs), gathered)
        return probs

    def log_prob(self, state, action):
        """fp32 [N]: log beta(action | state) of given (e.g. logged) actions -- item ids [N] or a one-hot
        [N, num_items] matrix, as ``forward`` takes -- the exact log-softmax of the logits, for off-policy estimation
        (``recnn_b200.utils.metrics.off_policy_estimates``).  Inference only: unlike ``forward`` it takes no step, and
        ``last_loss``, the weights, the optimizer state and the sharded block of the last ``forward`` stay as they
        are; nothing of size [N, num_items] is allocated.  On a vocabulary-parallel Beta it covers the whole vocabulary
        (one all-gather of O(N) records) and every rank returns the same bits; on a data-parallel replica it stays
        local.  A bad shape raises ValueError, an id outside [0, num_items) IndexError."""
        from .models import _log_prob_errors
        d = self.dims
        state = self._states(state)
        n = int(state.shape[0])
        vp = self.__dict__.get("_recnn_vp")
        items = d.num_items if vp is None else vp.num_items
        target = self._targets(action, n, items)
        dev = self.net[0].weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (Beta is on %s); call .cuda() first" % dev)
        logp = torch.empty(n, device=dev, dtype=torch.float32)
        if n == 0:
            return logp
        L = _lib.lib()
        st = _lib.stream_ptr(dev)
        with torch.cuda.device(dev):
            state = state.detach().to(device=dev, dtype=torch.float32)
            if state.stride(1) != 1:
                state = state.contiguous()
            target = target.detach().to(device=dev, dtype=torch.int64).contiguous()
            flat = param_arena(self)
            chunk = _chunk_items(n, d.num_items)
            nbytes = L.recnn_beta_log_prob_workspace_bytes(d, n, chunk)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            flag = torch.zeros(1, dtype=torch.int32, device=dev)
            if vp is None:
                _lib.check(L.recnn_beta_log_prob(d, flat.data_ptr(), state.data_ptr(), state.stride(0),
                                                 target.data_ptr(), n, chunk, logp.data_ptr(), flag.data_ptr(),
                                                 ws.data_ptr(), nbytes, st))
            else:
                shard = vp.shard()
                rec = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
                _lib.check(L.recnn_beta_shard_log_prob_stats(d, shard, flat.data_ptr(), state.data_ptr(),
                                                             state.stride(0), target.data_ptr(), n, chunk,
                                                             rec.data_ptr(), ws.data_ptr(), nbytes, st))
                del ws
                gathered = vp.all_gather(rec)
                _lib.check(L.recnn_vocab_log_prob_finish(shard, gathered.data_ptr(), target.data_ptr(), n,
                                                         logp.data_ptr(), flag.data_ptr(), st))
        _log_prob_errors(int(flag.item()), items)
        return logp

    def _row_parallel_grad(self, a, rows, n, dev, loss, error):
        """Data parallel: this rank's rows' share of the gradient of the cross-entropy mean over the global batch,
        all-reduced with the loss partial and the error flag.  Returns (loss, error) -- the same bits on every rank;
        the caller steps the optimizer on every rank or, on an error, on none."""
        a.n_rows_global = rows.rows(n)[1]
        a.optim = _lib.Optim(_lib.OPT_EXTERNAL, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0)
        _lib.check(_lib.lib().recnn_beta_step(a, _lib.stream_ptr(dev)))
        rows.all_reduce(grad_arena(self))
        tail = torch.cat([loss.reshape(1), (error != 0).float()])
        rows.all_reduce(tail)
        return tail[0], (tail[1:] > 0).to(torch.int32)

    def _sharded_step(self, a, vp, n, dev):
        """begin -> all-gather -> rows -> all-gather -> end; returns the gathered records of the first exchange."""
        L = _lib.lib()
        shard = vp.shard()
        st = _lib.stream_ptr(dev)
        rec = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
        _lib.check(L.recnn_beta_shard_begin(a, shard, rec.data_ptr(), st))
        gathered = vp.all_gather(rec)
        sums = torch.empty_like(rec)
        _lib.check(L.recnn_beta_shard_rows(a, shard, gathered.data_ptr(), sums.data_ptr(), st))
        _lib.check(L.recnn_beta_shard_end(a, shard, vp.all_gather(sums).data_ptr(), st))
        return gathered
