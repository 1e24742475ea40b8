"""Actor / Critic / DiscreteActor with the reference's constructor, attributes and state_dict
layout (recnn/nn/models.py:41-73, :76-184, :187-213), evaluated by the sm_90a kernels.

``forward`` is the inference / evaluation entry (no autograd graph): training
goes through recnn_b200.nn.update.*, which runs forward+backward+optimizer as
one fused device step.  There is no CPU implementation behind ``forward`` --
calling it on CPU tensors raises.
"""
from __future__ import annotations

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

    def topk(self, state, k, exclude=None):
        """``(values, indices)`` as ``torch.topk(self(state), k)`` without forming the [N, num_items] probabilities:
        the k items of highest logit per row (equal logits: the smaller id first), values fp32 [N, k] = pi(a|s),
        indices int64 [N, k] global item ids, on a vocabulary-parallel policy too (one all-gather of k candidates per
        row and rank).  ``exclude``: optional integer [N, E] (E <= 256) of ids never returned -- e.g. the frame's
        items -- that stay in the softmax's normaliser (values are not renormalised); negative ids are padding, an
        id >= num_items raises IndexError.  A row with fewer than k eligible items ends in id -1, value 0.
        1 <= k <= min(64, num_items).  Inference only: nothing saved for the policy update is touched."""
        from .update.reinforce import _chunk_items
        vp = self.__dict__.get("_recnn_vp")
        d = self.dims
        items = d.num_items if vp is None else vp.num_items
        if isinstance(k, bool) or not isinstance(k, int) or not 1 <= k <= min(64, items):
            raise ValueError("k must be an int in [1, min(64, num_items)] = [1, %d], got %r" % (min(64, items), k))
        if not torch.is_tensor(state) or state.dim() != 2 or state.shape[1] != d.state_dim:
            raise ValueError("state must be a [N, %d] tensor" % d.state_dim)
        n = state.shape[0]
        n_ex = 0
        if exclude is not None:
            if (not torch.is_tensor(exclude) or exclude.dim() != 2 or exclude.shape[0] != n
                    or exclude.shape[1] > 256 or exclude.dtype.is_floating_point or exclude.dtype == torch.bool):
                raise ValueError("exclude must be an integer tensor [N, E] with N = %d rows and E <= 256 (got %s)"
                                 % (n, tuple(exclude.shape) if torch.is_tensor(exclude) else type(exclude).__name__))
            n_ex = exclude.shape[1]
        dev = self.linear1.weight.device
        if dev.type != "cuda":
            raise _lib.RecnnError("recnn_b200 nets run on CUDA only (module is on %s); call .cuda() first" % dev)
        values = torch.empty(n, k, device=dev, dtype=torch.float32)
        ids = torch.empty(n, k, device=dev, dtype=torch.int64)
        if n == 0:
            return values, ids
        _, (state,) = _device_check(self, state)
        ex = None if n_ex == 0 else exclude.detach().to(device=dev, dtype=torch.int64).contiguous()
        L = _lib.lib()
        flat = param_arena(self)
        chunk = _chunk_items(n, d.num_items)
        nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
        ws = torch.empty(nbytes, device=dev, dtype=torch.uint8)
        flag = torch.empty(1, dtype=torch.int32, device=dev)
        with torch.cuda.device(dev):
            if vp is None:
                _lib.check(L.recnn_discrete_topk(d, flat.data_ptr(), state.data_ptr(), n, k, _lib.ptr(ex), n_ex, chunk,
                                                 values.data_ptr(), ids.data_ptr(), flag.data_ptr(), ws.data_ptr(),
                                                 nbytes, _lib.stream_ptr(dev)))
            else:
                shard = vp.shard()
                rec = torch.empty(L.recnn_vocab_topk_record_floats(n, k), device=dev, dtype=torch.float32)
                _lib.check(L.recnn_discrete_shard_topk(d, shard, flat.data_ptr(), state.data_ptr(), n, k, _lib.ptr(ex),
                                                       n_ex, chunk, rec.data_ptr(), ws.data_ptr(), nbytes,
                                                       _lib.stream_ptr(dev)))
                del ws
                gathered = vp.all_gather(rec)
                _lib.check(L.recnn_discrete_shard_topk_finish(d, shard, gathered.data_ptr(), n, k, _lib.ptr(ex), n_ex,
                                                              values.data_ptr(), ids.data_ptr(), flag.data_ptr(),
                                                              _lib.stream_ptr(dev)))
        bits = int(flag.item())
        if bits & 2:
            raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
        if bits & 1:
            raise IndexError("an excluded item id is out of range for the policy's %d items" % items)
        return values, ids

    def gc(self):
        del self.rewards[:]
        del self.saved_log_probs[:]
        del self.correction[:]
        del self.lambda_k[:]
        del self._saved[:]

    # -- Categorical(probs).sample() / .log_prob() on the device ----------------------------------------------------
    def _sample(self, probs, gathered=None):
        """(action int64 [N], log_prob fp32 [N]) of one draw per row.  ``gathered``: the records of the sharded
        forward that made ``probs`` (the rank's column block); the draw is then over the whole vocabulary."""
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
        pi_action, pi_log_prob = self._sample(pi_probs, gathered)
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
        # the pi draw is made first, then the beta draw (models.py:133-136)
        pi_draw = self._sample(pi_probs, gathered)
        beta_draw = self._sample(beta_probs, beta_gathered)
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
