"""Item-id actions for the REINFORCE critic (recnn/nn/update/reinforce.py:92-102 -> misc.py:10-55).

The reference feeds the critic the batch action as a dense one-hot [N, num_items] and the target policy's
probabilities [N, num_items].  When ``batch["action"]`` is an integer tensor of item ids [N] instead, the critic step is
``recnn_discrete_value_step``: the one-hot product is a gathered weight column, the target policy's probabilities are
streamed over item chunks straight into the target critic's layer 1, and the action block of the gradient is a
scatter of the selected columns.  Nothing of size [N, num_items] is allocated, so the step fits at a million items.
"""
from __future__ import annotations

import torch

from ... import _lib
from ... import optim as _optim
from ..arena import param_arena, grad_arena
from ._engine import MASK_KEY


def is_item_ids(action) -> bool:
    """True when ``action`` is an item-id batch action (an integer tensor [N]); raises ValueError for the shapes that
    are neither that nor the dense [N, num_items] action (a float [N] tensor, an integer matrix)."""
    if not torch.is_tensor(action):
        action = torch.as_tensor(action)
    integer = not (action.dtype.is_floating_point or action.dtype.is_complex or action.dtype == torch.bool)
    if action.dim() == 1:
        if not integer:
            raise ValueError("a 1-D batch['action'] must hold integer item ids (got %s)" % action.dtype)
        return True
    if integer:
        raise ValueError("an integer batch['action'] must be 1-D item ids [N] (got shape %s)" % (tuple(action.shape),))
    return False


def reject_ids(batch, what):
    """The update steps that have no item-id mode (DDPG / TD3 with an Actor policy) refuse such a batch."""
    if batch.get("action") is not None and is_item_ids(batch["action"]):
        raise ValueError("%s has no item-id action mode: item ids go with a DiscreteActor target policy and the "
                         "DDPG-style critic step (value_update / reinforce_update)" % what)


def _is_discrete(net):
    return hasattr(net, "linear2") and not hasattr(net, "linear3")


def _chunk(rows, num_items):
    from .reinforce import _chunk_items           # the policy gradient's chunk rule (reinforce.py imports this module)
    return _chunk_items(rows, num_items)


def _stream_device(net):
    dev = net.linear1.weight.device
    if dev.type != "cuda":
        raise _lib.RecnnError("recnn_b200 nets run on CUDA only (net is on %s)" % dev)
    return dev


def _critic_dims(value_net, num_items):
    S = value_net.linear1.in_features - num_items
    return _lib.Dims(S, num_items, value_net.linear1.out_features, 0)


def critic_action_term(value_net, probs=None, policy=None, state=None, chunk_items=None):
    """[N, H] = probs @ W1a^T for the critic's action block W1a = linear1.weight[:, S:], from dense probabilities or from
    ``policy(state)`` (softmax folded over item chunks).  No [N, num_items] buffer is allocated for a policy source."""
    dev = _stream_device(value_net)
    if (probs is None) == (policy is None):
        raise ValueError("give probs or (policy, state)")
    if probs is not None:
        probs = probs.detach().to(device=dev, dtype=torch.float32)
        if probs.stride(1) != 1:
            probs = probs.contiguous()
        n, items = probs.shape
    else:
        state = state.detach().to(device=dev, dtype=torch.float32).contiguous()
        n, items = state.shape[0], policy.linear2.out_features
    d = _critic_dims(value_net, items)
    pd = policy.dims if policy is not None else None
    chunk = chunk_items if chunk_items is not None else _chunk(n, items)
    L = _lib.lib()
    out = torch.empty(n, d.hidden, device=dev, dtype=torch.float32)
    if n == 0:
        return out
    scratch = torch.empty(L.recnn_critic_action_term_scratch_floats(d, pd, n, chunk), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(L.recnn_critic_action_term_chunked(
            d, param_arena(value_net).data_ptr(), pd, None if policy is None else param_arena(policy).data_ptr(),
            None if state is None else state.data_ptr(), None if probs is None else probs.data_ptr(),
            0 if probs is None else probs.stride(0), n, chunk, out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
    return out


def critic_value_of_probs(value_net, state, probs):
    """value_net(state, probs) [N, 1] through the chunked action term instead of a re-pitched [N, num_items] image
    (same dropout convention as Critic.forward: fresh masks in train mode).  On a vocabulary-parallel critic ``probs``
    is the rank's column block: the ranks' action terms are all-reduced, and the value is the same on every rank."""
    from ..models import _train_masks
    dev = _stream_device(value_net)
    state = state.detach().to(device=dev, dtype=torch.float32).contiguous()
    n, items = probs.shape
    d = _critic_dims(value_net, items)
    term = critic_action_term(value_net, probs=probs)
    vp = value_net.__dict__.get("_recnn_vp")
    if vp is not None and n > 0:
        vp.all_reduce(term)
    m1, m2 = _train_masks(value_net, n, d.hidden, dev)
    out = torch.empty(n, 1, device=dev, dtype=torch.float32)
    if n == 0:
        return out
    L = _lib.lib()
    scratch = torch.empty(L.recnn_forward_scratch_floats(d, n, 0), device=dev, dtype=torch.float32)
    with torch.cuda.device(dev):
        _lib.check(L.recnn_critic_forward_action_term(
            d, param_arena(value_net).data_ptr(), state.data_ptr(), term.data_ptr(), n, _lib.ptr(m1), _lib.ptr(m2),
            out.data_ptr(), scratch.data_ptr(), _lib.stream_ptr(dev)))
    return out


class IdsValueStep:
    """Host side of recnn_discrete_value_step for one set of nets: staging, arenas, the optimizer and the single
    synchronisation that reads the loss and the error bits back."""

    def __init__(self, nets, device):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise _lib.RecnnError("recnn_b200 update functions run on CUDA only (device=%s); there is no CPU path"
                                  % self.device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        policy, value = nets["target_policy_net"], nets["value_net"]
        if not _is_discrete(policy):
            raise ValueError("item-id actions need a DiscreteActor target policy (nets['target_policy_net'])")
        self.pdims = policy.dims
        items = self.pdims.num_items
        self.dims = _critic_dims(value, items)
        if (self.dims.state_dim != self.pdims.state_dim or value.linear3.out_features != 1
                or nets["target_value_net"].linear1.weight.shape != value.linear1.weight.shape):
            raise ValueError("critic shape does not match the policy (expects input state_dim + num_items, 1 output)")
        self.seed = int(torch.initial_seed()) & 0xFFFFFFFFFFFFFFFF
        self.losses = torch.zeros(8, dtype=torch.float32, device=self.device)
        self.losses_host = torch.zeros(8, dtype=torch.float32).pin_memory()
        self.rng_step = torch.zeros(1, dtype=torch.int64, device=self.device)
        self.workspace = None

    def _net(self, module, opt, with_grads):
        flat = param_arena(module)
        if flat.device != self.device:
            raise _lib.RecnnError("net is on %s but the update runs on %s" % (flat.device, self.device))
        if not with_grads:
            return _lib.Net(flat.data_ptr(), None, None, None, None, None)
        if isinstance(opt, _optim._ArenaOptimizer):
            if opt._module is not module:
                opt.bind(module)
            return opt.c_net(module)
        return _lib.Net(flat.data_ptr(), grad_arena(module).data_ptr(), None, None, None, None)

    def run(self, batch, params, nets, optimizer, learn, debug):
        dev = self.device
        with torch.cuda.device(dev):
            f32 = dict(device=dev, dtype=torch.float32)
            state = torch.as_tensor(batch["state"]).detach().to(**f32).contiguous()
            next_state = torch.as_tensor(batch["next_state"]).detach().to(**f32).contiguous()
            action = torch.as_tensor(batch["action"]).detach().to(device=dev, dtype=torch.int64).contiguous()
            n = int(action.shape[0])
            reward = torch.as_tensor(batch["reward"]).detach().to(**f32).reshape(n).contiguous()
            done = torch.as_tensor(batch["done"]).detach().to(**f32).reshape(n).contiguous()
            d, pd = self.dims, self.pdims
            if tuple(state.shape) != (n, d.state_dim) or tuple(next_state.shape) != (n, d.state_dim):
                raise ValueError("batch shapes do not match the nets")
            value = nets["value_net"]
            H = d.hidden
            masks = batch.get(MASK_KEY)
            if masks is not None:
                if len(masks) not in (2, 6):
                    raise ValueError("%s needs the six masks of the DDPG step (or the critic's two)" % MASK_KEY)
                masks = [torch.as_tensor(m).to(device=dev, dtype=torch.uint8).reshape(n, H).contiguous()
                         for m in masks[:2]]
            vo = optimizer.get("value_optimizer") if learn else None
            a = _lib.DiscreteValueArgs()
            a.dims, a.policy_dims = d, pd
            a.learn = int(bool(learn))
            a.dropout = int(bool(value.training))
            a.chunk_items = _chunk(n, pd.num_items)
            a.n_rows = n
            a.state, a.next_state, a.action = state.data_ptr(), next_state.data_ptr(), action.data_ptr()
            a.reward, a.done = reward.data_ptr(), done.data_ptr()
            a.value = self._net(value, vo, learn)
            a.target_value = self._net(nets["target_value_net"], None, False)
            a.target_policy = param_arena(nets["target_policy_net"]).data_ptr()
            a.value_optim = (vo.c_optim() if isinstance(vo, _optim._ArenaOptimizer)
                             else _lib.Optim(_lib.OPT_EXTERNAL, 0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0))
            a.gamma = float(params["gamma"])
            a.min_value = float(params["min_value"])
            a.max_value = float(params["max_value"])
            if masks is not None and value.training:
                a.masks[0], a.masks[1] = masks[0].data_ptr(), masks[1].data_ptr()
            a.seed = self.seed
            a.rng_step = self.rng_step.data_ptr()
            a.losses = self.losses.data_ptr()
            a.losses_host = self.losses_host.data_ptr()
            L = _lib.lib()
            nbytes = L.recnn_discrete_value_workspace_bytes(d, pd, n, a.chunk_items)
            if self.workspace is None or self.workspace.numel() < nbytes:
                self.workspace = None
                self.workspace = torch.empty(nbytes, dtype=torch.uint8, device=dev)
            a.workspace = self.workspace.data_ptr()
            a.workspace_bytes = self.workspace.numel()
            self._launch(L, a, dev)
            if learn and a.value_optim.kind == _lib.OPT_EXTERNAL and vo is not None:
                grad_arena(value)          # re-attach p.grad views if zero_grad(set_to_none) dropped them
                vo.step()
            torch.cuda.current_stream(dev).synchronize()
            bits = int(self.losses_host.view(torch.int32)[4])
            if bits & 2:
                raise RuntimeError("the ranks disagree on the vocabulary shard plan or on the number of rows")
            if bits & 1:
                raise IndexError("batch['action'] holds an item id outside [0, num_items) (the update was applied with "
                                 "the offending rows' action term set to zero)")
            if not learn:
                debug["next_action"] = nets["target_policy_net"](next_state)       # the reference's debug contract
            return float(self.losses_host[0])

    def _launch(self, L, a, dev):
        _lib.check(L.recnn_discrete_value_step(a, _lib.stream_ptr(dev)))


class ShardedIdsValueStep(IdsValueStep):
    """IdsValueStep of nets sharded over the item vocabulary (recnn_b200.dist.enable_vocab_parallel on the agent): the
    critics hold the action columns of the rank's item block, the target policy its rows.  The step is the three phases
    of recnn_discrete_value_shard_* with an all-gather of the records and an all-reduce of the [2, N, H] action terms
    between them; the loss and the error bits come back with the same single synchronisation and are the same on every
    rank."""

    def __init__(self, nets, device):
        super().__init__(nets, device)
        self.vp = nets["value_net"].__dict__["_recnn_vp"]

    def _launch(self, L, a, dev):
        vp, shard, st = self.vp, self.vp.shard(), _lib.stream_ptr(dev)
        n = a.n_rows
        record = torch.empty(L.recnn_vocab_record_floats(n), device=dev, dtype=torch.float32)
        _lib.check(L.recnn_discrete_value_shard_begin(a, shard, record.data_ptr(), st))
        gathered = vp.all_gather(record)
        terms = torch.empty(2 * n * a.dims.hidden, device=dev, dtype=torch.float32)
        _lib.check(L.recnn_discrete_value_shard_merge(a, shard, gathered.data_ptr(), terms.data_ptr(), st))
        vp.all_reduce(terms)
        _lib.check(L.recnn_discrete_value_shard_end(a, shard, terms.data_ptr(), st))


def vocab_parallel_of(nets, names=("value_net", "target_value_net", "target_policy_net")):
    """The VocabParallel the named nets share, or None when none is sharded; RuntimeError when only some are, or they
    were sharded apart."""
    vps = [nets[k].__dict__.get("_recnn_vp") for k in names]
    if all(v is None for v in vps):
        return None
    if any(v is not vps[0] for v in vps):
        raise RuntimeError("%s must be sharded together: recnn_b200.dist.enable_vocab_parallel(agent or nets dict)"
                           % ", ".join(names))
    return vps[0]


def get_ids_step(nets, device) -> IdsValueStep:
    """Cached on the value net, like the step engines on the policy net."""
    if nets["policy_net"].__dict__.get("_recnn_dp") is not None and nets["policy_net"].__dict__["_recnn_dp"][1] > 1:
        raise ValueError("item-id actions run on one GPU: data parallel is not supported in this mode")
    cls = IdsValueStep if vocab_parallel_of(nets) is None else ShardedIdsValueStep
    value = nets["value_net"]
    cache = value.__dict__.setdefault("_recnn_ids_steps", {})
    dev = torch.device(device)
    key = (dev.type, dev.index)
    s = cache.get(key)
    if s is None or type(s) is not cls or s.pdims.num_items != nets["target_policy_net"].dims.num_items:
        s = cls(nets, dev)
        cache[key] = s
    return s
