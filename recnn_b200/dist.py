"""Data-parallel sharding of the update step across the GPUs of one node.

The path shards by sample row (SURVEY.md 8e): every rank holds a replica of the
embedding table, the nets and the optimizer state, processes its own rows, and
the ranks exchange exactly one thing -- the summed weight gradients (critic every
step, actor on policy steps) plus the loss scalars -- with an all-reduce before
the (identical) optimizer step.  Local loss terms are already scaled by
1/N_global on the device, so SUM over ranks gives the single-device gradient.

One process per GPU (torchrun).  torch.distributed supplies rendezvous, the weight broadcast and a
NCCL fallback; the per-step gradient exchange itself runs inside the step's CUDA graph as kernels that
read the peers' staging buffers over NVLink (``PeerComm`` -> ``recnn_comm_*`` in include/recnn_b200.h).
"""
from __future__ import annotations

import ctypes
import os
import warnings

import torch
import torch.distributed as dist

from . import _lib
from .nn.arena import param_arena


class PeerComm:
    """cudaIpc-mapped staging buffers of all ranks + the in-kernel all-reduce that uses them."""

    def __init__(self, group, device, capacity_floats):
        L = _lib.lib()
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.device = torch.device(device)
        self.capacity = -(-int(capacity_floats) // 4) * 4         # the library rounds the staging capacity up to 4
        self.handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _lib.check(L.recnn_comm_create(self.rank, self.world, int(capacity_floats), ctypes.byref(self.handle)))
            nbytes = L.recnn_comm_handle_bytes()
            mine = ctypes.create_string_buffer(nbytes)
            _lib.check(L.recnn_comm_local_handle(self.handle, mine))
            everyone = [None] * self.world
            dist.all_gather_object(everyone, bytes(mine.raw), group=group)
            status = L.recnn_comm_connect(self.handle, b"".join(everyone))
            # all ranks must agree, otherwise some would wait in a kernel for peers that use NCCL
            ok = [None] * self.world
            dist.all_gather_object(ok, int(status), group=group)
            if any(ok):
                msg = L.recnn_b200_last_error().decode() if status else "a peer could not map the staging buffers"
                L.recnn_comm_destroy(self.handle)
                self.handle = None
                raise _lib.RecnnError("peer-memory communicator unavailable: " + msg)

    @property
    def ptr(self):
        return self.handle.value

    def all_reduce(self, t: torch.Tensor):
        """In-place sum over the ranks (fp32, contiguous); same bits on every rank."""
        assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
        _lib.check(_lib.lib().recnn_comm_allreduce(self.handle, t.data_ptr(), t.numel(),
                                                   torch.cuda.current_stream(t.device).cuda_stream))
        return t

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        """[world * n]: every rank's n words of ``t`` in rank order, the same bits on every rank (fp32 or int32)."""
        assert t.is_cuda and t.dtype in (torch.float32, torch.int32) and t.is_contiguous()
        out = torch.empty(self.world * t.numel(), dtype=t.dtype, device=t.device)
        _lib.check(_lib.lib().recnn_comm_allgather(self.handle, t.data_ptr(), t.numel(), out.data_ptr(),
                                                   torch.cuda.current_stream(t.device).cuda_stream))
        return out

    def close(self):
        if self.handle is not None:
            _lib.lib().recnn_comm_destroy(self.handle)
            self.handle = None


def shard_rows(n_rows: int, rank: int, world: int):
    """Contiguous, balanced row range of this rank (first ``n_rows % world`` ranks get one more)."""
    base, extra = divmod(n_rows, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def broadcast_nets(nets: dict, group=None, src: int = 0):
    """Make every replica bit-identical to rank ``src`` (one broadcast per net arena)."""
    for name in sorted(nets):
        dist.broadcast(param_arena(nets[name]), src=src, group=group)


def enable_data_parallel(agent_or_nets, group=None, sync_weights=True):
    """Turn on gradient all-reduce for an Algo (or a nets dict).  Must be called on every
    rank after the nets are on their CUDA device."""
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    nets = agent_or_nets.nets if hasattr(agent_or_nets, "nets") else agent_or_nets
    world = dist.get_world_size(group)
    if sync_weights:
        broadcast_nets(nets, group)
    policy = nets["policy_net"]
    comm = None
    arena = param_arena(policy)
    if world > 1 and arena.is_cuda and os.environ.get("RECNN_B200_COMM", "peer") != "nccl":
        try:
            comm = PeerComm(group, arena.device, max(param_arena(m).numel() for m in nets.values()))
        except _lib.RecnnError as exc:     # e.g. no peer access between the GPUs: NCCL between the phases instead
            warnings.warn("recnn_b200: %s; falling back to NCCL all-reduces between the step's phases" % exc)
    policy.__dict__["_recnn_dp"] = (group, world, comm)
    for eng in policy.__dict__.get("_recnn_engines", {}).values():
        eng.group, eng.world, eng.comm = group, world, comm
        eng.graphs.clear()
        eng._fast.clear()
    return agent_or_nets


# ----------------------------------------------------------------------------------------------------------------------
# Vocabulary parallelism of the REINFORCE policy (DiscreteActor): rank r holds rows [lo_r, hi_r) of linear2 and their
# optimizer state; linear1 is replicated.  Every rank is fed the same saved rows.  A policy update exchanges a few
# floats per row and rank (all-gather) and the layer-1 gradient (all-reduce); see recnn_reinforce_shard_* in
# include/recnn_b200.h.
def vocab_shard(num_items: int, rank: int, world: int):
    """Contiguous item range [lo, hi) of ``rank``: blocks of ceil(num_items / world) items, the last one shorter.
    Raises ValueError when the rank's block would be empty."""
    per = -(-num_items // world)
    lo, hi = min(rank * per, num_items), min((rank + 1) * per, num_items)
    if hi <= lo:
        raise ValueError("%d items over %d ranks leave rank %d without items; use fewer ranks" % (num_items, world, rank))
    return lo, hi


def check_vocab_plans(plans):
    """``plans``: every rank's (lo, hi, num_items) in rank order.  Raises ValueError unless they tile [0, num_items)
    with non-empty, contiguous blocks and agree on num_items."""
    items = {p[2] for p in plans}
    if len(items) != 1:
        raise ValueError("the ranks disagree on the vocabulary size: %s" % sorted(items))
    expect = 0
    for r, (lo, hi, _) in enumerate(plans):
        if lo != expect or hi <= lo:
            raise ValueError("rank %d holds items [%d, %d), expected a non-empty block from %d" % (r, lo, hi, expect))
        expect = hi
    if expect != items.pop():
        raise ValueError("the shards end at item %d, not at the vocabulary size" % expect)


def layer1_floats(dims) -> int:
    """Floats of the layer-1 block (linear1 weight and bias) at the head of a DiscreteActor arena."""
    buf = (ctypes.c_int64 * 7)()
    _lib.check(_lib.lib().recnn_discrete_layout(dims, buf))
    return int(buf[2])


def vocab_comm_floats(dims, world: int, rows: int) -> int:
    """Staging capacity a sharded policy's communicator needs for ``rows`` saved rows: the layer-1 all-reduce, or the
    all-gather of ``world`` records of ``rows`` rows, whichever is larger."""
    return max(layer1_floats(dims), world * int(_lib.lib().recnn_vocab_record_floats(rows)))


class VocabParallel:
    """What ``enable_vocab_parallel`` records on a policy: its block [lo, hi) of the ``num_items`` items, the process
    group, rank, world size, and the peer communicator of the exchanges."""

    def __init__(self, lo, hi, num_items, group, rank, world, comm):
        self.lo, self.hi, self.num_items = lo, hi, num_items
        self.group, self.rank, self.world, self.comm = group, rank, world, comm

    def shard(self):
        return _lib.VocabShard(self.lo, self.num_items, self.rank, self.world)

    def _fit(self, need, device):
        """Grow the communicator (collectively: every rank asks for the same size) to ``need`` floats."""
        if need > self.comm.capacity:
            grown = PeerComm(self.group, device, max(need, 2 * self.comm.capacity))
            self.comm.close()
            self.comm = grown

    def all_gather(self, t: torch.Tensor) -> torch.Tensor:
        """PeerComm.all_gather; the communicator grows (collectively: every rank gathers the same size) when the
        records outgrow it."""
        self._fit(self.world * t.numel(), t.device)
        return self.comm.all_gather(t)

    def all_reduce(self, t: torch.Tensor) -> torch.Tensor:
        """PeerComm.all_reduce (in place, the same bits on every rank); the communicator grows as for all_gather."""
        self._fit(t.numel(), t.device)
        return self.comm.all_reduce(t)

    def __deepcopy__(self, memo):
        # a copied net (a target net) shares the online net's plan and communicator: there is one peer mapping per
        # process group, and every net of an agent exchanges over it in the same order on every rank
        return self


def _shard_policy_rows(policy, lo, hi):
    from .nn.arena import grad_arena
    with torch.no_grad():
        for p in (policy.linear2.weight, policy.linear2.bias):
            p.grad = None
            p.data = p.data[lo:hi].clone()
    policy.linear2.out_features = hi - lo
    policy.__dict__.pop("_recnn_engines", None)
    grad_arena(policy)                                  # the local arenas (param_arena rebuilds on the new shapes)


def _shard_critic_columns(critic, lo, hi):
    """Keep the state block of linear1 and the action columns [lo, hi): a Critic(S, hi - lo, H)."""
    from .nn.arena import grad_arena
    S = critic.linear1.in_features - critic._action_dim
    with torch.no_grad():
        w = critic.linear1.weight
        w.grad = None
        w.data = torch.cat([w.data[:, :S], w.data[:, S + lo:S + hi]], 1).contiguous()
        critic.linear1.bias.grad = None
    critic.linear1.in_features = S + hi - lo
    critic._action_dim = hi - lo
    critic.__dict__.pop("_recnn_ids_steps", None)
    critic.__dict__.pop("_recnn_engines", None)
    grad_arena(critic)


_AGENT_NETS = ("policy_net", "target_policy_net", "value_net", "target_value_net")


def _critic_shape_error(name, net, S, num_items):
    from .nn.arena import _is_discrete
    if (_is_discrete(net) or not hasattr(net, "_action_dim") or net.linear3.out_features != 1
            or net._action_dim != num_items or net.linear1.in_features != S + num_items):
        return ("nets[%r] must be a Critic(%d, %d, H) (state_dim and num_items of the policy) to be sharded with it"
                % (name, S, num_items))
    return None


def _optimizer_state_error(key, opt):
    """Why ``opt`` cannot be carried to the local arenas, or None: its moments would have the unsharded shapes."""
    from . import optim as _optim
    if isinstance(opt, _optim._ArenaOptimizer):
        if opt._t is not None:
            return "%s has already stepped; enable vocabulary parallelism before the first update" % key
    elif len(getattr(opt, "state", {})) != 0:
        return "%s already holds state; enable vocabulary parallelism before the first update" % key
    return None


def _rebuild_optimizers(optimizers, nets):
    """The agent's optimizers on the local arenas: built-in arena optimizers are rebuilt with the same hyperparameters
    (their state arenas take the local geometry); torch optimizers keep their Parameter objects, which now hold the
    local blocks.  Optimizers that already hold state are refused (their moments have the unsharded shapes)."""
    from . import optim as _optim
    owner = {id(p): name for name, net in nets.items() for p in net.parameters()}
    for key, opt in list(optimizers.items()):
        if opt is None:
            continue
        err = _optimizer_state_error("optimizers[%r]" % key, opt)
        if err:
            raise RuntimeError(err)
        if isinstance(opt, _optim._ArenaOptimizer):
            group = opt.param_groups[0]
            net = nets.get(owner.get(id(group["params"][0])))
            fresh = type(opt)(group["params"], **{k: group[k] for k in opt.defaults})
            if net is not None:
                fresh.bind(net)
            optimizers[key] = fresh


def _beta_refusal(beta, S, num_items):
    """Why ``beta`` cannot be sharded with a policy of state_dim S over num_items items, or None (checked on every rank
    before any exchange)."""
    from .nn.arena import _is_beta
    if not _is_beta(beta):
        return TypeError("beta must be a recnn_b200.nn.Beta (got %s)" % type(beta).__name__)
    if "_recnn_vp" in beta.__dict__:
        return RuntimeError("beta is already vocabulary-parallel")
    lin = beta.net[0]
    if (lin.in_features, lin.out_features) != (S, num_items):
        return ValueError("beta must be a Beta(%d, %d) (state_dim and num_items of the policy) to be sharded with it; "
                          "got Beta(%d, %d)" % (S, num_items, lin.in_features, lin.out_features))
    err = _optimizer_state_error("beta.optim", beta.optim)
    return None if err is None else RuntimeError(err)


def _shard_beta_rows(beta, lo, hi):
    """Keep rows [lo, hi) of net.0 (weight and bias) and rebuild the built-in optimizer on the local arenas."""
    from . import optim as _optim
    from .nn.arena import grad_arena
    lin = beta.net[0]
    with torch.no_grad():
        for p in (lin.weight, lin.bias):
            p.grad = None
            p.data = p.data[lo:hi].clone()
    lin.out_features = hi - lo
    beta._workspace = None
    grad_arena(beta)
    opt = beta.optim
    if isinstance(opt, _optim._ArenaOptimizer):
        # not bound: the Beta holds its optimizer (see Beta.forward)
        beta.optim = type(opt)(opt.param_groups[0]["params"], **{k: opt.param_groups[0][k] for k in opt.defaults})


def enable_vocab_parallel(policy_or_agent, group=None, beta=None):
    """Shard a DiscreteActor's item layer -- or a whole REINFORCE agent -- over the ranks of ``group``.  Call it on
    every rank after the nets are on their CUDA device.  The weights are first made identical to rank 0's.  At world 1
    everything computes exactly what it did unsharded.

    A DiscreteActor: rank r keeps rows vocab_shard(num_items, r, world) of linear2 (so ``state_dict`` holds the local
    block); call it before the policy's optimizer is built.  On a sharded policy, ``forward`` / ``select_action``
    return the rank's COLUMN BLOCK [N, hi - lo] of the softmax over all items (the reference returns [N, num_items]);
    sampled ids, log-probs, ``saved_log_probs``, ``correction`` and ``lambda_k`` are global and identical on every rank.
    ``ChooseREINFORCE`` trains it.

    A ``Reinforce`` agent (or its nets dict with policy_net, target_policy_net, value_net and target_value_net): both
    policies are sharded as above and both critics, which must be Critic(S, num_items, H) for the policy's S and
    num_items, keep linear1's state block and the action columns [lo, hi) of the same plan: their ``state_dict`` holds
    the local action block.  The four nets share one ``VocabParallel`` (and so one communicator).  An agent's optimizers
    are rebuilt on the local arenas with the same hyperparameters (a nets dict's optimizers are the caller's: build them
    afterwards).  ``value_update`` / ``reinforce_update`` / ``Reinforce.update()`` then run vocabulary-parallel on
    item-id batch actions (recnn_discrete_value_shard_* in include/recnn_b200.h); a dense [N, num_items] action is
    refused.  ``debug["next_action"]`` (learn=False) is the rank's column block.

    ``beta``: the Top-K notebook's behaviour policy (an ``nn.Beta`` of the policy's state_dim and num_items, on its
    device, whose optimizer has not stepped), sharded in the same call over the policy's plan and sharing its
    ``VocabParallel``.  Rank r keeps rows [lo, hi) of ``net.0`` (its ``state_dict`` holds the local block) and its
    built-in RAdam is rebuilt on the local arenas with the same hyperparameters.  ``beta(state, action)`` then returns
    the rank's column block [N, hi - lo] of the probabilities (recnn_beta_shard_* in include/recnn_b200.h), and
    ``DiscreteActor.pi_beta_sample`` draws from that block over the whole vocabulary.

    Every rank must be fed the same batches and states, seeded the same (torch.manual_seed, or the same
    ``uniform_source``) and must make the same calls in the same order: dropout masks -- given in the batch or drawn --
    and the masks of reinforce_update's reward line must agree across ranks."""
    from .nn.arena import _is_discrete, _is_beta
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    agent = policy_or_agent if hasattr(policy_or_agent, "nets") else None
    if agent is not None or isinstance(policy_or_agent, dict):
        nets = agent.nets if agent is not None else policy_or_agent
        missing = [k for k in _AGENT_NETS if nets.get(k) is None]
        if missing:
            raise ValueError("a REINFORCE agent's nets need %s" % ", ".join(missing))
        policy = nets["policy_net"]
    else:
        nets, policy = None, policy_or_agent
    if _is_beta(policy) or not _is_discrete(policy):
        raise TypeError("enable_vocab_parallel shards a DiscreteActor")
    shard_nets = {"policy_net": policy} if nets is None else {k: nets[k] for k in _AGENT_NETS}
    for name, net in shard_nets.items():
        if "_recnn_vp" in net.__dict__:
            raise RuntimeError("the policy is already vocabulary-parallel" if nets is None
                               else "nets[%r] is already vocabulary-parallel" % name)
    S, num_items = policy.linear1.in_features, policy.linear2.out_features
    if nets is not None:
        # refused on this rank before any exchange; the shape exchange below makes every rank refuse together
        tp = nets["target_policy_net"]
        if (_is_beta(tp) or not _is_discrete(tp) or tp.linear2.weight.shape != policy.linear2.weight.shape
                or tp.linear1.weight.shape != policy.linear1.weight.shape):
            raise ValueError("nets['target_policy_net'] must be a DiscreteActor of the policy's shape")
        for name in ("value_net", "target_value_net"):
            err = _critic_shape_error(name, nets[name], S, num_items)
            if err:
                raise ValueError(err)
        if nets["target_value_net"].linear1.weight.shape != nets["value_net"].linear1.weight.shape:
            raise ValueError("nets['target_value_net'] and nets['value_net'] differ in shape")
    if beta is not None:
        err = _beta_refusal(beta, S, num_items)
        if err is not None:
            raise err
    arena = param_arena(policy)
    if not arena.is_cuda:
        raise _lib.RecnnError("enable_vocab_parallel needs the policy on its CUDA device")
    if nets is not None:
        for name, net in shard_nets.items():
            if param_arena(net).device != arena.device:
                raise _lib.RecnnError("nets[%r] is on %s, the policy on %s" % (name, param_arena(net).device,
                                                                               arena.device))
    if beta is not None and param_arena(beta).device != arena.device:
        raise ValueError("beta is on %s, the policy on %s" % (param_arena(beta).device, arena.device))
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    # every rank checks every rank's plan, so a refused plan raises on all of them (none is left in a collective)
    shape = (S, policy.linear1.out_features, num_items)
    if nets is not None:
        shape += (tuple(nets["value_net"].linear1.weight.shape),)
    if beta is not None:
        shape += (("beta",) + tuple(beta.net[0].weight.shape),)
    sizes = [None] * world
    dist.all_gather_object(sizes, shape, group=group)
    if len(set(sizes)) != 1:
        raise ValueError("the ranks' nets differ in shape: %s" % sizes)
    plans = [vocab_shard(num_items, r, world) + (num_items,) for r in range(world)]
    check_vocab_plans(plans)
    lo, hi, _ = plans[rank]
    broadcast_nets(shard_nets, group)
    for name, net in shard_nets.items():
        if name.endswith("policy_net"):
            _shard_policy_rows(net, lo, hi)
        else:
            _shard_critic_columns(net, lo, hi)
    comm = PeerComm(group, arena.device, vocab_comm_floats(policy.dims, world, 1))
    vp = VocabParallel(lo, hi, num_items, group, rank, world, comm)
    for net in shard_nets.values():
        net.__dict__["_recnn_vp"] = vp
    if beta is not None:
        from .nn import beta as _beta
        dist.broadcast(param_arena(beta), src=0, group=group)
        _shard_beta_rows(beta, lo, hi)
        beta.__dict__["_recnn_vp"] = vp
        _beta._SHARDED.add(beta)
    if agent is not None and getattr(agent, "optimizers", None):
        _rebuild_optimizers(agent.optimizers, nets)
    return policy_or_agent
