"""Data-parallel sharding of the update step across the GPUs of one node.

The path shards by sample row (SURVEY.md 8e): every rank holds a replica of the
embedding table, the nets and the optimizer state, processes its own rows, and
the ranks exchange exactly one thing -- the summed weight gradients (critic every
step, actor on policy steps) plus the loss scalars -- with an all-reduce before
the (identical) optimizer step.  Local loss terms are already scaled by
1/N_global on the device, so SUM over ranks gives the single-device gradient.

One process per GPU (torchrun).  torch.distributed supplies rendezvous and the weight broadcast; the
per-step gradient exchange itself runs inside the step's CUDA graph as kernels that read the peers'
staging buffers over NVLink (``PeerComm`` -> ``recnn_comm_*`` in include/recnn_b200.h), so the GPUs of
the node need peer access to each other.
"""
from __future__ import annotations

import ctypes

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
            # all ranks must agree: a rank that went on would wait in a kernel for peers that raise here
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


def enable_data_parallel(agent_or_nets, group=None, sync_weights=True, beta=None):
    """Turn on gradient all-reduce for an Algo (or a nets dict).  Must be called on every
    rank after the nets are on their CUDA device.  The all-reduce runs over a peer communicator
    (PeerComm), so the GPUs need peer access to each other; without it every rank raises RecnnError.

    With a DiscreteActor policy (REINFORCE) the agent trains row-parallel instead (RowParallel below): the nets -- and
    ``beta``, the Top-K behaviour policy -- are made identical to rank 0's, one peer communicator is built and
    data_parallel_in_place attaches the plan.  Each rank then feeds its own rows of every batch
    (``shard_rows(N, rank, world)``) with the same seed on every rank."""
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    nets = agent_or_nets.nets if hasattr(agent_or_nets, "nets") else agent_or_nets
    from .nn.arena import _is_beta, _is_discrete
    policy = nets.get("policy_net") if isinstance(nets, dict) else None
    if policy is not None and _is_discrete(policy) and not _is_beta(policy):
        return _enable_row_parallel(agent_or_nets, group, sync_weights, beta)
    if beta is not None:
        raise TypeError("beta goes with a DiscreteActor policy (REINFORCE); this agent's policy is %s"
                        % type(policy).__name__)
    world = dist.get_world_size(group)
    if sync_weights:
        broadcast_nets(nets, group)
    policy = nets["policy_net"]
    comm = None
    arena = param_arena(policy)
    if world > 1 and arena.is_cuda:
        comm = PeerComm(group, arena.device, max(param_arena(m).numel() for m in nets.values()))
    policy.__dict__["_recnn_dp"] = (group, world, comm)
    for eng in policy.__dict__.get("_recnn_engines", {}).values():
        eng.world, eng.comm = world, comm
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


class _Exchanges:
    """The exchanges of a plan over its communicator ``comm`` (a PeerComm, or a test's stand-in with the same two
    calls): the process group, rank and world size, and the collective growth of the staging buffers."""

    def __init__(self, group, rank, world, comm):
        self.group, self.rank, self.world, self.comm = group, rank, world, comm

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


class VocabParallel(_Exchanges):
    """What ``enable_vocab_parallel`` records on a policy: its block [lo, hi) of the ``num_items`` items, the process
    group, rank, world size, and the peer communicator of the exchanges."""

    def __init__(self, lo, hi, num_items, group, rank, world, comm):
        super().__init__(group, rank, world, comm)
        self.lo, self.hi, self.num_items = lo, hi, num_items

    def shard(self):
        return _lib.VocabShard(self.lo, self.num_items, self.rank, self.world)


class RowParallel(_Exchanges):
    """What ``enable_data_parallel`` records on the nets of a REINFORCE agent: every rank holds full replicas of the
    nets and of β and its own rows of each batch; the process group, rank, world size and the peer communicator of the
    row exchanges.  The data-parallel counterpart of VocabParallel."""

    def row_counts(self, n_local):
        """Every rank's row count, in rank order (one all-gather; a collective).  Raises ValueError on every rank when
        a rank has no rows."""
        dev = torch.device("cuda", torch.cuda.current_device())
        counts = self.all_gather(torch.tensor([int(n_local)], dtype=torch.int32, device=dev)).tolist()
        if min(counts) <= 0:
            raise ValueError("a data-parallel rank got no rows (rows per rank: %s): every rank needs at least one "
                             "row of each batch" % counts)
        return counts

    def rows(self, n_local):
        """(row_offset, n_rows_global) of this rank's ``n_local`` rows: the ranks' rows, in rank order, are the rows
        of the whole batch (uneven shards included).  A collective."""
        counts = self.row_counts(n_local)
        return sum(counts[:self.rank]), sum(counts)


def row_parallel_of(net):
    """The RowParallel attached to ``net`` by enable_data_parallel, or None."""
    return net.__dict__.get("_recnn_rows")


def _row_parallel_refusal(nets, beta, optimizers):
    """Why these nets (and β, and the agent's optimizers) cannot be made row-parallel, or None."""
    for name, net in list(nets.items()) + ([("beta", beta)] if beta is not None else []):
        label = name if name == "beta" else "nets[%r]" % name
        if "_recnn_vp" in net.__dict__:
            return RuntimeError("%s is vocabulary-parallel: data parallel and vocabulary parallel do not combine" % label)
        if "_recnn_rows" in net.__dict__:
            return RuntimeError("%s is already data-parallel" % label)
    opts = [("optimizers[%r]" % k, o) for k, o in sorted((optimizers or {}).items()) if o is not None]
    if beta is not None:
        opts.append(("beta.optim", beta.optim))
    for label, opt in opts:
        err = _optimizer_state_error(label, opt)
        if err:
            return RuntimeError(err.replace("vocabulary parallelism", "data parallelism"))
    return None


def data_parallel_in_place(nets, plan, beta=None, optimizers=None):
    """The local half of enable_data_parallel on a REINFORCE agent, with no exchange: attach the RowParallel ``plan``
    to ``nets`` ({name: net}: the policy, target policy and both critics) and to ``beta``.  The nets stay full replicas
    (their ``state_dict`` and checkpoints are the unsharded ones); they must hold identical weights on every rank.
    ``optimizers`` ({key: optimizer}) must not hold state yet.  The counterpart of shard_in_place."""
    err = _row_parallel_refusal(nets, beta, optimizers)
    if err is not None:
        raise err
    for net in nets.values():
        net.__dict__.pop("_recnn_engines", None)
        net.__dict__.pop("_recnn_ids_steps", None)
        net.__dict__["_recnn_rows"] = plan
    if beta is not None:
        beta.__dict__["_recnn_rows"] = plan


def _enable_row_parallel(agent_or_nets, group, sync_weights, beta):
    agent, nets = _vocab_nets(agent_or_nets, beta, "data parallel REINFORCE trains a DiscreteActor")
    optimizers = getattr(agent, "optimizers", None)
    err = _row_parallel_refusal(nets, beta, optimizers)
    arena = param_arena(nets["policy_net"])
    if err is None and not arena.is_cuda:
        err = _lib.RecnnError("enable_data_parallel needs the nets on their CUDA device")
    if err is None:
        for name, net in list(nets.items()) + ([("beta", beta)] if beta is not None else []):
            if param_arena(net).device != arena.device:
                err = _lib.RecnnError("%s is on %s, the policy on %s" % (name, param_arena(net).device, arena.device))
                break
    # every rank learns every rank's refusal, so a refused call raises on all of them before any device work
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    everyone = [None] * world
    dist.all_gather_object(everyone, None if err is None else (type(err).__name__, str(err)), group=group)
    bad = [(q, e) for q, e in enumerate(everyone) if e is not None]
    if err is not None:
        raise err
    if bad:
        raise RuntimeError("rank %d refuses data parallel: %s: %s" % (bad[0][0], bad[0][1][0], bad[0][1][1]))
    if sync_weights:
        broadcast_nets(nets, group)
        if beta is not None:
            dist.broadcast(param_arena(beta), src=0, group=group)
    sizes = [param_arena(m).numel() for m in nets.values()] + ([param_arena(beta).numel()] if beta is not None else [])
    comm = PeerComm(group, arena.device, max(sizes))
    data_parallel_in_place(nets, RowParallel(group, rank, world, comm), beta, optimizers)
    return agent_or_nets


def _item_axes(net):
    """Per parameter of ``net`` (arena order), the (axis, first) of its item coordinate -- item j sits at index
    first + j of that axis -- or None when the parameter is replicated over the ranks: rows of the policy's linear2
    and of β's net.0, the action columns of a critic's linear1 (after its S state columns)."""
    from .nn.arena import _is_beta, _is_discrete
    if _is_beta(net):
        return [(0, 0), (0, 0)]
    if _is_discrete(net):
        return [None, None, (0, 0), (0, 0)]
    return [(1, net.linear1.in_features - net._action_dim)] + [None] * 5


def _item_part(t, ax, lo, n):
    """Items [lo, lo + n) of ``t`` along its item axis ``ax`` (a view)."""
    return t.narrow(ax[0], ax[1] + lo, n)


def _shared_part(t, ax):
    """The replicated part of ``t`` (a view): all of it, the critic's state columns, or None."""
    if ax is None:
        return t
    return t.narrow(ax[0], 0, ax[1]) if ax[1] else None


def _block(t, ax, lo, hi):
    """What the rank holding items [lo, hi) keeps of the full tensor ``t``: a new contiguous tensor (``t`` itself when
    it is replicated)."""
    if ax is None:
        return t
    shared = _shared_part(t, ax)
    item = _item_part(t, ax, lo, hi - lo)
    return item.clone(memory_format=torch.contiguous_format) if shared is None else torch.cat([shared, item], ax[0])


def _shard_params(net, lo, hi):
    """Replace every sharded parameter of ``net`` by its block [lo, hi) (the module's features are the caller's)."""
    from .nn.arena import _params
    with torch.no_grad():
        for p, ax in zip(_params(net), _item_axes(net)):
            if ax is not None:
                p.grad = None
                p.data = _block(p.data, ax, lo, hi)


def _shard_policy_rows(policy, lo, hi):
    from .nn.arena import grad_arena
    _shard_params(policy, lo, hi)
    policy.linear2.out_features = hi - lo
    policy.__dict__.pop("_recnn_engines", None)
    grad_arena(policy)                                  # the local arenas (param_arena rebuilds on the new shapes)


def _shard_critic_columns(critic, lo, hi):
    """Keep the state block of linear1 and the action columns [lo, hi): a Critic(S, hi - lo, H)."""
    from .nn.arena import grad_arena
    S = critic.linear1.in_features - critic._action_dim
    _shard_params(critic, lo, hi)
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
    """Why the Beta ``beta`` cannot be sharded with a policy of state_dim S over num_items items, or None (checked on
    every rank before any exchange)."""
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
    _shard_params(beta, lo, hi)
    beta.net[0].out_features = hi - lo
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
    from .nn.arena import _is_beta, _is_discrete
    if not dist.is_initialized():
        raise RuntimeError("torch.distributed is not initialised")
    agent, nets = _vocab_nets(policy_or_agent, beta, "enable_vocab_parallel shards a DiscreteActor")
    lone = "value_net" not in nets
    policy = nets["policy_net"]
    for name, net in list(nets.items()) + ([("beta", beta)] if beta is not None else []):
        if "_recnn_rows" in net.__dict__:
            raise RuntimeError("%s is data-parallel: data parallel and vocabulary parallel do not combine"
                               % (name if name == "beta" else "nets[%r]" % name))
    for name, net in nets.items():
        if "_recnn_vp" in net.__dict__:
            raise RuntimeError("the policy is already vocabulary-parallel" if lone
                               else "nets[%r] is already vocabulary-parallel" % name)
    S, num_items = policy.linear1.in_features, policy.linear2.out_features
    if not lone:
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
    for name, net in nets.items():
        if param_arena(net).device != arena.device:
            raise _lib.RecnnError("nets[%r] is on %s, the policy on %s" % (name, param_arena(net).device,
                                                                           arena.device))
    if beta is not None and param_arena(beta).device != arena.device:
        raise ValueError("beta is on %s, the policy on %s" % (param_arena(beta).device, arena.device))
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    # every rank checks every rank's plan, so a refused plan raises on all of them (none is left in a collective)
    shape = (S, policy.linear1.out_features, num_items)
    if not lone:
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
    # the communicator first: a peer mapping that fails leaves the nets as they were (its size is the layer-1 block's,
    # which sharding does not change)
    comm = PeerComm(group, arena.device, vocab_comm_floats(policy.dims, world, 1))
    broadcast_nets(nets, group)
    if beta is not None:
        dist.broadcast(param_arena(beta), src=0, group=group)
    shard_in_place(nets, VocabParallel(lo, hi, num_items, group, rank, world, comm), beta,
                   getattr(agent, "optimizers", None))
    return policy_or_agent


def _vocab_nets(policy_or_agent, beta, refusal):
    """(the agent or None, {name: net}) of what enable_vocab_parallel and the checkpoint functions take: a lone
    DiscreteActor as "policy_net", or an agent's (or nets dict's) policy_net, target_policy_net, value_net and
    target_value_net.  Raises ValueError when an agent lacks one of them, TypeError(``refusal``) when the policy is not
    a DiscreteActor, TypeError when ``beta`` is given and is not a Beta."""
    from .nn.arena import _is_beta, _is_discrete
    agent = policy_or_agent if hasattr(policy_or_agent, "nets") else None
    if agent is not None or isinstance(policy_or_agent, dict):
        src = agent.nets if agent is not None else policy_or_agent
        missing = [k for k in _AGENT_NETS if src.get(k) is None]
        if missing:
            raise ValueError("a REINFORCE agent's nets need %s" % ", ".join(missing))
        nets = {k: src[k] for k in _AGENT_NETS}
    else:
        nets = {"policy_net": policy_or_agent}
    if _is_beta(nets["policy_net"]) or not _is_discrete(nets["policy_net"]):
        raise TypeError(refusal)
    if beta is not None and not _is_beta(beta):
        raise TypeError("beta must be a recnn_b200.nn.Beta (got %s)" % type(beta).__name__)
    return agent, nets


def shard_in_place(nets, vp, beta=None, optimizers=None):
    """The local half of enable_vocab_parallel, with no exchange: shard ``nets`` ({name: net}: DiscreteActors under
    names ending in "policy_net", Critic(S, num_items, H)s otherwise) and ``beta`` to the block [vp.lo, vp.hi) of the
    VocabParallel ``vp`` and record ``vp`` on each.  ``optimizers`` ({key: optimizer} of those nets, or None): built-in
    ones are rebuilt on the local arenas (see enable_vocab_parallel).  The nets must hold full, identical weights on
    every rank."""
    for name, net in nets.items():
        if name.endswith("policy_net"):
            _shard_policy_rows(net, vp.lo, vp.hi)
        else:
            _shard_critic_columns(net, vp.lo, vp.hi)
        net.__dict__["_recnn_vp"] = vp
    if beta is not None:
        from .nn import beta as _beta
        _shard_beta_rows(beta, vp.lo, vp.hi)
        beta.__dict__["_recnn_vp"] = vp
        _beta._SHARDED.add(beta)
    if optimizers:
        _rebuild_optimizers(optimizers, nets)


# ----------------------------------------------------------------------------------------------------------------------
# Full checkpoints of vocabulary-parallel nets.  A sharded net's arenas hold the rank's block; a checkpoint holds what
# the unsharded net would: the reference's state_dict keys and shapes, and the built-in optimizers' arenas in the full
# arena's geometry.  Every tensor is converted per parameter (arena._views on the local and on the full geometry),
# since the critic's layer-1 pitch is pad4(S + hi - lo) locally and pad4(S + num_items) in full.  Each tensor has a
# replicated part (taken from one rank) and an item part (rank r's items [lo_r, hi_r)), moved in row slices of at most
# _SLICE_FLOATS floats, so no device holds more than its arenas and one slice beyond them.
_SLICE_FLOATS = (256 << 20) // 4


def _slices(t):
    """Views of ``t`` over consecutive ranges of its first axis, at most _SLICE_FLOATS elements each (one row at
    least)."""
    rows = t.shape[0]
    per = max(1, _SLICE_FLOATS // max(1, t[0].numel() if rows else 1))
    for r in range(0, rows, per):
        yield t.narrow(0, r, min(per, rows - r))


def _copy_sliced(dst, src):
    """``dst.copy_(src)`` one slice at a time: a copy between host and device stages at most one slice."""
    for d, s in zip(_slices(dst), _slices(src)):
        d.copy_(s)


class _Leaf:
    """One tensor of a checkpoint: the rank's local tensor, the full tensor (on the gathering rank; None elsewhere) and
    the item axis of its parameter (None: replicated)."""
    __slots__ = ("local", "full", "ax")

    def __init__(self, local, full, ax):
        self.local, self.full, self.ax = local, full, ax


def _outbox(leaves, n):
    """Sender half: the rank's item parts (``n`` = hi - lo items) as contiguous slices, in leaf order."""
    for leaf in leaves:
        if leaf.ax is not None:
            for s in _slices(_item_part(leaf.local, leaf.ax, 0, n)):
                yield s.contiguous()


def _inbox(leaves, lo, hi):
    """Receiver half: the full tensors' views rank [lo, hi)'s slices land in, in _outbox's order and shapes."""
    for leaf in leaves:
        if leaf.ax is not None:
            yield from _slices(_item_part(leaf.full, leaf.ax, lo, hi - lo))


def _copy_shared(leaves):
    """The gathering rank's replicated parts into the full tensors."""
    for leaf in leaves:
        shared = _shared_part(leaf.local, leaf.ax)
        if shared is not None:
            _copy_sliced(_shared_part(leaf.full, leaf.ax), shared)


def _load_leaves(locals_, fulls, axes, lo, hi):
    """Full -> local: each local tensor takes its replicated part whole and items [lo, hi) of the full tensor."""
    for local, full, ax in zip(locals_, fulls, axes):
        shared = _shared_part(local, ax)
        if shared is not None:
            _copy_sliced(shared, _shared_part(full, ax))
        if ax is not None:
            _copy_sliced(_item_part(local, ax, 0, hi - lo), _item_part(full, ax, lo, hi - lo))


def _full_twin(net, num_items):
    """A parameter-less (meta) net of ``net``'s class with all ``num_items`` items: the full geometry."""
    from .nn.arena import _is_beta, _is_discrete
    from .nn import models
    from .nn.beta import Beta
    with torch.device("meta"):
        if _is_beta(net):
            return Beta(net.net[0].in_features, num_items)
        if _is_discrete(net):
            return models.DiscreteActor(net.linear1.in_features, num_items, net.linear1.out_features)
        return models.Critic(net.linear1.in_features - net._action_dim, num_items, net.linear1.out_features)


def _checkpoint_parts(agent_or_policy, beta):
    """({name: net} of every sharded net, β included as "beta", {key: optimizer} of an agent or None, VocabParallel).
    Raises unless every net is vocabulary-parallel on the policy's plan."""
    agent, nets = _vocab_nets(agent_or_policy, beta,
                              "a vocabulary-parallel checkpoint is of a DiscreteActor or a REINFORCE agent")
    if beta is not None:
        nets["beta"] = beta
    vp = nets["policy_net"].__dict__.get("_recnn_vp")
    for name, net in nets.items():
        if vp is None or net.__dict__.get("_recnn_vp") is not vp:
            raise RuntimeError("%s is not vocabulary-parallel with the policy: call enable_vocab_parallel first"
                               % (name if name == "beta" else "nets[%r]" % name))
    optimizers = None
    if agent is not None:
        optimizers = {k: o for k, o in (getattr(agent, "optimizers", None) or {}).items() if o is not None}
    return nets, optimizers, vp


def _owners(nets):
    """{id(parameter): (net name, index in the arena order)}."""
    from .nn.arena import _params
    return {id(p): (name, i) for name, net in nets.items() for i, p in enumerate(_params(net))}


def _opt_params(opt):
    return [p for g in opt.param_groups for p in g["params"]]


def _arena_owner(opt, owners, label):
    """The net name whose whole arena a built-in optimizer steps."""
    name = owners.get(id(opt.param_groups[0]["params"][0]), (None,))[0]
    if name is None:
        raise ValueError("%s does not step one of the nets" % label)
    return name


def _scalar(v):
    return float(v) if torch.is_tensor(v) and v.numel() == 1 else (repr(v) if torch.is_tensor(v) else v)


def _gather_begin(nets, optimizers, num_items, gathering):
    """Every rank: the checkpoint's leaves in one order (local tensors; full host tensors on the gathering rank), the
    scalar state the ranks must agree on, and the checkpoint that the transport fills (None on the other ranks)."""
    from collections import OrderedDict
    from . import optim as _optim
    from .nn.arena import _params, _views, net_layout, param_arena
    twins = {name: _full_twin(net, num_items) for name, net in nets.items()}
    owners = _owners(nets)
    leaves, agree = [], []

    def arena(name, flat):
        net, twin = nets[name], twins[name]
        full = torch.zeros(net_layout(twin)[2], dtype=torch.float32) if gathering else None
        fulls = _views(full, twin) if gathering else [None] * len(_params(net))
        leaves.extend(_Leaf(l, f, ax) for l, f, ax in zip(_views(flat, net), fulls, _item_axes(net)))
        return full

    def net_state(name):
        full = arena(name, param_arena(nets[name]))
        if gathering:
            keys = [k for k, _ in twins[name].named_parameters()]
            return OrderedDict(zip(keys, _views(full, twins[name])))

    def opt_state(label, opt):
        if isinstance(opt, _optim._ArenaOptimizer):
            name = _arena_owner(opt, owners, label)
            sd = torch.optim.Optimizer.state_dict(opt) if gathering else None
            t = None if opt._t is None else int(opt._t.item())
            agree.append((label, "t", t))
            if t is not None:
                arenas = {k: None if getattr(opt, "_" + k) is None else arena(name, getattr(opt, "_" + k))
                          for k in ("m", "v", "slow")}
                if gathering:
                    sd["recnn_arenas"] = dict(arenas, t=t)
            return sd
        sd = opt.state_dict()
        params = _opt_params(opt)
        state = {}
        for idx in sorted(sd["state"]):
            if id(params[idx]) not in owners:
                raise ValueError("%s steps a parameter outside the nets" % label)
            name, i = owners[id(params[idx])]
            ax, full_shape = _item_axes(nets[name])[i], _params(twins[name])[i].shape
            entry = {}
            for k, v in sd["state"][idx].items():
                if torch.is_tensor(v) and v.dim() > 0 and v.shape == params[idx].shape:
                    entry[k] = torch.zeros(full_shape, dtype=v.dtype) if gathering else None
                    leaves.append(_Leaf(v.detach(), entry[k], ax))
                    agree.append((label, idx, k, "block"))
                else:
                    entry[k] = v.detach().cpu().clone() if torch.is_tensor(v) else v
                    agree.append((label, idx, k, _scalar(v)))
            state[idx] = entry
        return {"state": state, "param_groups": sd["param_groups"]} if gathering else None

    out = {"nets": {name: net_state(name) for name in nets if name != "beta"}}
    if optimizers is not None:
        out["optimizers"] = {k: opt_state("optimizers[%r]" % k, optimizers[k]) for k in sorted(optimizers)}
    if "beta" in nets:
        out["beta"] = {"net": net_state("beta"), "optim": opt_state("beta.optim", nets["beta"].optim)}
    return leaves, agree, (out if gathering else None)


def gather_vocab_parallel_state(agent_or_policy, beta=None, dst=0):
    """The full checkpoint of a vocabulary-parallel DiscreteActor or REINFORCE agent (and ``beta``), on rank ``dst``
    of the policy's group; None on the other ranks.  A collective: call it on every rank.

    The checkpoint is what the unsharded nets would give, in host memory (CPU tensors)::

        {"nets": {name: net.state_dict()}, "optimizers": {key: opt.state_dict()},
         "beta": {"net": beta.state_dict(), "optim": beta.optim.state_dict()}}

    with only the parts passed in (a lone policy is ``nets["policy_net"]``; "optimizers" comes with an agent).  Net
    keys and shapes are the reference's.  Built-in optimizers' ``recnn_arenas`` have the full arena's geometry (pads
    zero); a torch optimizer's per-parameter state (``exp_avg``, ...) is gathered along the item axis.  Replicated
    parameters and their state are rank ``dst``'s.  The ranks must hold the same step counts and scalar optimizer
    state, else every rank raises RuntimeError.  Take it after a policy update: rows saved for the next one (``_saved``,
    rewards) are not part of it, nor are the agent's step and the policy's draw counter, as for the unsharded
    ``state_dict``.  The item blocks travel by point-to-point sends in slices of at most 256 MB."""
    nets, optimizers, vp = _checkpoint_parts(agent_or_policy, beta)
    if not 0 <= dst < vp.world:
        raise ValueError("dst %d is not a rank of the policy's group of %d" % (dst, vp.world))
    gathering = vp.rank == dst
    leaves, agree, out = _gather_begin(nets, optimizers, vp.num_items, gathering)
    everyone = [None] * vp.world
    dist.all_gather_object(everyone, agree, group=vp.group)
    if any(a != everyone[0] for a in everyone):
        bad = next(q for q, a in enumerate(everyone) if a != everyone[0])
        raise RuntimeError("the ranks' optimizer states disagree (step counts or scalar state): rank 0 holds %s, rank "
                           "%d holds %s" % (everyone[0], bad, everyone[bad]))
    if gathering:
        _copy_shared(leaves)
    # each slice is released before the next one is made, one slice on the device at a time (not zip: its reused
    # result tuple would hold the previous slice while the next one is made)
    for q in range(vp.world):
        if q == vp.rank == dst:
            mine = _outbox(leaves, vp.hi - vp.lo)
            for v in _inbox(leaves, vp.lo, vp.hi):
                v.copy_(next(mine))
        elif q == vp.rank:
            for s in _outbox(leaves, vp.hi - vp.lo):
                dist.send(s, group=vp.group, group_dst=dst)
                if s.is_cuda:
                    torch.cuda.current_stream(s.device).synchronize()
                del s
        elif gathering:
            lo, hi = vocab_shard(vp.num_items, q, vp.world)
            dev = leaves[0].local.device
            for v in _inbox(leaves, lo, hi):
                buf = torch.empty(v.shape, dtype=v.dtype, device=dev)
                dist.recv(buf, group=vp.group, group_src=q)
                v.copy_(buf)
                del buf
    return out


def _load_refusal(nets, optimizers, state, num_items):
    """Why ``state`` cannot be loaded into these nets and optimizers, or None."""
    from . import optim as _optim
    from .nn.arena import net_layout
    if not isinstance(state, dict) or not isinstance(state.get("nets"), dict):
        return "the checkpoint has no 'nets' dict"
    sections = {name: (("beta", "net") if name == "beta" else ("nets", name)) for name in nets}
    twins = {name: _full_twin(net, num_items) for name, net in nets.items()}
    owners = _owners(nets)

    def entry(path):
        d = state
        for k in path:
            if not isinstance(d, dict) or d.get(k) is None:
                return None
            d = d[k]
        return d

    for name in nets:
        sd = entry(sections[name])
        if sd is None:
            return "the checkpoint has no state[%s]" % "][".join(map(repr, sections[name]))
        for k, p in twins[name].named_parameters():
            if not torch.is_tensor(sd.get(k)) or tuple(sd[k].shape) != tuple(p.shape):
                return ("state[%s][%r] is %s; the nets need %s (their state_dim, hidden size and num_items)"
                        % ("][".join(map(repr, sections[name])), k,
                           tuple(sd[k].shape) if torch.is_tensor(sd.get(k)) else "missing", tuple(p.shape)))
    opts = [(("optimizers", k), v) for k, v in sorted((optimizers or {}).items())]
    if "beta" in nets:
        opts.append((("beta", "optim"), nets["beta"].optim))
    for path, opt in opts:
        label = "state[%s]" % "][".join(map(repr, path))
        sd = entry(path)
        if sd is None:
            return "the checkpoint has no %s" % label
        groups = sd.get("param_groups")
        if (not isinstance(groups, list) or len(groups) != len(opt.param_groups)
                or any(len(g["params"]) != len(o["params"]) for g, o in zip(groups, opt.param_groups))):
            return "%s has other parameter groups than the optimizer" % label
        arenas = sd.get("recnn_arenas")
        if isinstance(opt, _optim._ArenaOptimizer):
            if sd.get("state"):
                return "%s is a torch optimizer's state; the optimizer is a built-in %s" % (label, type(opt).__name__)
            if arenas is None:
                continue
            name = _arena_owner(opt, owners, label)
            need = {"m": True, "v": opt._recnn_kind in (_lib.OPT_ADAM, _lib.OPT_RANGER, _lib.OPT_RADAM),
                    "slow": opt._recnn_kind == _lib.OPT_RANGER}
            have = {k: arenas.get(k) is not None for k in need}
            if have != need:
                return ("%s holds the arenas %s, a %s needs %s" % (label, sorted(k for k in have if have[k]),
                                                                   type(opt).__name__,
                                                                   sorted(k for k in need if need[k])))
            count = net_layout(twins[name])[2]
            for k in need:
                if need[k] and arenas[k].numel() != count:
                    return "%s['recnn_arenas'][%r] has %d floats, the full arena %d" % (label, k, arenas[k].numel(),
                                                                                         count)
            if not isinstance(arenas.get("t"), int):
                return "%s['recnn_arenas'] has no step count" % label
        else:
            if arenas is not None:
                return "%s holds a built-in optimizer's arenas; the optimizer is a %s" % (label, type(opt).__name__)
            params = _opt_params(opt)
            for idx, st in (sd.get("state") or {}).items():
                if not isinstance(idx, int) or not 0 <= idx < len(params) or id(params[idx]) not in owners:
                    return "%s has state for parameter %r, which the optimizer does not step" % (label, idx)
                name, i = owners[id(params[idx])]
                full = tuple(list(twins[name].parameters())[i].shape)
                for k, v in st.items():
                    if torch.is_tensor(v) and v.dim() > 0 and tuple(v.shape) != full:
                        return "%s['state'][%d][%r] is %s; the parameter is %s" % (label, idx, k, tuple(v.shape),
                                                                                  full)
    return None


def load_vocab_parallel_state(agent_or_policy, state, beta=None):
    """Load a full checkpoint -- from gather_vocab_parallel_state, or an unsharded agent's own ``state_dict()``s in the
    same layout -- into a vocabulary-parallel DiscreteActor or REINFORCE agent (and ``beta``), at any world size.  Call
    it on every rank after enable_vocab_parallel, each with the whole ``state``.  Each rank takes its block [lo, hi) of
    every sharded tensor and the replicated parts whole; built-in optimizers get their arenas in the local geometry and
    their step count, torch optimizers their per-parameter state sliced the same way.  A checkpoint whose nets'
    state_dim, hidden size or num_items differ from these nets', that lacks a net or an optimizer, or whose optimizer
    state is of another kind (Ranger arenas into an Adam, a torch optimizer's state into a built-in one, ...) is refused
    on every rank (ValueError) before anything is loaded."""
    from . import optim as _optim
    from .nn.arena import _params, _views, param_arena
    nets, optimizers, vp = _checkpoint_parts(agent_or_policy, beta)
    err = _load_refusal(nets, optimizers, state, vp.num_items)
    everyone = [None] * vp.world
    dist.all_gather_object(everyone, err, group=vp.group)
    bad = [(q, e) for q, e in enumerate(everyone) if e]
    if bad:
        raise ValueError("rank %d refuses the checkpoint: %s" % bad[0])
    lo, hi = vp.lo, vp.hi
    twins = {name: _full_twin(net, vp.num_items) for name, net in nets.items()}
    owners = _owners(nets)
    with torch.no_grad():
        for name, net in nets.items():
            sd = state["beta"]["net"] if name == "beta" else state["nets"][name]
            fulls = [sd[k] for k, _ in twins[name].named_parameters()]
            _load_leaves(_views(param_arena(net), net), fulls, _item_axes(net), lo, hi)
        opts = [(optimizers[k], state["optimizers"][k]) for k in sorted(optimizers or {})]
        if "beta" in nets:
            opts.append((nets["beta"].optim, state["beta"]["optim"]))
        for opt, sd in opts:
            if isinstance(opt, _optim._ArenaOptimizer):
                arenas = sd.get("recnn_arenas")
                opt.load_state_dict({k: v for k, v in sd.items() if k != "recnn_arenas"})
                if arenas is None:
                    continue
                name = _arena_owner(opt, owners, "")
                net = nets[name]
                opt._state_arenas(param_arena(net))
                for k in ("m", "v", "slow"):
                    local = getattr(opt, "_" + k)
                    if local is not None:
                        _load_leaves(_views(local, net), _views(arenas[k], twins[name]), _item_axes(net), lo, hi)
                opt._t.fill_(int(arenas["t"]))
                continue
            params = _opt_params(opt)
            local = {}
            for idx, st in sd["state"].items():
                name, i = owners[id(params[idx])]
                ax = _item_axes(nets[name])[i]
                local[idx] = {k: _block(v, ax, lo, hi) if torch.is_tensor(v) and v.dim() > 0 else v
                              for k, v in st.items()}
            opt.load_state_dict({"state": local, "param_groups": sd["param_groups"]})
    return agent_or_policy
