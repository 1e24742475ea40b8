"""Full checkpoints of vocabulary-parallel nets without a GPU: a random full agent state (policy, target policy, both
critics, β, every optimizer kind) sliced into W local states by the load path and put back together by the two halves
of the gather's transport, bit for bit; and the refusals of gather_vocab_parallel_state / load_vocab_parallel_state on
a world-1 gloo group.  A local net here is a net of the local geometry marked with its rank's VocabParallel, which is
what enable_vocab_parallel leaves on the device."""
from __future__ import annotations

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import dist as D
from recnn_b200.nn.arena import _views, param_arena
from tests._ranks import one_rank_cpu_group  # noqa: F401

S, H, ITEMS = 13, 10, 1003          # S % 4 != 0 and H % 4 != 0: every pitch pads; 1003 is not divisible by 2, 3 or 8
KINDS = ["sgd", "adam", "ranger", "radam", "torch_adam"]


def _optimizer(kind, net):
    ps = net.parameters()
    return {"sgd": lambda: recnn_b200.optim.SGD(ps, lr=0.1, momentum=0.9),
            "adam": lambda: recnn_b200.optim.Adam(ps, lr=1e-3),
            "ranger": lambda: recnn_b200.optim.Ranger(ps, lr=1e-5, weight_decay=1e-2),
            "radam": lambda: recnn_b200.optim.RAdam(ps, lr=1e-5, weight_decay=1e-5),
            "torch_adam": lambda: torch.optim.Adam(ps, lr=1e-3)}[kind]()


def _agent(kind, items, beta_kind=None):
    agent = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, items, H), recnn_b200.nn.Critic(S, items, H))
    agent.optimizers = {"policy_optimizer": _optimizer(kind, agent.nets["policy_net"]),
                        "value_optimizer": _optimizer(kind, agent.nets["value_net"])}
    beta = recnn_b200.nn.Beta(S, items)
    beta.optim = _optimizer(beta_kind or kind, beta)
    return agent, beta


def _randomize(agent, beta, seed):
    """Random weights and optimizer state; arena pads stay zero."""
    g = torch.Generator().manual_seed(seed)
    owners = {"policy_optimizer": "policy_net", "value_optimizer": "value_net"}
    with torch.no_grad():
        for net in list(agent.nets.values()) + [beta]:
            for v in _views(param_arena(net), net):
                v.copy_(torch.randn(v.shape, generator=g))
        for opt, net in [(o, agent.nets[owners[k]]) for k, o in agent.optimizers.items()] + [(beta.optim, beta)]:
            if isinstance(opt, recnn_b200.optim._ArenaOptimizer):
                opt._state_arenas(param_arena(net))
                for a in (opt._m, opt._v, opt._slow):
                    if a is not None:
                        for v in _views(a, net):
                            v.copy_(torch.randn(v.shape, generator=g))
                opt._t.fill_(7)
            else:
                for p in net.parameters():
                    p.grad = torch.randn(p.shape, generator=g)
                opt.step()
                for st in opt.state.values():
                    for k in ("exp_avg", "exp_avg_sq"):
                        st[k].copy_(torch.randn(st[k].shape, generator=g).abs())


def _full_state(agent, beta):
    return {"nets": {k: v.state_dict() for k, v in agent.nets.items()},
            "optimizers": {k: v.state_dict() for k, v in agent.optimizers.items()},
            "beta": {"net": beta.state_dict(), "optim": beta.optim.state_dict()}}


def _local(kind, lo, hi, rank, world):
    agent, beta = _agent(kind, ITEMS)
    D.shard_in_place(agent.nets, D.VocabParallel(lo, hi, ITEMS, None, rank, world, None), beta, agent.optimizers)
    return agent, beta


def _same(a, b, where=""):
    """Bit-identical nested checkpoints (tensors by value and dtype, on any device)."""
    if torch.is_tensor(a):
        assert torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape, where
        assert torch.equal(a.detach().cpu().contiguous().view(torch.int32) if a.dtype == torch.float32 else a.cpu(),
                           b.detach().cpu().contiguous().view(torch.int32) if b.dtype == torch.float32 else b.cpu()), where
    elif isinstance(a, dict):
        assert isinstance(b, dict) and set(a) == set(b), (where, sorted(a), sorted(b))
        for k in a:
            _same(a[k], b[k], "%s/%s" % (where, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s/%d" % (where, i))
    else:
        assert a == b, (where, a, b)


def _pads_zero(flat, net):
    rest = flat.clone()
    for v in _views(rest, net):
        v.zero_()
    return not bool(rest.any())


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("kind", KINDS)
def test_virtual_ranks_full_to_local_to_full(one_rank_cpu_group, monkeypatch, world, kind):
    monkeypatch.setattr(D, "_SLICE_FLOATS", 1000)          # several slices per block
    agent, beta = _agent(kind, ITEMS)
    _randomize(agent, beta, world)
    full = _full_state(agent, beta)
    ranks = []
    for r in range(world):
        lo, hi = D.vocab_shard(ITEMS, r, world)
        la, lb = _local(kind, lo, hi, r, world)
        D.load_vocab_parallel_state(la, full, beta=lb)
        for name, net in list(la.nets.items()) + [("beta", lb)]:
            assert _pads_zero(param_arena(net), net), name
        for opt, net in ((la.optimizers["value_optimizer"], la.nets["value_net"]), (lb.optim, lb)):
            if kind != "torch_adam":
                assert opt.steps_taken() == 7
                assert all(_pads_zero(a, net) for a in (opt._m, opt._v, opt._slow) if a is not None)
        # a local block is the full tensor's block
        w = la.nets["value_net"].linear1.weight
        assert torch.equal(w[:, S:], full["nets"]["value_net"]["linear1.weight"][:, S + lo:S + hi])
        assert torch.equal(lb.net[0].bias, full["beta"]["net"]["net.0.bias"][lo:hi])
        nets, opts, vp = D._checkpoint_parts(la, lb)
        ranks.append((D._gather_begin(nets, opts, ITEMS, r == 0), hi - lo))
    (leaves, agree, out), _ = ranks[0]
    assert all(x[0][1] == agree for x in ranks)
    D._copy_shared(leaves)
    for q, ((q_leaves, _, q_out), n) in enumerate(ranks):
        assert q_out is None or q == 0
        lo, hi = D.vocab_shard(ITEMS, q, world)
        inbox, outbox = list(D._inbox(leaves, lo, hi)), list(D._outbox(q_leaves, n))
        assert len(inbox) == len(outbox) > 0
        for v, s in zip(inbox, outbox):
            v.copy_(s)
    _same(out, full)


@pytest.mark.parametrize("kind", ["ranger", "torch_adam"])
def test_world1_gather_returns_the_state_it_was_loaded_from(one_rank_cpu_group, kind):
    agent, beta = _agent(kind, ITEMS)
    _randomize(agent, beta, 5)
    full = _full_state(agent, beta)
    la, lb = _local(kind, 0, ITEMS, 0, 1)
    D.load_vocab_parallel_state(la, full, beta=lb)
    _same(D.gather_vocab_parallel_state(la, beta=lb), full)
    # a lone policy and a nets dict carry only their parts
    got = D.gather_vocab_parallel_state(la.nets["policy_net"])
    assert set(got) == {"nets"} and set(got["nets"]) == {"policy_net"}
    _same(got["nets"]["policy_net"], full["nets"]["policy_net"])
    got = D.gather_vocab_parallel_state(la.nets)
    assert set(got) == {"nets"}
    _same(got["nets"], full["nets"])


def test_gather_and_load_refuse_unsharded_nets(one_rank_cpu_group):
    agent, beta = _agent("ranger", ITEMS)
    with pytest.raises(RuntimeError, match="not vocabulary-parallel"):
        D.gather_vocab_parallel_state(agent)
    with pytest.raises(RuntimeError, match="not vocabulary-parallel"):
        D.gather_vocab_parallel_state(agent.nets["policy_net"])
    with pytest.raises(RuntimeError, match="not vocabulary-parallel"):
        D.load_vocab_parallel_state(agent, _full_state(agent, beta))
    la, lb = _local("ranger", 0, ITEMS, 0, 1)
    with pytest.raises(RuntimeError, match="beta is not vocabulary-parallel"):
        D.gather_vocab_parallel_state(la, beta=beta)
    with pytest.raises(TypeError):
        D.gather_vocab_parallel_state(lb)


def _refused(agent, beta, state, match):
    before = [param_arena(n).clone() for n in list(agent.nets.values()) + [beta]]
    with pytest.raises(ValueError, match=match):
        D.load_vocab_parallel_state(agent, state, beta=beta)
    after = [param_arena(n) for n in list(agent.nets.values()) + [beta]]
    assert all(torch.equal(x, y) for x, y in zip(before, after))


def test_load_refusals(one_rank_cpu_group):
    import copy
    agent, beta = _agent("ranger", ITEMS, beta_kind="radam")
    _randomize(agent, beta, 3)
    full = _full_state(agent, beta)
    la, lb = _local("ranger", 0, ITEMS, 0, 1)
    lb.optim = _optimizer("radam", lb)
    for items, s, h, what in ((ITEMS + 1, S, H, "num_items"), (ITEMS, S + 1, H, "state_dim"),
                              (ITEMS, S, H + 1, "hidden")):
        other = recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(s, items, h), recnn_b200.nn.Critic(s, items, h))
        bad = dict(full, nets={k: v.state_dict() for k, v in other.nets.items()})
        _refused(la, lb, bad, "state_dim, hidden size and num_items")
    bad = copy.deepcopy(full)
    del bad["nets"]["target_value_net"]
    _refused(la, lb, bad, "no state\\['nets'\\]\\['target_value_net'\\]")
    bad = copy.deepcopy(full)
    del bad["optimizers"]["value_optimizer"]
    _refused(la, lb, bad, "no state\\['optimizers'\\]\\['value_optimizer'\\]")
    bad = copy.deepcopy(full)
    del bad["beta"]
    _refused(la, lb, bad, "no state\\['beta'\\]")
    bad = copy.deepcopy(full)
    bad["optimizers"]["policy_optimizer"]["recnn_arenas"]["slow"] = None
    _refused(la, lb, bad, "a Ranger needs")
    bad = copy.deepcopy(full)                           # Ranger arenas into β's RAdam
    bad["beta"]["optim"]["recnn_arenas"]["slow"] = bad["beta"]["optim"]["recnn_arenas"]["m"].clone()
    _refused(la, lb, bad, "a RAdam needs")
    bad = copy.deepcopy(full)
    bad["optimizers"]["value_optimizer"]["recnn_arenas"]["m"] = torch.zeros(5)
    _refused(la, lb, bad, "the full arena")
    ta, tb = _agent("torch_adam", ITEMS)
    _randomize(ta, tb, 4)
    torch_state = _full_state(ta, tb)
    _refused(la, lb, dict(full, optimizers=torch_state["optimizers"]), "torch optimizer's state")
    lt, ltb = _local("torch_adam", 0, ITEMS, 0, 1)
    _refused(lt, ltb, full, "built-in optimizer's arenas")
    bad = copy.deepcopy(torch_state)
    bad["optimizers"]["policy_optimizer"]["state"][2]["exp_avg"] = torch.zeros(ITEMS - 1, H)
    _refused(lt, ltb, bad, "the parameter is")
    D.load_vocab_parallel_state(la, full, beta=lb)      # the good one loads


def test_ranks_that_disagree_on_the_step_count_raise(one_rank_cpu_group, monkeypatch):
    agent, beta = _agent("adam", ITEMS)
    _randomize(agent, beta, 6)
    la, lb = _local("adam", 0, 502, 0, 2)              # rank 0 of 2, the other rank stood in for below
    monkeypatch.setattr(D.dist, "all_gather_object", lambda out, obj, group=None: out.__setitem__(slice(None),
                                                                                                  [None, None]))
    D.load_vocab_parallel_state(la, _full_state(agent, beta), beta=lb)

    def other_rank_stepped_more(out, obj, group=None):
        out[0] = obj
        out[1] = [(a[0], a[1], a[2] + 1) if a[1] == "t" else a for a in obj]
    monkeypatch.setattr(D.dist, "all_gather_object", other_rank_stepped_more)
    with pytest.raises(RuntimeError, match="disagree"):
        D.gather_vocab_parallel_state(la, beta=lb)
