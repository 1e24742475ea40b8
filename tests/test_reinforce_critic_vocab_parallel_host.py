"""Host-side checks of the vocabulary-parallel item-id critic: the float64 formulation of the sharded step (begin /
all-gather / merge / all-reduce / end) against the unsharded one-hot step, the agent-level plan checks and refusals of
enable_vocab_parallel and reinforce_update, the C symbols and the phase memory.  No kernel is launched."""
from __future__ import annotations

import ctypes
import os
import re

import numpy as np
import pytest
import torch

import recnn_b200
from oracle import recnn_oracle as O
from oracle import reinforce_oracle as RO
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.nn.update import _ids
from tests import _critic_vocab_oracle as CV
from tests._ranks import one_rank_cpu_group  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORLDS = [1, 2, 3, 8]
PARAMS = dict(gamma=0.99, min_value=-10, max_value=10)


def _case(S, H, Hp, I, n, seed, world):
    """37 items: shards of 37 / 19+18 / 13+13+11 / 5 x 7 + 2.  Ids at every shard edge, a quarter of the rows repeating
    ids of other rows."""
    rng = np.random.default_rng(seed)
    pp = RO.make_discrete_actor(rng, S, I, Hp)
    pp["w2"] = (pp["w2"] * 6).astype(np.float32)             # a peaked softmax: shards carry very different masses
    cp = O.make_critic(rng, S, I, H, 0.3)
    tcp = O.make_critic(rng, S, I, H, 0.3)
    a = rng.integers(0, I, n)
    a[:n // 4] = a[n // 4:n // 2]
    edges = sorted({e for lo, hi in CV.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
    a[n // 2:n // 2 + len(edges)] = edges
    batch = {"state": rng.normal(0, 1, (n, S)).astype(np.float32), "next_state": rng.normal(0, 1, (n, S)).astype(np.float32),
             "action": a, "reward": (rng.integers(1, 6, n) - 3).astype(np.float32),
             "done": (rng.random(n) < 0.1).astype(np.float32)}
    return rng, pp, cp, tcp, batch


def _steps(p, g, kind):
    """One optimizer step of the oracle (elementwise: a rank steps its arena as the unsharded net would)."""
    q = {k: np.asarray(p[k], np.float32).copy() for k in O.PARAM_ORDER}
    O.optimizer_step(O.make_optimizer(kind, lr=1e-2), q, {k: g[k] for k in O.PARAM_ORDER})
    return q


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("train", [False, True], ids=["eval", "masks"])
def test_sharded_step_equals_the_one_hot_step(world, train):
    S, H, Hp, I, n = 11, 16, 12, 37, 40
    rng, pp, cp, tcp, batch = _case(S, H, Hp, I, n, 7 * world + int(train), world)
    masks = [(rng.random((n, H)) >= 0.5).astype(np.uint8) for _ in range(2)] if train else None
    nets = {"value_net": cp, "target_value_net": tcp, "target_policy_net": pp}
    want_loss, want, oob = CV.value_step(nets, batch, PARAMS, masks)
    assert not oob
    # the float64 restatement of the dense step agrees with the fp32 oracle of reinforce_update's critic half
    onehot = dict(batch, action=np.eye(I, dtype=np.float32)[batch["action"]])
    fp32_loss, _ = RO.value_update(onehot, PARAMS, {k: O.copy_net(v) if k != "target_policy_net" else v
                                                    for k, v in nets.items()},
                                   {"value_optimizer": O.make_optimizer("sgd", lr=0.0)}, masks, learn=False)
    assert float(fp32_loss) == pytest.approx(want_loss, rel=2e-5)

    cs, tcs = CV.shard_critic(cp, S, world), CV.shard_critic(tcp, S, world)
    losses, grads, flags, _ = CV.sharded_value_step(cs, tcs, RO.shard_policy(pp, world), batch, PARAMS, masks)
    assert flags == [False] * world
    for loss in losses:
        assert loss == pytest.approx(want_loss, rel=1e-12, abs=1e-15)
    for g in grads:
        for k in ("b1", "w2", "b2", "w3", "b3"):
            np.testing.assert_allclose(g[k], want[k], rtol=1e-10, atol=1e-15)
        np.testing.assert_allclose(g["w1"][:, :S], want["w1"][:, :S], rtol=1e-10, atol=1e-15)
    block = np.concatenate([g["w1"][:, S:] for g in grads], 1)
    np.testing.assert_allclose(block, want["w1"][:, S:], rtol=1e-10, atol=1e-15)
    unselected = np.setdiff1d(np.arange(I), batch["action"])
    assert unselected.size > 0 and np.all(block[:, unselected] == 0.0)
    # one SGD and one Adam step: each rank's local arena against the same columns of the unsharded step
    for kind in ("sgd", "adam"):
        full = _steps(cp, want, kind)
        for r, (c, g) in enumerate(zip(cs, grads)):
            got = _steps(c, g, kind)
            lo, hi = CV.item_plan(I, world)[r]
            for k in O.PARAM_ORDER:
                ref = full[k] if k != "w1" else np.concatenate([full["w1"][:, :S], full["w1"][:, S + lo:S + hi]], 1)
                np.testing.assert_allclose(got[k], ref, rtol=1e-6, atol=1e-7 * np.abs(ref).max(), err_msg=(kind, k))


@pytest.mark.parametrize("world", [1, 3])
def test_an_id_outside_the_vocabulary_is_a_zero_term_on_every_rank(world):
    S, H, Hp, I, n = 11, 16, 12, 37, 24
    _, pp, cp, tcp, batch = _case(S, H, Hp, I, n, 99, world)
    batch["action"][[3, 5]] = [I, -1]
    nets = {"value_net": cp, "target_value_net": tcp, "target_policy_net": pp}
    want_loss, want, oob = CV.value_step(nets, batch, PARAMS)
    assert oob
    losses, grads, flags, terms = CV.sharded_value_step(CV.shard_critic(cp, S, world), CV.shard_critic(tcp, S, world),
                                                        RO.shard_policy(pp, world), batch, PARAMS)
    assert flags == [True] * world
    assert np.all(terms["add"][[3, 5]] == 0.0)
    assert losses[0] == pytest.approx(want_loss, rel=1e-12)
    np.testing.assert_allclose(np.concatenate([g["w1"][:, S:] for g in grads], 1), want["w1"][:, S:], rtol=1e-10,
                               atol=1e-15)


# ----------------------------------------------------------------------------- the agent-level plan and refusals
def _agent(S=6, H=8, I=10, critic_items=None):
    torch.manual_seed(0)
    policy = recnn_b200.nn.DiscreteActor(S, I, H)
    value = recnn_b200.nn.Critic(S, I if critic_items is None else critic_items, H)
    return recnn_b200.nn.Reinforce(policy, value)


def test_critics_that_do_not_match_the_policy_are_refused(one_rank_cpu_group):
    with pytest.raises(ValueError, match="Critic"):
        D.enable_vocab_parallel(_agent(critic_items=9))
    agent = _agent()
    nets = dict(agent.nets, target_value_net=recnn_b200.nn.Critic(6, 11, 8))
    with pytest.raises(ValueError, match="Critic"):
        D.enable_vocab_parallel(nets)
    nets = dict(agent.nets, target_value_net=recnn_b200.nn.Critic(5, 11, 8))      # same width, other split
    with pytest.raises(ValueError, match="Critic"):
        D.enable_vocab_parallel(nets)
    with pytest.raises(ValueError, match="target_policy_net"):
        D.enable_vocab_parallel({k: v for k, v in agent.nets.items() if k != "target_policy_net"})
    with pytest.raises(TypeError):
        D.enable_vocab_parallel(dict(agent.nets, policy_net=recnn_b200.nn.Actor(6, 10, 8)))
    for net in agent.nets.values():
        assert "_recnn_vp" not in net.__dict__


def test_nets_sharded_apart_are_refused():
    agent = _agent()
    a = D.VocabParallel(0, 10, 10, None, 0, 1, None)
    b = D.VocabParallel(0, 10, 10, None, 0, 1, None)
    assert _ids.vocab_parallel_of(agent.nets) is None
    for k in ("value_net", "target_value_net", "target_policy_net"):
        agent.nets[k].__dict__["_recnn_vp"] = a
    assert _ids.vocab_parallel_of(agent.nets) is a
    agent.nets["target_value_net"].__dict__["_recnn_vp"] = b
    with pytest.raises(RuntimeError, match="sharded together"):
        _ids.vocab_parallel_of(agent.nets)
    del agent.nets["target_policy_net"].__dict__["_recnn_vp"]
    with pytest.raises(RuntimeError, match="sharded together"):
        _ids.vocab_parallel_of(agent.nets)


def test_a_copied_net_shares_the_plan():
    """algo._target_of deep-copies the online net: a sharded net's copy shares its VocabParallel (and communicator)."""
    from recnn_b200.nn.algo import _target_of
    policy = recnn_b200.nn.DiscreteActor(6, 10, 8)
    vp = D.VocabParallel(0, 10, 10, object(), 0, 1, object())
    policy.__dict__["_recnn_vp"] = vp
    assert _target_of(policy).__dict__["_recnn_vp"] is vp


def test_reinforce_update_refusals_name_choose_reinforce():
    """On a sharded policy: a dense [N, num_items] action, or item ids with critics not sharded with it, are refused
    before any net but the policy is touched."""
    agent = _agent()
    vp = D.VocabParallel(0, 10, 10, None, 0, 1, None)
    agent.nets["policy_net"].__dict__["_recnn_vp"] = vp
    N = 4
    state = torch.zeros(N, 6)
    with pytest.raises(RuntimeError, match="ChooseREINFORCE"):
        recnn_b200.nn.reinforce_update({"state": state, "action": torch.zeros(N, 10)}, {},
                                       {"policy_net": agent.nets["policy_net"]}, {})
    with pytest.raises(RuntimeError, match="ChooseREINFORCE"):
        recnn_b200.nn.reinforce_update({"state": state, "action": torch.zeros(N, dtype=torch.int64)}, {},
                                       agent.nets, {})
    for k in ("value_net", "target_value_net", "target_policy_net"):
        agent.nets[k].__dict__["_recnn_vp"] = vp
    with pytest.raises(RuntimeError, match="ChooseREINFORCE"):
        recnn_b200.nn.reinforce_update({"state": state, "action": torch.zeros(N, 10)}, {}, agent.nets, {})
    with pytest.raises(RuntimeError, match="item-id"):
        recnn_b200.nn.value_update({"state": state, "action": torch.zeros(N, 10), "next_state": state,
                                    "reward": torch.zeros(N), "done": torch.zeros(N)}, {}, agent.nets, {})


# ----------------------------------------------------------------------------- the C ABI
NEW_SYMBOLS = ("recnn_discrete_value_shard_begin", "recnn_discrete_value_shard_merge", "recnn_discrete_value_shard_end")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))


def test_phase_memory_does_not_grow_with_the_vocabulary():
    """A rank's workspace (recnn_discrete_value_workspace_bytes of its local dims), its record and the [2, N, H] terms:
    once the chunk is narrower than the local block, none depends on the vocabulary."""
    L = _lib.lib()
    for S, H, N, chunk, world in [(2570, 256, 16_384, 1024, 8), (2570, 256, 2048, 4096, 8), (52, 64, 40, 128, 3)]:
        sizes = set()
        for items in (world * (chunk + 1), 262_144, 1_000_000, 8_000_003):
            for r in (0, world - 1):
                lo, hi = D.vocab_shard(items, r, world)
                d, pd = _lib.Dims(S, hi - lo, H, 0), _lib.DiscreteDims(S, H, hi - lo, 0)
                ws = L.recnn_discrete_value_workspace_bytes(d, pd, N, chunk)
                assert ws > 0
                sizes.add((ws, L.recnn_vocab_record_floats(N)))
        assert len(sizes) == 1, (S, H, N, chunk, sizes)
        ws, rec = sizes.pop()
        assert rec == 4 + 3 * N
        # one logits chunk, three state images, [N, H] buffers and the projection's split-K partials
        assert ws < N * (chunk + 4) * 4 + N * (3 * (S + 4) + 24 * H) * 4 + (64 << 20)
    assert ctypes.sizeof(_lib.VocabShard) == 16
