"""Host-side checks of the vocabulary-parallel behaviour policy beta: the float64 two-exchange formulation against the
unsharded float64 oracle, the phase memory, the C symbols and the refusals of enable_vocab_parallel(..., beta=).  No
kernel is launched."""
from __future__ import annotations

import os
import re

import numpy as np
import pytest
import torch

import recnn_b200
from oracle import beta_oracle as B
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.nn.arena import param_arena
from tests import _beta_vocab_oracle as BV
from tests._ranks import one_rank_cpu_group  # noqa: F401

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _case(S, items, n, seed, improbable=False):
    rng = np.random.default_rng(seed)
    w = rng.uniform(-0.3, 0.3, (items, S)).astype(np.float32)
    b = rng.uniform(-0.3, 0.3, items).astype(np.float32)
    ids = rng.integers(0, items, n)
    edges = sorted({e for lo, hi in BV.item_plan(items, 8) for e in (lo - 1, lo, hi - 1) if 0 <= e < items})
    ids[:len(edges)] = edges[:n]
    if improbable:
        b[ids] = -60.0              # p_a ~ 0: every dL/dz is the (e^p - U) / T term
    return w, b, rng.normal(0, 1, (n, S)).astype(np.float32), ids


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("improbable", [False, True], ids=["plain", "improbable"])
def test_two_exchanges_equal_the_unsharded_call(world, improbable):
    """1,003 items: shards of 1003 / 502+501 / 335+335+333 / 126 x 7 + 121."""
    w, b, s, ids = _case(13, 1003, 40, world + 10 * improbable, improbable)
    p, loss, dw, db = B.loss_and_grads(w, b, s, ids)
    out = BV.sharded_call(w, b, s, ids, world)
    assert [o[4] for o in out] == [0] * world
    for o in out:
        assert o[1] == pytest.approx(loss, rel=1e-12, abs=1e-15)
    np.testing.assert_allclose(np.concatenate([o[0] for o in out], 1), p, rtol=1e-12, atol=1e-18)
    np.testing.assert_allclose(np.concatenate([o[2] for o in out], 0), dw, rtol=1e-9, atol=1e-12 * np.abs(dw).max())
    np.testing.assert_allclose(np.concatenate([o[3] for o in out], 0), db, rtol=1e-9, atol=1e-12 * np.abs(db).max())
    if improbable:
        assert np.abs(p[np.arange(len(ids)), ids]).max() < 1e-20


def test_bad_ids_and_rank_order_set_the_error_bits():
    w, b, s, ids = _case(7, 101, 12, 5)
    ids[3] = 101
    assert [o[4] for o in BV.sharded_call(w, b, s, ids, 3)] == [1, 1, 1]
    ids[3] = 0
    assert [o[4] for o in BV.sharded_call(w, b, s, ids, 3, order=[1, 0, 2])] == [2, 2, 2]


def test_phase_memory_does_not_grow_with_the_vocabulary():
    """A rank's workspace (recnn_beta_workspace_bytes of its local dims) and its two records: once the chunk is
    narrower than the local block, neither depends on the vocabulary."""
    L = _lib.lib()
    for S, N, chunk, world in [(2570, 2048, 131072 // 2, 8), (1290, 2048, 4096, 8), (37, 33, 128, 3)]:
        sizes = set()
        for items in (world * (chunk + 1), 1 << 20, 8_000_003):
            for r in (0, world - 1):
                lo, hi = D.vocab_shard(items, r, world)
                ws = L.recnn_beta_workspace_bytes(_lib.BetaDims(S, hi - lo, (0, 0)), N, chunk)
                assert ws > 0
                sizes.add((ws, L.recnn_vocab_record_floats(N)))
        assert len(sizes) == 1, (S, N, chunk, sizes)
        ws, rec = sizes.pop()
        assert rec == 4 + 3 * N
        # the state image, one dZ chunk, seven row vectors and one chunk's split-K partials
        assert ws < N * (S + 4) * 4 + N * chunk * 4 + chunk * (S + 1) * 4 * 8 + (64 << 20)


NEW_SYMBOLS = ("recnn_beta_shard_begin", "recnn_beta_shard_rows", "recnn_beta_shard_end")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))


# ----------------------------------------------------------------------------- refusals
def _agent(S=6, H=8, I=10):
    torch.manual_seed(0)
    return recnn_b200.nn.Reinforce(recnn_b200.nn.DiscreteActor(S, I, H), recnn_b200.nn.Critic(S, I, H))


def _untouched(*nets):
    for net in nets:
        assert "_recnn_vp" not in net.__dict__


def test_betas_that_do_not_match_the_policy_are_refused(one_rank_cpu_group):
    agent = _agent()
    for bad in (recnn_b200.nn.Beta(5, 10), recnn_b200.nn.Beta(6, 11)):
        with pytest.raises(ValueError, match="Beta\\(6, 10\\)"):
            D.enable_vocab_parallel(agent, beta=bad)
        _untouched(bad, *agent.nets.values())
    policy = recnn_b200.nn.DiscreteActor(6, 10, 8)
    with pytest.raises(ValueError, match="Beta\\(6, 10\\)"):
        D.enable_vocab_parallel(policy, beta=recnn_b200.nn.Beta(6, 9))
    with pytest.raises(TypeError):
        D.enable_vocab_parallel(policy, beta=recnn_b200.nn.DiscreteActor(6, 10, 8))
    _untouched(policy)


def test_a_beta_optimizer_with_state_is_refused(one_rank_cpu_group):
    policy = recnn_b200.nn.DiscreteActor(6, 10, 8)
    beta = recnn_b200.nn.Beta(6, 10)
    beta.optim._state_arenas(param_arena(beta))          # what its first step leaves: moments and a step count
    with pytest.raises(RuntimeError, match="already stepped"):
        D.enable_vocab_parallel(policy, beta=beta)
    beta = recnn_b200.nn.Beta(6, 10)
    beta.optim = torch.optim.SGD(beta.net.parameters(), lr=0.1, momentum=0.9)
    for p in beta.net.parameters():
        p.grad = torch.ones_like(p)
    beta.optim.step()
    with pytest.raises(RuntimeError, match="holds state"):
        D.enable_vocab_parallel(policy, beta=beta)
    _untouched(policy, beta)


def test_a_beta_as_the_first_argument_is_still_a_type_error(one_rank_cpu_group):
    beta = recnn_b200.nn.Beta(6, 10)
    with pytest.raises(TypeError):
        D.enable_vocab_parallel(beta)
    with pytest.raises(TypeError):
        D.enable_vocab_parallel(beta, beta=recnn_b200.nn.Beta(6, 10))
    _untouched(beta)


def test_beta_outputs_a_sharded_policy_cannot_draw_from_are_refused():
    """DiscreteActor._beta_records: a column block without its records (a copy), a sharded Beta's block given to an
    unsharded policy, and a Beta sharded on another plan are refused with the reason."""
    import weakref
    from recnn_b200.nn import beta as BM
    vp = D.VocabParallel(0, 5, 10, None, 0, 2, None)
    policy = recnn_b200.nn.DiscreteActor(6, 5, 8)
    policy.__dict__["_recnn_vp"] = vp
    assert policy._beta_records(torch.zeros(4, 10)) is None              # a replicated beta's full probabilities
    with pytest.raises(ValueError, match="without its records"):
        policy._beta_records(torch.zeros(4, 5))
    beta = recnn_b200.nn.Beta(6, 5)
    block, records = torch.zeros(4, 5), torch.zeros(2 * (4 + 3 * 4))
    beta.__dict__["_recnn_vp"] = vp
    beta.__dict__["_recnn_block"] = (weakref.ref(block), records)
    BM._SHARDED.add(beta)
    assert policy._beta_records(block) is records
    with pytest.raises(ValueError, match="without its records"):
        policy._beta_records(block.clone())
    with pytest.raises(ValueError, match="not vocabulary-parallel"):
        recnn_b200.nn.DiscreteActor(6, 10, 8)._beta_records(block)
    other = recnn_b200.nn.DiscreteActor(6, 4, 8)
    other.__dict__["_recnn_vp"] = D.VocabParallel(0, 4, 10, None, 0, 3, None)
    with pytest.raises(ValueError, match="sharded on"):
        other._beta_records(block)
