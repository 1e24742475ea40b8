"""Host-side checks of the vocabulary-parallel REINFORCE policy: the float64 oracle of the device formulation (layer-1
gradient all-reduced instead of dh, the sharded draw) against the unsharded oracle, the shard plan and its refusals, the
communicator sizing and the scratch of the phases.  No kernel is launched."""
from __future__ import annotations

import numpy as np
import pytest

from oracle import reinforce_oracle as RO
from recnn_b200 import _lib
from recnn_b200 import dist as D
from tests import _vocab_oracle as VO

WORLDS = [1, 2, 3, 8]


def _case(S, H, I, n, seed):
    rng = np.random.default_rng(seed)
    p = RO.make_discrete_actor(rng, S, I, H)
    p["w2"] = (p["w2"] * 8).astype(np.float32)             # a peaked softmax: shards carry very different masses
    state = rng.normal(0, 1, (n, S)).astype(np.float32)
    action = rng.integers(0, I, n)
    blp = np.log(rng.uniform(0.01, 0.05, n)).astype(np.float32)
    ret = rng.normal(0, 1, n).astype(np.float32)
    return rng, p, state, action, blp, ret


@pytest.mark.parametrize("world", WORLDS)
@pytest.mark.parametrize("method", [RO.BASIC, RO.CORRECTED, RO.TOPK])
def test_layer1_allreduce_variant_equals_both_formulations(world, method):
    """37 items: shards of 37 / 19+18 / 13+13+11 / 5 x 7 + 2 -- uneven at every W > 1.  Action ids at every shard
    edge (lo - 1, lo, hi - 1)."""
    S, H, I, n = 11, 16, 37, 40
    _, p, state, action, blp, ret = _case(S, H, I, n, 100 + world + 10 * method)
    shards = RO.shard_policy(p, world)
    edges = sorted({e for sh in shards for e in (sh["offset"] - 1, sh["offset"], sh["offset"] + len(sh["b2"]) - 1)
                    if 0 <= e < I})
    action[:len(edges)] = edges
    beta = None if method == RO.BASIC else blp
    want_loss, want, _ = RO.reinforce_policy_grad(p, state, action, beta, ret, method, 10)
    dh_loss, dh_grads = RO.sharded_policy_grad(shards, state, action, beta, ret, method, 10)
    loss, grads = VO.sharded_policy_grad_layer1(shards, state, action, beta, ret, method, 10)
    assert loss == pytest.approx(want_loss, rel=1e-12, abs=1e-12)
    assert loss == pytest.approx(dh_loss, rel=1e-12, abs=1e-12)
    for k in ("w1", "b1"):
        for gr, ref in zip(grads, dh_grads):
            np.testing.assert_allclose(gr[k], ref[k], rtol=1e-10, atol=1e-12)
            np.testing.assert_allclose(gr[k], want[k], rtol=1e-10, atol=1e-12)
    for k in ("w2", "b2"):
        np.testing.assert_allclose(np.concatenate([g[k] for g in grads]), want[k], rtol=1e-10, atol=1e-12)


@pytest.mark.parametrize("world", WORLDS)
def test_sharded_draw_picks_the_unsharded_item(world):
    """For the same u, the owner-then-inside draw picks the unsharded inverse-CDF item (rows within 1e-9 of an
    interval end are skipped); u at 0 and just below 1 included."""
    _, p, state, _, _, _ = _case(9, 12, 29, 400, 7 + world)
    probs, _ = RO.discrete_forward(p, state)
    u = np.random.default_rng(world).random(400)
    u[:2] = [0.0, np.nextafter(1.0, 0.0)]
    want, _, margin = RO.categorical_sample(probs, u)
    shards = RO.shard_policy(p, world)
    offsets = [sh["offset"] for sh in shards]
    blocks = [probs[:, o:o + len(sh["b2"])] for o, sh in zip(offsets, shards)]
    got = VO.sharded_sample(blocks, offsets, u)
    keep = margin > 1e-9
    assert keep.sum() > 380
    np.testing.assert_array_equal(got[keep], want[keep])


def test_shard_plan():
    assert D.vocab_shard(1_000_000, 7, 8) == (875_000, 1_000_000)
    assert [D.vocab_shard(37, r, 3) for r in range(3)] == [(0, 13), (13, 26), (26, 37)]
    assert [D.vocab_shard(37, r, 8) for r in range(8)][-2:] == [(30, 35), (35, 37)]
    assert D.vocab_shard(5, 0, 1) == (0, 5)
    for world in (1, 2, 3, 8):
        plans = [D.vocab_shard(1001, r, world) + (1001,) for r in range(world)]
        D.check_vocab_plans(plans)
        # the oracle's split
        assert [lo for lo, _, _ in plans] == [sh["offset"] for sh in RO.shard_policy({"w2": np.zeros((1001, 1)),
                                                                                        "b2": np.zeros(1001), "w1": 0,
                                                                                        "b1": 0}, world)]


@pytest.mark.parametrize("items,world,rank", [(9, 8, 5), (9, 8, 7), (3, 4, 3), (1, 2, 1)])
def test_empty_shards_are_refused(items, world, rank):
    with pytest.raises(ValueError, match="without items"):
        D.vocab_shard(items, rank, world)


@pytest.mark.parametrize("plans", [
    [(0, 5, 10), (5, 10, 11)],           # disagree on the vocabulary
    [(0, 5, 10), (6, 10, 10)],           # a gap
    [(0, 6, 10), (5, 10, 10)],           # an overlap
    [(0, 5, 10), (5, 9, 10)],            # short of the end
    [(0, 0, 10), (0, 10, 10)],           # an empty block
    [(5, 10, 10), (0, 5, 10)],           # out of rank order
])
def test_disagreeing_plans_are_refused(plans):
    with pytest.raises(ValueError):
        D.check_vocab_plans(plans)


def test_comm_sizing():
    """The layer-1 block (H x pad4(S) + pad4(H)) or W records of 4 + 3 rows floats, whichever is larger."""
    L = _lib.lib()
    assert [L.recnn_vocab_record_floats(n) for n in (1, 2, 163_840)] == [7, 10, 4 + 3 * 163_840]
    assert L.recnn_vocab_record_floats(0) == 0
    d = _lib.DiscreteDims(2570, 256, 125_000, 0)
    layer1 = 256 * 2572 + 256
    assert D.layer1_floats(d) == layer1
    assert D.vocab_comm_floats(d, 8, 1) == layer1
    assert D.vocab_comm_floats(d, 8, 163_840) == 8 * (4 + 3 * 163_840)
    assert D.vocab_comm_floats(_lib.DiscreteDims(13, 5, 7, 0), 3, 4) == max(5 * 16 + 8, 3 * 16)


def test_phase_scratch_does_not_grow_with_the_vocabulary():
    """A rank's stats / gradient phases take recnn_reinforce_scratch_floats of its local dims, the forward phase
    recnn_discrete_scratch_floats(..., 0): once the local chunk is narrower than the local slice, neither depends on the
    vocabulary."""
    L = _lib.lib()
    for S, H, R, chunk, world in [(2570, 256, 163_840, 1536, 8), (52, 64, 40, 128, 3), (1290, 256, 4096, 512, 2)]:
        sizes, fwd = set(), set()
        for items in (world * (chunk + 1), 262_144, 1_000_000, 8_000_003):
            for r in (0, world - 1):
                lo, hi = D.vocab_shard(items, r, world)
                d = _lib.DiscreteDims(S, H, hi - lo, 0)
                sizes.add(L.recnn_reinforce_scratch_floats(d, R, chunk))
                fwd.add(L.recnn_discrete_scratch_floats(d, R, 0))
        assert len(sizes) == 1 and len(fwd) == 1, (S, H, R, chunk, sizes, fwd)
        assert sizes.pop() < R * (S + 3 + 2 * H + chunk + 8) + 2 * (chunk + 64 * 1024) * (H + 1) + 4096
