"""The virtual-rank runner of tests/_ranks.py on CPU tensors: exchanges in rank order, per-rank results, every rank's
own copy of the caller's RNG stream, and every rank raising when the ranks' exchanges do not match."""
from __future__ import annotations

import pytest
import torch

from tests._ranks import RanksError, exchange, returned, run_ranks

WORLDS = [1, 2, 3, 8]


@pytest.mark.parametrize("world", WORLDS)
def test_gather_in_rank_order_and_results_per_rank(world):
    def fn(r):
        out = exchange().all_gather(torch.arange(3, dtype=torch.int32) + 10 * r)
        return r, out
    res = returned(run_ranks(world, fn))
    want = torch.cat([torch.arange(3, dtype=torch.int32) + 10 * q for q in range(world)])
    assert [r for r, _ in res] == list(range(world))
    for _, out in res:
        assert torch.equal(out, want)
    assert len({id(out) for _, out in res}) == world          # a new tensor per rank


def test_gather_under_a_permutation_of_one_exchange():
    log = []

    def fn(r):
        return [exchange().all_gather(torch.full((2,), float(r))) for _ in range(2)]
    res = returned(run_ranks(3, fn, order={1: [1, 0, 2]}, log=log))
    for first, second in res:
        assert first.tolist() == [0, 0, 1, 1, 2, 2]
        assert second.tolist() == [1, 1, 0, 0, 2, 2]
    assert [k for k, _ in log] == ["all_gather"] * 2 and torch.equal(log[1][1], res[0][1])


@pytest.mark.parametrize("world", WORLDS)
def test_reduce_is_the_in_order_sum_on_every_rank(world):
    g = torch.Generator().manual_seed(world)
    xs = [torch.randn(1001, generator=g) * 10 ** (q % 4) for q in range(world)]
    log = []

    def fn(r):
        t = xs[r].clone()
        assert exchange().all_reduce(t) is t
        return t
    res = returned(run_ranks(world, fn, log=log))
    want = xs[0].clone()
    for x in xs[1:]:
        want += x
    for t in res:
        assert torch.equal(t.view(torch.int32), want.view(torch.int32))
    assert log[0][0] == "all_reduce" and torch.equal(log[0][1], want)


@pytest.mark.parametrize("world", [2, 3])
def test_every_rank_draws_the_callers_stream(world):
    torch.manual_seed(1234)
    want = torch.rand(5), torch.rand(5)
    torch.manual_seed(1234)

    def fn(r):
        a = torch.rand(5)
        exchange().all_gather(torch.zeros(1))
        b = torch.rand(5)
        return a, b, torch.initial_seed()
    res = returned(run_ranks(world, fn))
    for a, b, seed in res:
        assert torch.equal(a, want[0]) and torch.equal(b, want[1]) and seed == 1234
    assert torch.equal(torch.rand(5), want[0])                 # the caller's state is restored


def _all_raise(res, own=None):
    for r, out in enumerate(res):
        assert isinstance(out, own if own is not None and r == 1 else RanksError), (r, out)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_a_rank_that_raises_makes_every_rank_raise(world):
    def fn(r):
        if r == 1:
            raise KeyError("boom")
        exchange().all_gather(torch.zeros(2))
        return r
    _all_raise(run_ranks(world, fn, timeout=30), KeyError)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_a_rank_that_returns_early_makes_every_rank_raise(world):
    def fn(r):
        exchange().all_reduce(torch.zeros(2))
        if r != 0:
            exchange().all_gather(torch.zeros(2))
        return r
    res = run_ranks(world, fn, timeout=30)
    assert all(isinstance(out, RanksError) for out in res), res


@pytest.mark.parametrize("world", [2, 3, 8])
def test_a_rank_that_gathers_another_size_makes_every_rank_raise(world):
    def fn(r):
        exchange().all_gather(torch.zeros(4 if r == world - 1 else 3))
        return r
    res = run_ranks(world, fn, timeout=30)
    assert all(isinstance(out, RanksError) for out in res), res
    res = run_ranks(world, lambda r: exchange().all_gather(torch.zeros(3, dtype=torch.int32 if r else torch.float32)),
                    timeout=30)
    assert all(isinstance(out, RanksError) for out in res), res


def test_ranks_that_raise_after_every_exchange_keep_their_errors():
    def fn(r):
        exchange().all_gather(torch.zeros(1))
        raise IndexError(r)
    res = run_ranks(3, fn)
    assert [type(e) for e in res] == [IndexError] * 3 and [e.args[0] for e in res] == [0, 1, 2]
