"""DiscreteActor.sample_topk / recnn_discrete_sample_topk / the sharded pair on the GPU: against the float64
restatement in tests/_policy_sample_oracle.py (the same Philox bits, logs in float64), against the dense forward, as
a distribution, across chunkings, seeds, exclusions, virtual vocabulary ranks and virtual row ranks (tests/_ranks.py),
and at 1M items."""
from __future__ import annotations

import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200 import dist as D
from recnn_b200.data import ItemSets
from recnn_b200.nn.arena import param_arena
from tests import _policy_sample_oracle as PS
from tests import _policy_topk_oracle as TK
from tests._discrete import make_policy
from tests._ranks import chunked, exchange, returned, run_ranks, shard
from tests.test_policy_sample_host import check_distribution
from tests.test_policy_topk_gpu import KS, SHAPES, Z_BAR, make_case
from tests.test_reinforce_chunked_gpu import REORDER_BAR

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def key_bar(z):
    """fp32 error of a perturbed key z + G: the logit's (Z_BAR, as the top-k tests) plus G's and the sum's rounding."""
    return Z_BAR * (1 + np.abs(z).max() + PS.G_MAX)


def padded(lists, width=None):
    width = max(len(x) for x in lists) if width is None else width
    out = np.full((len(lists), max(width, 1)), -1, dtype=np.int64)
    for r, x in enumerate(lists):
        out[r, :len(x)] = x
    return out


def check_slate(values, ids, z, k, seed, exclude=None, row0=0, what="", min_sure=0.8):
    """ids equal the float64 slate on every slot the fp32 bar settles (its perturbed key more than the bar from both
    neighbours), and as a set on every row whose k-th / (k+1)-th gap exceeds it; excluded ids never returned; -1 slots
    where the restatement has them; values within the logit bar of float64 pi at the returned ids.  Returns the worst
    relative value error."""
    kk = min(k + 1, z.shape[1])
    want_v, want_i, top_g = PS.sample_topk(z, kk, seed, exclude, row0)
    want_i = want_i[:, :k]
    got_v, got_i = values.cpu().numpy().astype(np.float64), ids.cpu().numpy()
    slot, whole = PS.determined(top_g, k, key_bar(z))
    assert slot.mean() >= min_sure, (what, slot.mean())
    assert np.array_equal(got_i[slot], want_i[slot]), (what, np.nonzero(((got_i != want_i) & slot).any(1))[0][:5])
    for r in np.nonzero(whole)[0]:
        assert sorted(got_i[r]) == sorted(want_i[r]), (what, r)
    assert ((got_i == -1) == (want_i == -1)).all(), what
    if exclude is not None:
        ex = np.asarray(exclude)
        assert not any(np.isin(got_i[r][got_i[r] >= 0], ex[r][ex[r] >= 0]).any() for r in range(len(got_i))), what
    live = got_i >= 0
    M = z.max(1, keepdims=True)
    pi = np.exp(z - M) / np.exp(z - M).sum(1, keepdims=True)
    want_at = np.where(live, np.take_along_axis(pi, np.maximum(got_i, 0), 1), 0.0)
    err = np.where(live, np.abs(got_v - want_at) / np.maximum(want_at, 1e-300), 0.0)
    assert err.max() <= 2 * key_bar(z), (what, err.max())
    assert (got_v[~live] == 0).all(), what
    return float(err.max())


def settled(z, k, seed, exclude=None):
    """[N, k] device bool: the slots the fp32 bar settles (PS.determined)."""
    top_g = PS.sample_topk(z, min(k + 1, z.shape[1]), seed, exclude)[2]
    return torch.from_numpy(PS.determined(top_g, k, key_bar(z))[0]).to(DEV)


def check_forward_values(m, st, values, ids, z, what=""):
    """values against forward() gathered at the ids: the top-k tests' reordering bar relative to the row's largest
    probability, and the logit bar per value."""
    probs = m(st)
    live = ids >= 0
    f = torch.where(live, probs.gather(1, ids.clamp(min=0)), torch.zeros_like(values))
    scale = probs.max(1, keepdim=True)[0]
    r = float(((values - f).abs() / scale).max())
    assert r <= REORDER_BAR, (what, r)
    rel = float(torch.where(live, (values - f).abs() / f.clamp(min=1e-30), torch.zeros_like(f)).max())
    assert rel <= 2 * key_bar(z), (what, rel)
    return r, rel


def run_sweep():
    """Every shape x k x chunking against float64 and against forward(); chunked against one chunk; repeats."""
    worst = [0.0, 0.0, 0.0]
    for S, H, I, N in SHAPES:
        p, state = make_case(S, H, I, N, S + I)
        m = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        for k in KS:
            seed = 1000 * k + I
            sure = settled(z, k, seed)
            one = None
            for chunk in (None, 128, 256):
                with chunked(N, chunk):
                    v, i = m.sample_topk(st, k, seed=seed)
                    v2, i2 = m.sample_topk(st, k, seed=seed)
                assert torch.equal(v2, v) and torch.equal(i2, i), (S, I, k, chunk)
                worst[0] = max(worst[0], check_slate(v, i, z, k, seed, what=(S, I, k, chunk)))
                r, rel = check_forward_values(m, st, v, i, z, what=(S, I, k, chunk))
                worst[1], worst[2] = max(worst[1], r), max(worst[2], rel)
                if one is None:
                    one = i
                else:
                    assert torch.equal(i[sure], one[sure]), (S, I, k, chunk)
        print("sample_topk S %d I %d N %d: ok" % (S, I, N))
    print("worst value error vs float64 %.2e, vs forward %.2e of the row max / %.2e relative" % tuple(worst))


def test_against_float64_forward_and_across_chunkings():
    run_sweep()


def test_against_float64_on_the_cuda_core_back_end():
    """The same sweep with every GEMM on the exact-fp32 CUDA-core kernel, in a process of its own."""
    code = "import sys; sys.path.insert(0, %r); from tests import test_policy_sample_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


def test_seeds():
    S, H, I, N = 37, 32, 2000, 300
    p, state = make_case(S, H, I, N, 21)
    m = make_policy(p, S, H, I)
    st = _t(state)
    _, a = m.sample_topk(st, 10, seed=5)
    _, b = m.sample_topk(st, 10, seed=6)
    assert float((a != b).any(1).float().mean()) > 0.9
    _, c = m.sample_topk(st, 10, seed=2 ** 64 - 1)
    assert float((a != c).any(1).float().mean()) > 0.9
    torch.manual_seed(77)
    v1, i1 = m.sample_topk(st, 10)
    v_next, i_next = m.sample_topk(st, 10)
    torch.manual_seed(77)
    v2, i2 = m.sample_topk(st, 10)
    assert torch.equal(v1, v2) and torch.equal(i1, i2)
    assert float((i_next != i1).any(1).float().mean()) > 0.9
    # batching: a row's slate does not depend on the rows around it when its global row is the same
    _, part = m.sample_topk(st[:17], 10, seed=5)
    z = TK.logits(p, state)
    sure = settled(z, 10, 5)[:17]
    assert torch.equal(part[sure], a[:17][sure])


def test_distribution_on_the_device():
    """12 items, 2^17 identical rows: first-position and ordered-pair frequencies against Plackett-Luce on pi from
    forward(), with and without an exclusion set, and the ids equal to the restatement."""
    S, H, I, R = 20, 16, 12, 1 << 17
    p, state = make_case(S, H, I, 1, 3, spread=1.5)
    m = make_policy(p, S, H, I)
    st = _t(np.repeat(state, R, 0))
    z1 = TK.logits(p, state)[0]
    for exclude in ((), (2, 7)):
        if exclude:
            sets = ItemSets.from_lists([list(exclude)], device=DEV)
            v, i = m.sample_topk(st, 3, exclude=sets, exclude_rows=torch.zeros(R, dtype=torch.int64, device=DEV),
                                 seed=2024)
        else:
            v, i = m.sample_topk(st, 3, seed=2024)
        ids = i.cpu().numpy()
        check_distribution(ids, z1, exclude)
        z = np.tile(z1, (R, 1))
        ex = None if not exclude else np.tile(np.array(exclude), (R, 1))
        _, want, top_g = PS.sample_topk(z, 4, 2024, ex)
        sure = PS.determined(top_g, 3, key_bar(z))[0]
        assert sure.mean() > 0.99 and np.array_equal(ids[sure], want[:, :3][sure])


def test_exclusion_dense_and_sets():
    S, H, I, N = 37, 32, 2000, 40
    p, state = make_case(S, H, I, N, 11)
    m = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    rng = np.random.default_rng(3)
    ex = np.stack([rng.permutation(np.argsort(-z[r])[:80])[:60] for r in range(N)])     # mostly the best items
    ex[:, 50:] = -1
    # sets straddling the 128 / 256 chunk edges, shared through a row map, a row without a set
    lists = [sorted(set(ex[r][ex[r] >= 0].tolist()) | {127, 128, 255, 256}) for r in range(N)]
    rows = np.arange(N)
    rows[5] = -1
    dense_of_rows = padded([lists[r] if r != 5 else [] for r in range(N)])
    sets = ItemSets.from_lists(lists, device=DEV)
    for chunk in (None, 128, 256):
        for k in (10, 64):
            with chunked(N, chunk):
                v, i = m.sample_topk(st, k, exclude=_t(ex), seed=k)
                check_slate(v, i, z, k, k, ex, what=("dense", chunk, k))
                vs, is_ = m.sample_topk(st, k, exclude=sets, exclude_rows=_t(rows), seed=k)
                check_slate(vs, is_, z, k, k, dense_of_rows, what=("sets", chunk, k))
                # the dense form and a table of the same ids give the same bits
                vt, it = m.sample_topk(st, k, exclude=ItemSets.from_lists([x[x >= 0] for x in ex], device=DEV),
                                       seed=k)
                assert torch.equal(vt, v) and torch.equal(it, i)
    bad = ex.copy()
    bad[5, 3] = I
    with pytest.raises(IndexError):
        m.sample_topk(st, 10, exclude=_t(bad))
    with pytest.raises(IndexError):
        m.sample_topk(st, 10, exclude=ItemSets.from_lists([[I]] * N, device=DEV))
    with pytest.raises(ValueError, match="malformed"):
        m.sample_topk(st, 10, exclude=sets, exclude_rows=_t(np.full(N, N)))
    t = ItemSets.from_lists([[1, 2, 3]] * N, device=DEV)
    t.ids[0], t.ids[2] = 9, 1                                # a descending set
    with pytest.raises(ValueError, match="malformed"):
        m.sample_topk(st, 10, exclude=t)


def test_exactly_k_and_fewer_than_k_eligible():
    S, H, I, N = 20, 16, 200, 6
    p, state = make_case(S, H, I, N, 4)
    m = make_policy(p, S, H, I)
    st = _t(state)
    keep = [3, 50, 128, 199]
    rest = [x for x in range(I) if x not in keep]
    sets = ItemSets.from_lists([rest] * N, device=DEV)
    v, i = m.sample_topk(st, 4, exclude=sets, seed=3)
    assert np.array_equal(np.sort(i.cpu().numpy(), 1), np.tile(keep, (N, 1)))
    assert bool((v > 0).all())
    v, i = m.sample_topk(st, 12, exclude=sets, seed=3)
    assert (i[:, 4:] == -1).all() and (v[:, 4:] == 0).all()
    assert np.array_equal(np.sort(i[:, :4].cpu().numpy(), 1), np.tile(keep, (N, 1)))
    check_slate(v, i, TK.logits(p, state), 12, 3, np.tile(rest, (N, 1)), what="short rows")


def test_sample_topk_leaves_the_policy_state_alone():
    S, H, I, N = 20, 16, 300, 8
    p, state = make_case(S, H, I, N, 8)
    m = make_policy(p, S, H, I)
    st = _t(state)
    m.select_action(st)
    saved = (len(m.saved_log_probs), len(m._saved), len(m.rewards), m._draws)
    arena = param_arena(m).clone()
    m.sample_topk(st, 5, seed=1)
    m.sample_topk(st, 5)
    assert (len(m.saved_log_probs), len(m._saved), len(m.rewards), m._draws) == saved
    assert torch.equal(param_arena(m), arena)


# ----------------------------------------------------------------------------- 1M items
def test_million_items_long_tailed_sets():
    """S 2570 / H 256, 2^20 items x 2,048 rows with the long-tailed history sets of the recommendation tests: peak
    memory is the top-k workspace plus the outputs, and sampled rows match a chunked float64 restatement."""
    S, H, I, N, k = 2570, 256, 1 << 20, 2048, 64
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    with torch.no_grad():
        m.linear2.weight.mul_(8.0)
    st = torch.randn(N, S, device=DEV)
    rng = np.random.default_rng(144)
    lengths = np.minimum(rng.pareto(1.6, N) * 75 + 20, 20000).astype(np.int64)
    lengths[::256] = 8192 + np.arange(len(lengths[::256]))
    rows_chk = np.arange(0, N, N // 16)
    with torch.no_grad():
        x = st[_t(rows_chk)].double()
        h = torch.relu(x @ m.linear1.weight.double().T + m.linear1.bias.double())
        z = torch.cat([h @ m.linear2.weight[c:c + 65536].double().T + m.linear2.bias[c:c + 65536].double()
                       for c in range(0, I, 65536)], 1).cpu().numpy()
    lists = [rng.integers(0, I, n) for n in lengths]
    g = PS.perturbed(z, 9, rows_chk)
    for j, r in enumerate(rows_chk):
        # make the checked rows' sets bite: up to 256 of their likeliest draws (deeper, adjacent perturbed keys are
        # closer than the fp32 bar: the gaps of the j-th best are ~1/j)
        bite = min(lengths[r] // 2, 256)
        best = np.argsort(-g[j])[:bite]
        lists[r] = np.concatenate([best, lists[r][:lengths[r] - bite]])
    sets = ItemSets.from_lists(lists, device=DEV)
    from recnn_b200.nn.update.reinforce import _chunk_items
    ws = L.recnn_discrete_topk_workspace_bytes(m.dims, N, k, _chunk_items(N, I))
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    v, i = m.sample_topk(st, k, exclude=sets, seed=9)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("1M items x %d rows with sets: peak extra %.3f GB, workspace %.3f GB" % (N, peak / 1e9, ws / 1e9))
    assert peak <= ws + N * k * 12 + (8 << 20)
    err = check_slate(v[_t(rows_chk)], i[_t(rows_chk)], z, k, 9, padded([lists[r] for r in rows_chk]),
                      row0=rows_chk, what="1M sets", min_sure=0.5)
    print("1M: worst value error vs float64 %.2e" % err)


# ----------------------------------------------------------------------------- virtual vocabulary ranks
def sharded_sample(full, world, state, k, seeds, chunk=None, exclude=None, exclude_rows=None, order=None):
    """policy.sample_topk on W virtual ranks sharded from ``full``, rank r with seed seeds[r]: each rank's
    (values, ids) or exception."""
    def rank(r):
        pol = shard({"policy_net": full})[0]["policy_net"]
        return pol.sample_topk(state, k, exclude=exclude, exclude_rows=exclude_rows, seed=seeds[r])
    with chunked(state.shape[0], chunk):
        return run_ranks(world, rank, order=order)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks(world):
    for S, H, I, N in [(52, 64, 1003, 40), (37, 32, 200, 17)]:      # 200 items over 8 ranks: 25 per block < k = 64
        p, state = make_case(S, H, I, N, I + world, spread=2.0)
        full = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        edges = sorted({e for lo, hi in TK.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
        lists = [edges[r % 3::3] + [r % I] for r in range(N)]   # sets straddling the shard edges
        sets = ItemSets.from_lists(lists, device=DEV)
        dense = padded([sorted(set(x)) for x in lists])
        for k in (10, 64):
            for chunk in (None, 128):
                for ex in (None, sets):
                    res = returned(sharded_sample(full, world, st, k, [k + 1] * world, chunk, ex))
                    vals, ids = res[0]
                    for x in res[1:]:
                        assert torch.equal(x[0], vals) and torch.equal(x[1], ids)
                    want = None if ex is None else dense
                    check_slate(vals, ids, z, k, k + 1, want, what=("W", world, I, k, chunk), min_sure=0.5)
                    with chunked(N, chunk):
                        one_v, one_i = full.sample_topk(st, k, exclude=ex, seed=k + 1)
                    if world == 1:
                        assert torch.equal(vals, one_v) and torch.equal(ids, one_i)
                    sure = settled(z, k, k + 1, want)
                    assert torch.equal(ids[sure], one_i[sure])
        # ranks that disagree on the seed, or records delivered out of rank order, raise on every rank
        res = sharded_sample(full, world, st, 10, [5] * (world - 1) + [6])
        if world > 1:
            assert all(isinstance(e, RuntimeError) and "seed" in str(e) for e in res), res
            res = sharded_sample(full, world, st, 10, [5] * world, order={0: [1, 0] + list(range(2, world))})
            assert all(isinstance(e, RuntimeError) and "disagree" in str(e) for e in res), res
        else:
            returned(res)
        del full


# ----------------------------------------------------------------------------- virtual row ranks
@pytest.mark.parametrize("world", [2, 3, 8])
def test_row_parallel_virtual_ranks_equal_the_whole_batch(world):
    """Data-parallel replicas on uneven row shards: the ranks' slates, concatenated, are the single-GPU call's over
    the whole batch (row r keyed by its global row)."""
    S, H, I, N = 37, 32, 2000, 61
    p, state = make_case(S, H, I, N, 40 + world)
    full = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    cuts = np.sort(np.random.default_rng(world).choice(np.arange(1, N), world - 1, replace=False))
    bounds = list(zip([0] + cuts.tolist(), cuts.tolist() + [N]))

    def rank(r):
        from tests._ranks import _copy
        m = _copy(full)
        ex = exchange()
        D.data_parallel_in_place({"policy_net": m}, D.RowParallel(None, ex.rank, ex.world, ex))
        lo, hi = bounds[r]
        return m.sample_topk(st[lo:hi], 16, seed=123)
    res = returned(run_ranks(world, rank))
    vals = torch.cat([x[0] for x in res])
    ids = torch.cat([x[1] for x in res])
    one_v, one_i = full.sample_topk(st, 16, seed=123)
    sure = settled(z, 16, 123)
    assert bool(sure.float().mean() > 0.8)
    assert torch.equal(ids[sure], one_i[sure])
    assert float(((vals - one_v).abs() / one_v[:, :1]).max()) <= REORDER_BAR
    check_slate(vals, ids, z, 16, 123, what=("rows", world))
