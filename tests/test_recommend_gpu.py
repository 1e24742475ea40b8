"""Serving with exclusion sets on the GPU: DiscreteActor.topk / ItemIndex.search with an ItemSets table (and the C calls
behind them) against float64 rankings with the sets as padded exclusion lists, bit identity with the dense form and
across virtual ranks (tests/_ranks.py), the device checks of malformed tables, and the feed's serving state and seen
items against the window gather and numpy."""
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
from recnn_b200.data import DeviceFrameFeed, HistoryCSR, ItemIndex, ItemSets
from recnn_b200.nn.arena import param_arena
from tests import _policy_topk_oracle as TK
from tests._discrete import make_policy
from tests._ranks import chunked, returned, run_ranks, shard
from tests.test_policy_topk_gpu import SHAPES, check_against_oracle, make_case

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()
KS = (1, 10, 17, 64)
STAGE = 4096                    # ids of a set searched in shared memory (kSetStage, csrc/topk.cuh)
FLT_MAX = float(np.finfo(np.float32).max)


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def padded(sets_np, rows):
    """The sets of `rows` (row -> set, -1 none) as a dense [N, E] list padded with -1: the oracle's exclusion."""
    e = max([1] + [len(sets_np[s]) for s in rows if s >= 0])
    out = np.full((len(rows), e), -1, dtype=np.int64)
    for r, s in enumerate(rows):
        if s >= 0:
            out[r, :len(sets_np[s])] = sets_np[s]
    return out


def make_sets(z, k, seed):
    """Sets of lengths 0, 1, 255, 257, above the stage and num_items - k + 1, drawn mostly from each row's best items,
    with duplicates and ids on the 128 / 256 chunk edges; returns (lists, row -> set) with shared sets and -1 rows."""
    rng = np.random.default_rng(seed)
    n, items = z.shape
    lengths = [0, 1, 255, 257, STAGE + 3, items - k + 1]
    lists = []
    for s in range(n):
        m = min(lengths[s % len(lengths)], items)
        best = np.argsort(-z[s])[:max(2 * m, 1)]
        x = rng.permutation(best)[:m]
        if m >= 8:
            x[:4] = [127, 128, 255, 256 % items]
            x[4:6] = x[6:8]                                     # duplicates
        if m == items - k + 1:
            x = np.argsort(-z[s])[:m]                            # leaves k - 1 eligible items
        lists.append(x.astype(np.int64))
    rows = np.arange(n)
    rows[1::7] = -1
    rows[2::5] = 3                                              # rows sharing set 3
    return lists, rows


def call_sets(m, state, k, sets, rows, chunk=None):
    """(values, ids, bits) of one recnn_discrete_topk_sets call on an ItemSets table (or raw (ids, offsets))."""
    d = m.dims
    n = state.shape[0]
    chunk = d.num_items if chunk is None or chunk >= d.num_items else chunk
    nbytes = L.recnn_discrete_topk_workspace_bytes(d, n, k, chunk)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    values = torch.empty(n, k, device=DEV)
    ids = torch.empty(n, k, dtype=torch.int64, device=DEV)
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    sid, off = (sets.ids, sets.offsets) if isinstance(sets, ItemSets) else sets
    rows = None if rows is None else _t(np.asarray(rows, dtype=np.int64))
    _lib.check(L.recnn_discrete_topk_sets(d, param_arena(m).data_ptr(), state.data_ptr(), n, k,
                                          sid.data_ptr() if sid.numel() else None, sid.numel(), off.data_ptr(),
                                          off.numel() - 1, _lib.ptr(rows), chunk, values.data_ptr(), ids.data_ptr(),
                                          flag.data_ptr(), ws.data_ptr(), nbytes, _lib.stream_ptr()))
    torch.cuda.synchronize()
    return values, ids, int(flag)


def run_sets_sweep():
    for S, H, I, N in SHAPES:
        p, state = make_case(S, H, I, N, 3 * S + I)
        m = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        for k in KS:
            lists, rows = make_sets(z, k, k)
            sets = ItemSets.from_lists(lists, device=DEV)
            ex = padded(lists, rows)
            for chunk in (None, 128):
                v, i, flag = call_sets(m, st, k, sets, rows, chunk)
                assert flag == 0
                check_against_oracle(v, i, z, k, ex, what=(S, I, k, chunk), min_sure=0)
                got = i.cpu().numpy()
                assert not any(np.isin(got[r], ex[r][ex[r] >= 0]).any() for r in range(N))
                v2, i2, _ = call_sets(m, st, k, sets, rows, chunk)
                assert torch.equal(v2, v) and torch.equal(i2, i)
                with chunked(N, chunk):
                    pv, pi = m.topk(st, k, exclude=sets, exclude_rows=_t(rows))
                assert torch.equal(pv, v) and torch.equal(pi, i)
        print("sets S %d I %d N %d: ok" % (S, I, N))


def test_sets_against_float64():
    run_sets_sweep()


def test_sets_against_float64_on_the_cuda_core_back_end():
    code = "import sys; sys.path.insert(0, %r); from tests import test_recommend_gpu as T; T.run_sets_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


def test_dense_list_and_equal_sets_give_the_same_bits():
    S, H, I, N = 37, 32, 2000, 300
    p, state = make_case(S, H, I, N, 21)
    m = make_policy(p, S, H, I)
    st = _t(state)
    rng = np.random.default_rng(5)
    ex = rng.integers(-1, I, (N, 256))
    ex[:, :10] = np.argsort(-TK.logits(p, state), 1)[:, :10]
    lists = [np.sort(x[x >= 0]) for x in ex]
    sets = ItemSets.from_lists(lists, device=DEV)
    for chunk in (None, 256):
        for k in (10, 64):
            with chunked(N, chunk):
                a = m.topk(st, k, exclude=_t(ex))
                b = m.topk(st, k, exclude=sets)
                c = m.topk(st, k, exclude=sets, exclude_rows=torch.arange(N, device=DEV))
            assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(b[0], c[0]), (chunk, k)
            assert torch.equal(b[1], c[1])


def test_a_set_covering_the_top_k_returns_the_next_items():
    S, H, I, N, k = 52, 64, 1003, 40, 17
    p, state = make_case(S, H, I, N, 8)
    m = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    _, first = TK.topk(z, k)
    want_v, want_i = TK.topk(z, 2 * k)
    sets = ItemSets.from_lists(list(first), device=DEV)
    v, i = m.topk(st, k, exclude=sets)
    sure = TK.boundary_gap(z, 2 * k) > 2e-5 * (1 + np.abs(z).max())
    got = i.cpu().numpy()
    for r in np.nonzero(sure)[0]:
        assert sorted(got[r]) == sorted(want_i[r, k:]), r
    check_against_oracle(v, i, z, k, first, what="covering")


# ----------------------------------------------------------------------------- virtual ranks
def sharded_sets_topk(full, world, state, k, sets, rows, chunk=None):
    def rank(r):
        pol = shard({"policy_net": full})[0]["policy_net"]
        return pol.topk(state, k, exclude=sets, exclude_rows=rows)
    with chunked(state.shape[0], chunk):
        return run_ranks(world, rank)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks_with_sets_on_shard_edges(world):
    S, H, I, N = 52, 64, 1003, 40
    p, state = make_case(S, H, I, N, world + 40)
    full = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    edges = sorted({e for lo, hi in TK.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
    order = np.argsort(-z, 1)
    lists = [np.concatenate([edges, order[r, :30 + r]]) for r in range(N // 2)]
    rows = np.arange(N) % (N // 2)
    rows[::9] = -1
    sets = ItemSets.from_lists(lists, device=DEV)
    rows_d = _t(rows)
    for k in (10, 64):
        for chunk in (None, 128):
            res = returned(sharded_sets_topk(full, world, st, k, sets, rows_d, chunk))
            vals, ids = res[0]
            for x in res[1:]:
                assert torch.equal(x[0], vals) and torch.equal(x[1], ids)
            check_against_oracle(vals, ids, z, k, padded(lists, rows), what=("W", world, k, chunk), min_sure=0)
            if world == 1:
                with chunked(N, chunk):
                    one = full.topk(st, k, exclude=sets, exclude_rows=rows_d)
                assert torch.equal(vals, one[0]) and torch.equal(ids, one[1])
    # bad input raises on every rank
    bad = [np.append(x, I) if r == 3 else x for r, x in enumerate(lists)]
    res = sharded_sets_topk(full, world, st, 10, ItemSets.from_lists(bad, device=DEV), rows_d)
    assert all(isinstance(e, IndexError) for e in res), res
    res = sharded_sets_topk(full, world, st, 10, sets, _t(np.where(rows == 5, N, rows)))
    assert all(isinstance(e, ValueError) for e in res), res
    unsorted = ItemSets.from_lists(lists, device=DEV)
    a, b = int(unsorted.offsets[2]), int(unsorted.offsets[3]) - 1
    unsorted.ids[[a, b]] = unsorted.ids[[b, a]].clone()
    res = sharded_sets_topk(full, world, st, 10, unsorted, rows_d)
    assert all(isinstance(e, ValueError) for e in res), res


# ----------------------------------------------------------------------------- malformed tables
def test_malformed_tables_raise():
    S, H, I, N = 37, 32, 2000, 12
    p, state = make_case(S, H, I, N, 13)
    m = make_policy(p, S, H, I)
    st = _t(state)
    lists = [np.arange(r, 300 + r) for r in range(N)]
    good = ItemSets.from_lists(lists, device=DEV)
    assert call_sets(m, st, 10, good, None)[2] == 0
    ids, off = good.ids.clone(), good.offsets.clone()
    neg = ids.clone(); neg[0] = -3                              # still ascending: only bit 1
    big = ids.clone(); big[299] = I                             # the last id of set 0
    unsorted = ids.clone(); unsorted[[10, 11]] = unsorted[[11, 10]].clone()
    assert call_sets(m, st, 10, (neg, off), None)[2] == 1
    assert call_sets(m, st, 10, (big, off), None)[2] == 1
    assert call_sets(m, st, 10, (unsorted, off), None)[2] == 4
    for at, value in ((1, -1), (3, int(off[2]) - 5), (N, ids.numel() + 9)):    # out of range / decreasing offsets
        bad = off.clone()
        bad[at] = value
        assert call_sets(m, st, 10, (ids, bad), None)[2] == 4, at
    assert call_sets(m, st, 10, (ids, off), np.full(N, N))[2] == 4
    assert call_sets(m, st, 10, (ids, off), np.full(N, -2))[2] == 4
    assert call_sets(m, st, 10, (ids, off), np.full(N, -1))[2] == 0
    with pytest.raises(IndexError):
        m.topk(st, 10, exclude=ItemSets.from_lists([[I]] * N, device=DEV))
    with pytest.raises(IndexError):
        m.topk(st, 10, exclude=ItemSets.from_lists([[-1]] * N, device=DEV))
    with pytest.raises(ValueError):
        m.topk(st, 10, exclude=good, exclude_rows=torch.full((N,), N, device=DEV))
    # only the sets the rows reference are checked
    poisoned = ItemSets.from_lists(lists + [[I + 5]], device=DEV)
    assert call_sets(m, st, 10, poisoned, np.arange(N))[2] == 0


# ----------------------------------------------------------------------------- retrieval
@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_retrieval_with_sets(metric):
    rng = np.random.default_rng(7)
    n_items, dim, n = 5003, 64, 70
    table = rng.normal(0, 1, (n_items, dim)).astype(np.float32)
    q = rng.normal(0, 1, (n, dim)).astype(np.float32)
    t64, q64 = table.astype(np.float64), q.astype(np.float64)
    if metric == "L2":
        key = (t64 ** 2).sum(1)[None] - 2 * q64 @ t64.T
    elif metric == "IP":
        key = -(q64 @ t64.T)
    else:
        key = -(q64 @ t64.T) / np.linalg.norm(t64, axis=1)[None]
    index = ItemIndex(_t(table), metric)
    k = 20
    lists, rows = make_sets(-key, k, 3)
    sets = ItemSets.from_lists(lists, device=DEV)
    res = index.search(_t(q), k, exclude=sets, exclude_rows=_t(rows))
    got = res.id().cpu().numpy()
    ex = padded(lists, rows)
    scale = 1e-4 * (1 + np.abs(key).max())
    for r in range(n):
        keep = np.setdiff1d(np.arange(n_items), ex[r])
        order = keep[np.lexsort((keep, key[r, keep]))]
        want = order[:k]
        gap = key[r, order[k]] - key[r, order[k - 1]] if len(order) > k else np.inf
        live = got[r] >= 0
        assert live.sum() == min(k, len(keep)), r
        assert not np.isin(got[r][live], ex[r][ex[r] >= 0]).any(), r
        if gap > scale:
            assert sorted(got[r][live]) == sorted(want), r
    dist = res.dist().cpu().numpy()
    pad = FLT_MAX if metric == "L2" else -FLT_MAX
    assert (dist[got < 0] == np.float32(pad)).all() and (got < 0).any()
    # every row_set -1: the plain call's bits
    plain = index.search(_t(q), k)
    none = index.search(_t(q), k, exclude=sets, exclude_rows=torch.full((n,), -1, device=DEV))
    assert torch.equal(plain.ids, none.ids) and torch.equal(plain.distances, none.distances)
    with pytest.raises(IndexError):
        index.search(_t(q[:1]), k, exclude=ItemSets.from_lists([[n_items]], device=DEV))



# ----------------------------------------------------------------------------- the feed
def _feed(F=4, n_users=60, items=500, dim=16, seed=2):
    rng = np.random.default_rng(seed)
    lengths = rng.integers(F + 1, 40, n_users)
    lengths[0] = F                                              # exactly F interactions: no window
    hist = [rng.integers(0, 60, n) for n in lengths]            # few items: repeats
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    table = torch.from_numpy(rng.normal(0, 1, (items, dim)).astype(np.float32))
    return DeviceFrameFeed(csr, table, DEV), hist


def test_feed_serving_state_and_seen_items():
    feed, hist = _feed()
    seen = feed.seen_items()
    assert seen is feed.seen_items() and len(seen) == len(hist)
    for u, h in enumerate(hist):
        assert np.array_equal(seen.set(u).cpu().numpy(), np.unique(h)), u
    pos = np.arange(1, len(hist))
    last = feed.csr.win_offsets[pos + 1] - 1
    want = feed.embed(feed.windows(last))["next_state"]
    got = feed.user_states(pos)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    one = feed.user_states([0])                                 # exactly F interactions
    F, D = feed.frame_size, feed.table.shape[1]
    ids = torch.from_numpy(hist[0]).to(DEV)
    assert torch.equal(one[0, :F * D], feed.table[ids].reshape(-1))
    assert torch.equal(one[0, F * D:], feed.hist_ratings[:F])
    short = HistoryCSR([0, 1], [[1, 2, 3, 4, 5], [1, 2]], [[1] * 5, [1] * 2], 4)
    f2 = DeviceFrameFeed(short, feed.table, DEV)
    with pytest.raises(ValueError):
        f2.user_states([1])
    # the serving loop
    S = F * D + F
    torch.manual_seed(0)
    pol = recnn_b200.nn.DiscreteActor(S, feed.table.shape[0], 32).to(DEV)
    v, i = pol.topk(feed.user_states(pos), 10, exclude=seen, exclude_rows=pos)
    got = i.cpu().numpy()
    assert not any(np.isin(got[r], hist[u]).any() for r, u in enumerate(pos))
    index = ItemIndex(feed.table, "IP")
    res = index.search(torch.randn(len(pos), D, device=DEV), 10, exclude=seen, exclude_rows=pos)
    got = res.id().cpu().numpy()
    assert not any(np.isin(got[r], hist[u]).any() for r, u in enumerate(pos))


# ----------------------------------------------------------------------------- 1M items
def test_million_items_long_tailed_sets():
    """S 2570 / H 256, 2^20 items x 2,048 rows with fixed-seed long-tailed sets (mean ~144, some >= 8,192): sampled rows
    against a chunked float64 reference; the call's peak memory is the top-k workspace plus the outputs."""
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
    for j, r in enumerate(rows_chk):                            # make the checked rows' sets bite: their best items
        best = np.argsort(-z[j])[:lengths[r]]
        lists[r] = np.concatenate([best[:lengths[r] // 2], lists[r][:lengths[r] - lengths[r] // 2]])
    print("set lengths: mean %.1f, max %d, >= 8192: %d" % (lengths.mean(), lengths.max(), (lengths >= 8192).sum()))
    sets = ItemSets.from_lists(lists, device=DEV)
    from recnn_b200.nn.update.reinforce import _chunk_items
    ws = L.recnn_discrete_topk_workspace_bytes(m.dims, N, k, _chunk_items(N, I))
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    v, i = m.topk(st, k, exclude=sets)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("1M items x %d rows with sets: peak extra %.3f GB, workspace %.3f GB, table %.1f MB"
          % (N, peak / 1e9, ws / 1e9, (sets.ids.numel() + sets.offsets.numel()) * 8 / 1e6))
    assert peak <= ws + N * k * 12 + (8 << 20)
    check_against_oracle(v[_t(rows_chk)], i[_t(rows_chk)], z, k, padded([lists[r] for r in rows_chk],
                                                                            np.arange(len(rows_chk))),
                         what="1M sets", min_sure=0.5)
