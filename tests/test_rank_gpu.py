"""Exact ranks of held-out items on the GPU: DiscreteActor.rank / recnn_discrete_rank(_sets) and the sharded phases, and
ItemIndex.rank, against float64 ranks, against the positions topk / search return on the same inputs and chunking
(the invariant the rank is defined by), across virtual ranks (tests/_ranks.py), at 1M items, and the feed's leave-
last-out rows."""
from __future__ import annotations

import copy
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
from recnn_b200.utils.metrics import ranking_metrics
from tests import _policy_topk_oracle as TK
from tests._discrete import make_policy
from tests._ranks import chunked, returned, run_ranks, shard, spawn
from tests.test_policy_topk_gpu import SHAPES, Z_BAR, _tie_policy, make_case
from tests.test_recommend_gpu import make_sets, padded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.lib()


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def oracle_rank(z, target, exclude=None):
    """(rank, near) float64: the eligible ids that beat the target (higher logit, equal logits the smaller id) and
    the count of eligible ids within the fp32 error bar of it, per row; exclude: padded [N, E] (negative: padding)."""
    n, items = z.shape
    bar = Z_BAR * (1 + np.abs(z).max())
    ok = np.ones(z.shape, dtype=bool)
    if exclude is not None:
        for r, row in enumerate(np.asarray(exclude)):
            ok[r, row[row >= 0]] = False
    ids = np.arange(items)
    rank = np.zeros(n, dtype=np.int64)
    near = np.zeros(n, dtype=np.int64)
    for r in range(n):
        t = target[r]
        ok[r, t] = True                                    # a target is never excluded
        elig = ok[r] & (ids != t)
        zt = z[r, t]
        rank[r] = (elig & ((z[r] > zt) | ((z[r] == zt) & (ids < t)))).sum()
        near[r] = (elig & (np.abs(z[r] - zt) <= bar)).sum()
    return rank, near


def log_softmax_at(z, target):
    M = z.max(1)
    return z[np.arange(len(z)), target] - M - np.log(np.exp(z - M[:, None]).sum(1))


def check_oracle(rank, logp, z, target, exclude=None, what="", min_sure=0.5):
    want, near = oracle_rank(z, target, exclude)
    got = rank.cpu().numpy()
    sure = near == 0
    assert sure.mean() >= min_sure, (what, sure.mean())
    assert np.array_equal(got[sure], want[sure]), (what, np.nonzero(got[sure] != want[sure]))
    assert (np.abs(got - want) <= near).all(), what
    if logp is not None:
        lp = log_softmax_at(z, target)
        err = np.abs(logp.cpu().numpy().astype(np.float64) - lp)
        assert err.max() <= 4 * Z_BAR * (1 + np.abs(z).max()), (what, err.max())
    return int(sure.sum())


def targets_for(z, seed):
    """Targets near the top of each row (ranks 0..~90) and anywhere, so both sides of k = 64 occur."""
    rng = np.random.default_rng(seed)
    n, items = z.shape
    order = np.argsort(-z, 1)
    t = order[np.arange(n), rng.integers(0, min(90, items), n)]
    far = rng.random(n) < 0.3
    t[far] = rng.integers(0, items, far.sum())
    return t.astype(np.int64)


def call_rank(m, state, target, chunk=None, sets=None, rows=None):
    """(rank, log_prob, error bits) of one explicit recnn_discrete_rank(_sets) call."""
    d = m.dims
    n = state.shape[0]
    chunk = d.num_items if chunk is None or chunk >= d.num_items else chunk
    nbytes = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
    assert nbytes > 0
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    rank = torch.empty(n, dtype=torch.int64, device=DEV)
    logp = torch.empty(n, device=DEV)
    flag = torch.full((1,), 7, dtype=torch.int32, device=DEV)
    tgt = _t(np.asarray(target, dtype=np.int64))
    if sets is None:
        _lib.check(L.recnn_discrete_rank(d, param_arena(m).data_ptr(), state.data_ptr(), tgt.data_ptr(), n, chunk,
                                         rank.data_ptr(), logp.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                         _lib.stream_ptr()))
    else:
        sid, off = (sets.ids, sets.offsets) if isinstance(sets, ItemSets) else sets
        rows = None if rows is None else _t(np.asarray(rows, dtype=np.int64))
        _lib.check(L.recnn_discrete_rank_sets(d, param_arena(m).data_ptr(), state.data_ptr(), tgt.data_ptr(), n,
                                              sid.data_ptr() if sid.numel() else None, sid.numel(), off.data_ptr(),
                                              off.numel() - 1, _lib.ptr(rows), chunk, rank.data_ptr(),
                                              logp.data_ptr(), flag.data_ptr(), ws.data_ptr(), nbytes,
                                              _lib.stream_ptr()))
    torch.cuda.synchronize()
    return rank, logp, int(flag)


def positions(ids, target):
    """Position of target[r] in ids[r] (numpy), -1 when absent."""
    hit = ids == target[:, None]
    return np.where(hit.any(1), hit.argmax(1), -1)


def check_topk_consistency(rank, topk_ids, target, what=""):
    """target at position rank of topk(64) when rank < 64, absent otherwise (rows whose target is not excluded)."""
    got = rank.cpu().numpy()
    pos = positions(topk_ids.cpu().numpy(), target)
    k = topk_ids.shape[1]
    assert np.array_equal(pos, np.where(got < k, got, -1)), (what, np.nonzero(pos != np.where(got < k, got, -1)))
    assert (got < k).any() and (got >= k).any(), what


def sets_without_target(z, k, seed, target):
    lists, rows = make_sets(z, k, seed)
    for r, s in enumerate(rows):                    # the invariant with topk is for targets outside their set
        if s >= 0:
            lists[s] = lists[s][lists[s] != target[r]]
    for r, s in enumerate(rows):
        if s >= 0 and np.isin(target[r], lists[s]):
            rows[r] = -1
    return lists, rows


# ----------------------------------------------------------------------------- 1. float64 oracle, both back ends
def run_sweep():
    for S, H, I, N in SHAPES:
        p, state = make_case(S, H, I, N, 5 * S + I)
        m = make_policy(p, S, H, I)
        st = _t(state)
        z = TK.logits(p, state)
        target = targets_for(z, S)
        lists, rows = make_sets(z, 17, S)
        sets = ItemSets.from_lists(lists, device=DEV)
        ex = padded(lists, rows)
        for chunk in (None, 128, 256):
            rank, logp, flag = call_rank(m, st, target, chunk)
            assert flag == 0
            check_oracle(rank, logp, z, target, what=(S, I, chunk))
            rank_s, logp_s, flag = call_rank(m, st, target, chunk, sets, rows)
            assert flag == 0
            check_oracle(rank_s, logp_s, z, target, ex, what=(S, I, chunk, "sets"))
            assert torch.equal(logp_s, logp)
            assert bool((rank_s <= rank).all())
        print("rank S %d I %d N %d: ok" % (S, I, N))


def test_against_float64():
    run_sweep()


def test_against_float64_on_the_cuda_core_back_end():
    code = "import sys; sys.path.insert(0, %r); from tests import test_rank_gpu as T; T.run_sweep()" % ROOT
    env = dict(os.environ, RECNN_B200_MATH="simt")
    r = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, cwd=ROOT)
    print(r.stdout[-3000:], r.stderr[-3000:])
    assert r.returncode == 0


# ----------------------------------------------------------------------------- 2. consistency with topk
@pytest.mark.parametrize("S,H,I,N", SHAPES)
def test_rank_is_the_position_in_topk(S, H, I, N):
    p, state = make_case(S, H, I, N, 7 * S + I)
    m = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    target = targets_for(z, I)
    lists, rows = sets_without_target(z, 64, I, target)
    sets = ItemSets.from_lists(lists, device=DEV)
    tgt = _t(target)
    for chunk in (None, 128, 256):
        with chunked(N, chunk):
            rank, logp = m.rank(st, tgt)
            _, ids = m.topk(st, 64)
            check_topk_consistency(rank, ids, target, (S, I, chunk))
            rank_s, logp_s = m.rank(st, tgt, exclude=sets, exclude_rows=_t(rows))
            _, ids_s = m.topk(st, 64, exclude=sets, exclude_rows=_t(rows))
            check_topk_consistency(rank_s, ids_s, target, (S, I, chunk, "sets"))
            again = m.rank(st, tgt, exclude=sets, exclude_rows=_t(rows))
        assert torch.equal(again[0], rank_s) and torch.equal(again[1].view(torch.int32), logp_s.view(torch.int32))
        r2, l2, _ = call_rank(m, st, target, chunk, sets, rows)
        assert torch.equal(r2, rank_s) and torch.equal(l2, logp_s)


def test_exact_ties_and_sets_across_chunk_edges():
    groups = [[500, 3, 128, 127, 129], [255, 256, 1002]]           # across the 128- and 256-chunk edges
    p, state = _tie_policy(1003, groups)
    m = make_policy(p, 36, 32, 1003)
    st = _t(state)
    N = state.shape[0]
    tied = sorted(groups[0]) + sorted(groups[1])
    target = np.array([tied[r % len(tied)] for r in range(N)], dtype=np.int64)
    lists = [[x for x in (127, 128, 129, 255, 256, 3) if x != target[r]] for r in range(N)]
    lists[::3] = [[] for _ in lists[::3]]
    sets = ItemSets.from_lists(lists, device=DEV)
    for chunk in (None, 128, 256):
        with chunked(N, chunk):
            rank, _ = m.rank(st, _t(target))
            assert np.array_equal(rank.cpu().numpy(), np.array([tied.index(t) for t in target])), chunk
            _, ids = m.topk(st, 64)
            assert np.array_equal(positions(ids.cpu().numpy(), target), rank.cpu().numpy())
            rank_s, _ = m.rank(st, _t(target), exclude=sets)
            _, ids_s = m.topk(st, 64, exclude=sets)
            assert np.array_equal(positions(ids_s.cpu().numpy(), target), rank_s.cpu().numpy()), chunk
            want = [sum(1 for x in tied[:tied.index(t)] if x not in lists[r]) for r, t in enumerate(target)]
            assert np.array_equal(rank_s.cpu().numpy(), want), chunk


# ----------------------------------------------------------------------------- 3. exclusion semantics, errors
def test_exclusion_semantics_and_errors():
    S, H, I, N = 37, 32, 2000, 40
    p, state = make_case(S, H, I, N, 17)
    m = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    target = targets_for(z, 3)
    tgt = _t(target)
    order = np.argsort(-z, 1)
    base = [order[r, :50] for r in range(N)]
    for chunk in (None, 128):
        with chunked(N, chunk):
            plain, _ = m.rank(st, tgt)
            without = m.rank(st, tgt, exclude=ItemSets.from_lists([b[b != t] for b, t in zip(base, target)],
                                                                   device=DEV))[0]
            with_t = m.rank(st, tgt, exclude=ItemSets.from_lists([np.append(b, t) for b, t in zip(base, target)],
                                                                  device=DEV))[0]
            assert torch.equal(with_t, without), chunk                     # the target is never excluded
            dup = m.rank(st, tgt, exclude=ItemSets.from_lists([np.concatenate([b, b[:20], b[:5]]) for b in base],
                                                               device=DEV))[0]
            assert torch.equal(dup, without), chunk                        # repeated ids count once
            cover = [order[r, :int(plain[r]) + 1] for r in range(N)]       # everything that beats t (and t)
            zero = m.rank(st, tgt, exclude=ItemSets.from_lists(cover, device=DEV))[0]
            sure = oracle_rank(z, target)[1] == 0
            assert bool((zero.cpu()[torch.from_numpy(sure)] == 0).all()), chunk
    with pytest.raises(IndexError):
        m.rank(st, _t(np.where(np.arange(N) == 4, I, target)))
    with pytest.raises(IndexError):
        m.rank(st, _t(np.where(np.arange(N) == 4, -1, target)))
    _, _, flag = call_rank(m, st, np.where(np.arange(N) == 4, I, target))
    assert flag == 1
    with pytest.raises(IndexError):
        m.rank(st, tgt, exclude=ItemSets.from_lists([[I]] * N, device=DEV))
    good = ItemSets.from_lists(base, device=DEV)
    unsorted = ItemSets.from_lists(base, device=DEV)
    unsorted.ids[[3, 4]] = unsorted.ids[[4, 3]].clone()
    with pytest.raises(ValueError):
        m.rank(st, tgt, exclude=unsorted)
    with pytest.raises(ValueError):
        m.rank(st, tgt, exclude=good, exclude_rows=torch.full((N,), N, device=DEV))
    assert call_rank(m, st, target, None, unsorted, None)[2] == 4


# ----------------------------------------------------------------------------- 4. virtual ranks
def sharded_rank(full, world, state, target, chunk=None, sets=None, rows=None, order=None, topk=False):
    def rank(r):
        pol = shard({"policy_net": full})[0]["policy_net"]
        out = pol.rank(state, target, exclude=sets, exclude_rows=rows)
        return out + (pol.topk(state, 64, exclude=sets, exclude_rows=rows) if topk else ())
    with chunked(state.shape[0], chunk):
        return run_ranks(world, rank, order=order)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_virtual_ranks(world):
    S, H, I, N = 52, 64, 1003, 40
    p, state = make_case(S, H, I, N, world + 70)
    full = make_policy(p, S, H, I)
    st = _t(state)
    z = TK.logits(p, state)
    edges = sorted({e for lo, hi in TK.item_plan(I, world) for e in (lo - 1, lo, hi - 1) if 0 <= e < I})
    target = targets_for(z, world)
    target[:len(edges)] = edges                                     # targets on the shard edges
    tgt = _t(target)
    order = np.argsort(-z, 1)
    lists = [np.concatenate([[e for e in edges if e != target[r]], order[r, :30 + r]]) for r in range(N)]
    lists = [x[x != target[r]] for r, x in enumerate(lists)]
    sets = ItemSets.from_lists(lists, device=DEV)
    for ex in (None, sets):
        for chunk in (None, 128):
            res = returned(sharded_rank(full, world, st, tgt, chunk, ex, topk=True))
            rank, logp = res[0][0], res[0][1]
            for x in res[1:]:
                assert torch.equal(x[0], rank) and torch.equal(x[1].view(torch.int32), logp.view(torch.int32))
            check_topk_consistency(rank, res[0][3], target, ("W", world, chunk, ex is not None))
            check_oracle(rank, logp, z, target, None if ex is None else padded(lists, np.arange(N)),
                         what=("W", world, chunk))
            if world == 1:
                with chunked(N, chunk):
                    one = full.rank(st, tgt, exclude=ex)
                assert torch.equal(one[0], rank) and torch.equal(one[1].view(torch.int32), logp.view(torch.int32))
    if world > 1:
        for i in (0, 1):                                            # either all-gather out of rank order
            res = sharded_rank(full, world, st, tgt, order={i: [1, 0] + list(range(2, world))})
            assert all(isinstance(e, RuntimeError) and "disagree on the vocabulary shard plan" in str(e)
                       for e in res), res
    res = sharded_rank(full, world, st, _t(np.where(np.arange(N) == 2, I, target)))
    assert all(isinstance(e, IndexError) for e in res), res


def _rank_worker(rank, world, port, q):
    import torch.distributed as dist
    from recnn_b200 import dist as D
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        S, H, I, N = 52, 64, 1003, 48
        p, state = make_case(S, H, I, N, 78)
        m = make_policy(p, S, H, I).to(dev)
        D.enable_vocab_parallel(m)
        z = TK.logits(p, state)
        target = torch.from_numpy(targets_for(z, 5)).to(dev)
        sets = ItemSets.from_lists([np.arange(r, 3 * r + 1) % I for r in range(N)], device=dev)
        r_, lp = m.rank(torch.from_numpy(state).to(dev), target, exclude=sets)
        q.put((rank, r_.cpu().numpy(), lp.cpu().numpy()))
        torch.cuda.synchronize()
        m.__dict__["_recnn_vp"].comm.close()
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 4, 8])
def test_multi_process_matches_float64(world):
    if torch.cuda.device_count() < world:
        pytest.skip("needs %d GPUs" % world)
    res = {r: (a, b) for r, a, b in spawn(_rank_worker, world)}
    S, H, I, N = 52, 64, 1003, 48
    p, state = make_case(S, H, I, N, 78)
    z = TK.logits(p, state)
    target = targets_for(z, 5)
    for r in range(world):
        assert np.array_equal(res[r][0], res[0][0]) and np.array_equal(res[r][1].view(np.int32), res[0][1].view(np.int32))
    lists = [np.arange(r, 3 * r + 1) % I for r in range(N)]
    check_oracle(torch.from_numpy(res[0][0]), torch.from_numpy(res[0][1]), z, target, padded(lists, np.arange(N)),
                 what=("processes", world))


# ----------------------------------------------------------------------------- 5. retrieval
def _index_case(metric, n_items, dim, n, seed):
    rng = np.random.default_rng(seed)
    table = rng.normal(0, 1, (n_items, dim)).astype(np.float32)
    q = rng.normal(0, 1, (n, dim)).astype(np.float32)
    t64, q64 = table.astype(np.float64), q.astype(np.float64)
    if metric == "L2":
        key = (t64 ** 2).sum(1)[None] - 2 * q64 @ t64.T
    elif metric == "IP":
        key = -(q64 @ t64.T)
    else:
        key = -(q64 @ t64.T) / np.linalg.norm(t64, axis=1)[None]
    return table, q, key


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_index_rank(metric):
    # 100,003 items: 128 queries per slab, so 300 queries take three slabs
    for n_items, dim, n in ((5003, 64, 70), (100003, 32, 300)):
        table, q, key = _index_case(metric, n_items, dim, n, n_items)
        index = ItemIndex(_t(table), metric)
        target = targets_for(-key, n)
        tgt = _t(target)
        qd = _t(q)
        rank = index.rank(qd, tgt)
        res = index.search(qd, 64)
        check_topk_consistency(rank, res.ids, target, (metric, n_items))
        scale = 1e-4 * (1 + np.abs(key).max())
        want = np.array([((key[r] < key[r, t]) | ((key[r] == key[r, t]) & (np.arange(n_items) < t))).sum()
                         for r, t in enumerate(target)])
        near = np.array([(np.abs(key[r] - key[r, t]) <= scale).sum() - 1 for r, t in enumerate(target)])
        got = rank.cpu().numpy()
        sure = near == 0
        assert sure.mean() >= 0.3 and np.array_equal(got[sure], want[sure]), metric
        assert (np.abs(got - want) <= near).all(), metric
        lists, rows = sets_without_target(-key, 64, 3, target)
        sets = ItemSets.from_lists(lists, device=DEV)
        rank_s = index.rank(qd, tgt, exclude=sets, exclude_rows=_t(rows))
        res_s = index.search(qd, 64, exclude=sets, exclude_rows=_t(rows))
        check_topk_consistency(rank_s, res_s.ids, target, (metric, n_items, "sets"))
        assert torch.equal(index.rank(qd, tgt, exclude=sets, exclude_rows=_t(rows)), rank_s)
        none = index.rank(qd, tgt, exclude=sets, exclude_rows=torch.full((n,), -1, device=DEV))
        assert torch.equal(none, rank)
    with pytest.raises(IndexError):
        index.rank(qd[:2], torch.tensor([0, n_items], device=DEV))
    with pytest.raises(IndexError):
        index.rank(qd[:1], tgt[:1], exclude=ItemSets.from_lists([[n_items]], device=DEV))


# ----------------------------------------------------------------------------- 6. 1M items
def test_million_items_memory_and_sampled_rows():
    """S 2570 / H 256, 2^20 items x 2,048 rows with long-tailed sets: the call's extra memory is the rank workspace plus
    the outputs (no [N, num_items] buffer), and sampled rows match a chunked float64 rank."""
    S, H, I, N = 2570, 256, 1 << 20, 2048
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(S, I, H).to(DEV)
    with torch.no_grad():
        m.linear2.weight.mul_(8.0)
    st = torch.randn(N, S, device=DEV)
    rng = np.random.default_rng(145)
    rows_chk = np.arange(0, N, N // 16)
    with torch.no_grad():
        x = st[_t(rows_chk)].double()
        h = torch.relu(x @ m.linear1.weight.double().T + m.linear1.bias.double())
        z = torch.cat([h @ m.linear2.weight[c:c + 65536].double().T + m.linear2.bias[c:c + 65536].double()
                       for c in range(0, I, 65536)], 1).cpu().numpy()
    target = rng.integers(0, I, N)
    target[rows_chk] = targets_for(z, 1)
    lengths = np.minimum(rng.pareto(1.6, N) * 75 + 20, 20000).astype(np.int64)
    lists = [rng.integers(0, I, n) for n in lengths]
    for j, r in enumerate(rows_chk):
        best = np.argsort(-z[j])[:lengths[r]]
        lists[r] = np.concatenate([best[:lengths[r] // 2], lists[r][:lengths[r] - lengths[r] // 2]])
    sets = ItemSets.from_lists(lists, device=DEV)
    tgt = _t(target)
    from recnn_b200.nn.update.reinforce import _chunk_items
    ws = L.recnn_discrete_rank_workspace_bytes(m.dims, N, _chunk_items(N, I))
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    rank, logp = m.rank(st, tgt, exclude=sets)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print("1M items x %d rows: rank peak extra %.3f GB, workspace %.3f GB" % (N, peak / 1e9, ws / 1e9))
    assert peak <= ws + N * 12 + (8 << 20)
    assert peak < N * I * 4 / 4
    sel = _t(rows_chk)
    check_oracle(rank[sel], logp[sel], z, target[rows_chk], padded([lists[r] for r in rows_chk],
                                                                     np.arange(len(rows_chk))), what="1M", min_sure=0.3)
    plain, _ = m.rank(st[sel], tgt[sel])
    _, ids = m.topk(st[sel], 64)
    check_topk_consistency(plain, ids, target[rows_chk], "1M topk")


# ----------------------------------------------------------------------------- 7. the feed
def test_feed_holdout_rows_and_metrics():
    rng = np.random.default_rng(4)
    F, n_users, items, dim = 4, 50, 300, 16
    lengths = rng.integers(F + 1, 40, n_users)
    hist = [rng.integers(0, 80, n) for n in lengths]
    rat = [rng.integers(1, 6, n).astype(np.float32) for n in lengths]
    csr = HistoryCSR(np.arange(n_users), hist, rat, F)
    feed = DeviceFrameFeed(csr, torch.from_numpy(rng.normal(0, 1, (items, dim)).astype(np.float32)), DEV)
    pos = np.arange(n_users)[::-1].copy()
    h = feed.holdout(pos)
    last = csr.win_offsets[pos + 1] - 1
    want = feed.embed(feed.windows(last))["state"]
    assert torch.equal(h["state"].view(torch.int32), want.view(torch.int32))
    assert np.array_equal(h["target"].cpu().numpy(), [hist[u][-1] for u in pos])
    assert np.array_equal(h["exclude_rows"].cpu().numpy(), pos)
    torch.manual_seed(1)
    pol = recnn_b200.nn.DiscreteActor(F * dim + F, items, 32).to(DEV)
    seen = feed.seen_items()
    ranks, logp = pol.rank(h["state"], h["target"], exclude=seen, exclude_rows=h["exclude_rows"])
    # the whole history holds the target, which is never excluded: the same ranks as "rated before the last item"
    earlier = ItemSets.from_lists([hist[u][:-1] for u in pos], device=DEV)
    before, _ = pol.rank(h["state"], h["target"], exclude=earlier)
    assert torch.equal(before, ranks)
    _, ids = pol.topk(h["state"], 64, exclude=earlier)
    got = ranks.cpu().numpy()
    tg = h["target"].cpu().numpy()
    checked = 0
    for r, u in enumerate(pos):
        if tg[r] not in set(hist[u][:-1].tolist()):                  # the target is eligible to topk
            p_ = positions(ids[r:r + 1].cpu().numpy(), tg[r:r + 1])[0]
            assert p_ == (got[r] if got[r] < 64 else -1), r
            checked += 1
    assert checked > 0
    met = ranking_metrics(ranks)
    assert met["n"] == n_users and 0 <= met["mrr"] <= 1
    short = HistoryCSR([0, 1], [[1, 2, 3, 4, 5], [1, 2, 3, 4]], [[1] * 5, [1] * 4], 4)
    with pytest.raises(ValueError):
        DeviceFrameFeed(short, feed.table, DEV).holdout([1])


# ----------------------------------------------------------------------------- 8. the policy's saved state
def test_rank_leaves_the_policy_state_alone():
    S, H, I, N = 20, 16, 300, 8
    p, state = make_case(S, H, I, N, 9)
    m = make_policy(p, S, H, I)
    st = _t(state)
    m.select_action(st)
    saved = (len(m.saved_log_probs), len(m._saved), m._draws)
    snap = [dict(x) for x in m._saved]
    logp0 = m.saved_log_probs[0].clone()
    arena = param_arena(m).clone()
    rank, logp = m.rank(st, m._saved[0]["action"])
    twin = copy.deepcopy(m)
    assert (len(m.saved_log_probs), len(m._saved), m._draws) == saved
    assert torch.equal(m.saved_log_probs[0], logp0) and torch.equal(param_arena(m), arena)
    assert all(torch.equal(a["state"], b["state"]) and torch.equal(a["action"], b["action"])
               for a, b in zip(m._saved, snap))
    r2, l2 = twin.rank(st, m._saved[0]["action"])
    assert torch.equal(r2, rank) and torch.equal(l2, logp)
    # the drawn action's log-prob is the sampler's within the clamp
    assert torch.allclose(logp, logp0, atol=1e-4)
