"""Host-side checks of offline evaluation: the rank entry points in the header, the library and the ctypes table; the
refusals of DiscreteActor.rank / ItemIndex.rank before any device work; the leave-last-out plan of a HistoryCSR
against numpy; the ranking metrics against hand-computed values, and their all-reduce through a gloo world of 2.
No kernel is launched."""
from __future__ import annotations

import math
import os
import re
import socket

import numpy as np
import pytest
import torch

import recnn_b200
from recnn_b200 import _lib
from recnn_b200.data import HistoryCSR, ItemIndex, ItemSets
from recnn_b200.utils.metrics import hit_rate, mrr, ndcg, ranking_metrics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NEW_SYMBOLS = ("recnn_discrete_rank_workspace_bytes", "recnn_discrete_rank", "recnn_discrete_rank_sets",
               "recnn_vocab_rank_record_floats", "recnn_discrete_shard_rank_stats", "recnn_discrete_shard_rank",
               "recnn_discrete_shard_rank_sets", "recnn_discrete_shard_rank_finish",
               "recnn_retrieve_rank_workspace_bytes", "recnn_retrieve_rank", "recnn_retrieve_rank_sets")


def test_new_symbols_in_header_library_and_ctypes_table():
    with open(os.path.join(ROOT, "include", "recnn_b200.h")) as fh:
        declared = set(re.findall(r"RECNN_API\s+[\w\s\*]+?\b(recnn_\w+)\s*\(", fh.read()))
    L = _lib.lib()
    for name in NEW_SYMBOLS:
        assert name in declared and name in _lib.SIGNATURES, name
        assert getattr(L, name) is not None
    assert declared <= set(_lib.SIGNATURES), sorted(declared - set(_lib.SIGNATURES))


def test_workspace_and_record_sizes():
    """The rank workspace holds one [N, chunk] logits block (no gradient scratch, no [N, num_items] buffer) and is
    below top-k's at the same chunk; the count record is the header plus N int32 words."""
    L = _lib.lib()
    d = _lib.DiscreteDims(2570, 256, 1 << 20, 0)
    for n, chunk in [(2048, 131072), (128, 1 << 20), (16384, 16384)]:
        ws = L.recnn_discrete_rank_workspace_bytes(d, n, chunk)
        assert n * chunk * 4 < ws < n * (2572 + 256 + chunk + 4) * 4 + 16 * 256
        assert ws <= L.recnn_discrete_topk_workspace_bytes(d, n, 10, chunk)
    assert L.recnn_discrete_rank_workspace_bytes(d, 16, 100) == 0                   # chunk refused
    assert L.recnn_vocab_rank_record_floats(100) == 4 + 100
    assert L.recnn_vocab_rank_record_floats(0) == 0
    assert 0 < L.recnn_retrieve_rank_workspace_bytes(2048, 1 << 20) <= L.recnn_retrieve_workspace_bytes(2048, 1 << 20, 10)


def test_policy_refusals_happen_before_device_work():
    L = _lib.lib()
    torch.manual_seed(0)
    m = recnn_b200.nn.DiscreteActor(6, 10, 8)
    st = torch.zeros(3, 6)
    tgt = torch.tensor([1, 2, 3])
    sets = ItemSets.from_lists([[1], [2, 3]])
    k0 = L.recnn_b200_launch_count()
    with pytest.raises(ValueError, match="state"):
        m.rank(torch.zeros(3, 5), tgt)
    for bad in (torch.tensor([1, 2]), torch.tensor([[1, 2, 3]]), torch.tensor([1.0, 2.0, 3.0]),
                torch.tensor([True, False, True]), [1, 2, 3]):
        with pytest.raises(ValueError, match="target"):
            m.rank(st, bad)
    with pytest.raises(ValueError, match="sets but the call has 3 rows"):
        m.rank(st, tgt, exclude=sets)
    with pytest.raises(ValueError, match="ItemSets"):
        m.rank(st, tgt, exclude=torch.zeros(3, 2, dtype=torch.int64))
    with pytest.raises(ValueError, match="exclude_rows"):
        m.rank(st, tgt, exclude_rows=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(ValueError, match="exclude_rows"):
        m.rank(st, tgt, exclude=sets, exclude_rows=torch.zeros(2, dtype=torch.int64))
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        m.rank(st, tgt, exclude=sets, exclude_rows=torch.tensor([0, -1, 1]))
    with pytest.raises(_lib.RecnnError, match="CUDA only"):
        m.rank(st, tgt.int())
    assert L.recnn_b200_launch_count() == k0


def test_index_refusals_happen_before_device_work():
    idx = ItemIndex.__new__(ItemIndex)                         # an index needs a device table; its checks do not
    idx.dim, idx.n_items = 4, 10
    q = torch.zeros(3, 4)
    with pytest.raises(ValueError, match="search_vecs"):
        idx.rank(torch.zeros(3, 5), torch.tensor([0, 1, 2]))
    for bad in (torch.tensor([0, 1]), torch.tensor([0.0, 1.0, 2.0]), None):
        with pytest.raises(ValueError, match="target"):
            idx.rank(q, bad)
    with pytest.raises(ValueError, match="ItemSets"):
        idx.rank(q, torch.tensor([0, 1, 2]), exclude=[[1], [2], [3]])
    with pytest.raises(ValueError, match="exclude_rows"):
        idx.rank(q, torch.tensor([0, 1, 2]), exclude_rows=torch.zeros(3, dtype=torch.int64))
    with pytest.raises(_lib.RecnnError):
        ItemIndex(torch.zeros(10, 4), "IP")


def test_holdout_plan_against_numpy():
    rng = np.random.default_rng(0)
    F = 3
    lengths = rng.integers(F + 1, 20, 30)
    hist = [rng.integers(0, 50, n) for n in lengths]
    csr = HistoryCSR(np.arange(30), hist, [np.ones(n) for n in lengths], F)
    pos = rng.permutation(30)[:17]
    last = csr.holdout_windows(pos)
    # the collate's windows over all users, in order: user u contributes len_u - F windows
    windows = [(u, i) for u in range(30) for i in range(lengths[u] - F)]
    for w, u in zip(last, pos):
        assert windows[w] == (u, lengths[u] - F - 1)
        first = csr.offsets[u] + windows[w][1]
        assert csr.items[first + F] == hist[u][-1]
    short = HistoryCSR([0, 1, 2], [[1, 2, 3, 4], [1, 2, 3], [1, 2]], [[1] * 4, [1] * 3, [1] * 2], F)
    assert short.holdout_windows([0]).tolist() == [0]
    with pytest.raises(ValueError, match="held-out"):
        short.holdout_windows([0, 1])                          # exactly F items: a state but no window
    with pytest.raises(ValueError, match="fewer than frame_size"):
        short.holdout_windows([2])
    with pytest.raises(IndexError):
        short.holdout_windows([3])


def test_metrics_by_hand():
    r = torch.tensor([0, 1, 4, 9, 30])
    assert hit_rate(r, 1) == pytest.approx(1 / 5)
    assert hit_rate(r, 5) == pytest.approx(3 / 5)
    assert hit_rate(r, 10) == pytest.approx(4 / 5)
    assert ndcg(r, 5) == pytest.approx((1 + 1 / math.log2(3) + 1 / math.log2(6)) / 5)
    assert ndcg(r, 1) == pytest.approx(1 / 5)
    assert mrr(r) == pytest.approx((1 + 1 / 2 + 1 / 5 + 1 / 10 + 1 / 31) / 5)
    m = ranking_metrics(r, ks=(1, 5))
    assert m == pytest.approx({"hit@1": 0.2, "ndcg@1": 0.2, "hit@5": 0.6,
                               "ndcg@5": (1 + 1 / math.log2(3) + 1 / math.log2(6)) / 5,
                               "mrr": (1 + 1 / 2 + 1 / 5 + 1 / 10 + 1 / 31) / 5, "n": 5})
    for bad in (torch.tensor([0.5]), torch.tensor([[1]]), torch.tensor([-1, 2])):
        with pytest.raises(ValueError, match="ranks"):
            mrr(bad)
    with pytest.raises(ValueError, match="k"):
        hit_rate(r, 0)
    empty = ranking_metrics(torch.zeros(0, dtype=torch.int64))
    assert empty["n"] == 0 and math.isnan(empty["mrr"])


def _gloo_worker(rank, world, port, q):
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method="tcp://127.0.0.1:%d" % port, rank=rank, world_size=world)
    try:
        mine = torch.tensor([0, 3, 12]) if rank == 0 else torch.tensor([1, 40])
        q.put((rank, ranking_metrics(mine, ks=(1, 5, 20), group=dist.group.WORLD)))
    finally:
        dist.destroy_process_group()


def test_ranking_metrics_all_reduce_over_gloo():
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = dict(q.get(timeout=120) for _ in range(2))
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = ranking_metrics(torch.tensor([0, 3, 12, 1, 40]), ks=(1, 5, 20))
    assert got[0] == pytest.approx(want) and got[1] == pytest.approx(want) and want["n"] == 5
