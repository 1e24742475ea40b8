"""The graph-index oracle on the host (tests/_graph_oracle.py) and the C ABI of recnn_graph_build / recnn_graph_search."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest
import torch

from recnn_b200 import _lib
from recnn_b200.data.db_con import graph_entry_points
from tests import _exact_retrieval as X
from tests import _graph_oracle as G


def _check_graph(graph, d):
    n = graph.shape[0]
    assert graph.shape == (n, d)
    for u in range(n):
        assert len(set(graph[u].tolist())) == d and u not in graph[u]


def test_detour_count_reorders_the_kept_edges():
    # N(0) = [1, 2, 3, 4].  The count c_j of node 0, over the lists of the nodes before j:
    #   j = 1 (item 2): N(1) holds 2 at p = 0 < 1                                  -> c = 1
    #   j = 2 (item 3): N(1) holds 3 at p = 1 < 2, N(2) at p = 0                   -> c = 2
    #   j = 3 (item 4): N(1), N(2) hold 4 at p = 3, N(3) at p = 3: none with p < 3 -> c = 0
    # so (c, j) order is j = 0, 3, 1, 2: the farthest neighbour 4 is kept over 2 and 3, reachable through 1
    knn = np.array([[1, 2, 3, 4],
                    [2, 3, 0, 4],
                    [3, 1, 0, 4],
                    [0, 1, 2, 4],
                    [0, 1, 2, 3]])
    P = G.prune(knn, 2)
    assert P[0].tolist() == [1, 4]
    assert G.prune(knn, 4)[0].tolist() == [1, 4, 2, 3]
    assert P.shape == (5, 2)


def test_reverse_and_merge_fill_with_the_duplicate_skip():
    # d = 4: P(0) = [1, 2, 3, 4]; reverse candidates of 0 come from every node listing it, by (rank, id)
    P = np.array([[1, 2, 3, 4],
                  [0, 2, 3, 4],
                  [0, 1, 3, 4],
                  [1, 0, 2, 4],
                  [2, 3, 1, 0],
                  [0, 1, 2, 3]])
    g = G.reverse_merge(P)
    # node 0: first half [1, 2]; reverse candidates (r, u): (0, 1), (0, 2), (0, 5), (1, 3), (3, 4) -> 1, 2 skipped,
    # then 5 and 3
    assert g[0].tolist() == [1, 2, 5, 3]
    # node 5: first half [0, 1]; no reverse candidates; the rest of P(5): 2, 3
    assert g[5].tolist() == [0, 1, 2, 3]
    _check_graph(g, 4)


@pytest.mark.parametrize("d,D", [(16, 32), (32, 64), (64, 64)])
def test_oracle_graph_has_d_distinct_neighbours(d, D):
    rng = np.random.default_rng(d + D)
    x = rng.standard_normal((300, 8)).astype(np.float32)
    t = torch.from_numpy(x)
    keys = X.keys32(X.scores64(t, t, None), X.norms32(t, "L2", None), "L2").numpy()
    knn = G.exact_knn(keys, D)
    assert not (knn == np.arange(300)[:, None]).any()
    _check_graph(G.build(knn, d), d)


@pytest.mark.parametrize("metric", ["L2", "IP", "COS"])
def test_replay_on_a_complete_graph_is_exact_topk(metric):
    rng = np.random.default_rng(5)
    n = 40
    table, queries = X.small_ints(rng, (n, 6)), X.small_ints(rng, (5, 6))
    graph = np.array([[v for v in range(n) if v != u] for u in range(n)])
    keys = X.keys32(X.scores64(queries, table), X.norms32(table, metric), metric).numpy()
    qn = X.qnorm32(queries)
    finish = lambda r, kk: X.finish32(torch.from_numpy(kk)[None], qn[r:r + 1], metric)[0].numpy()
    pad = X.FLT_MAX if metric == "L2" else -X.FLT_MAX
    entry = graph_entry_points(n, 0).numpy()
    for T, W in [(32, 1), (64, 2)]:
        ids, dist, _ = G.search(keys, graph, entry, T, W, 0, 10, finish, pad)
        want_i, want_d = X.topk(queries, table, metric, 10)
        np.testing.assert_array_equal(ids, want_i)
        np.testing.assert_array_equal(dist, want_d)


def test_replay_caps_iterations_and_pads():
    rng = np.random.default_rng(6)
    n = 50
    keys = rng.standard_normal((1, n)).astype(np.float32)
    graph = np.array([[(u + s) % n for s in range(1, 17)] for u in range(n)])
    entry = np.arange(n)[::-1]
    buf, it = G.replay(keys[0], graph, entry, 32, 1, 2)
    assert it == 2
    buf, it = G.replay(keys[0], graph, entry, 32, 1, 0)
    assert it >= 2 and sum(i != G.NO_ID for _, i in buf) == 32
    ex = [list(range(n))]
    ids, dist, _ = G.search(keys, graph, entry, 32, 1, 0, 5, lambda r, kk: kk, X.FLT_MAX, exclude=ex)
    assert (ids == -1).all() and (dist == X.FLT_MAX).all()


def test_hash_clears_leave_the_replay_unchanged():
    # the device's visited hash is a model of the "already in the buffer" check; the oracle counts its clears
    rng = np.random.default_rng(9)
    n = 3000
    keys = rng.standard_normal(n).astype(np.float32)
    graph = np.array([rng.choice(np.delete(np.arange(n), u), 32, replace=False) for u in range(n)])
    entry = graph_entry_points(n, 0).numpy()
    assert G.hash_clears(keys, graph, entry, 256, 8, hash_fill=300) >= 2
    assert G.hash_clears(keys, graph, entry, 256, 8, hash_fill=10 ** 9) == 0


def test_entry_points_are_a_seeded_permutation_prefix():
    e = graph_entry_points(1000, 3)
    g = torch.Generator().manual_seed(3)
    np.testing.assert_array_equal(e.numpy(), torch.randperm(1000, generator=g)[:512].numpy())
    assert len(graph_entry_points(100, 0)) == 100


def test_graph_symbols_are_bound():
    for name in ("recnn_graph_build_workspace_bytes", "recnn_graph_build", "recnn_graph_search_workspace_bytes",
                 "recnn_graph_search", "recnn_sizeof_graph_index"):
        assert name in _lib.SIGNATURES


def test_argument_structs_match_the_library():
    L = _lib.lib()
    assert L.recnn_sizeof_graph_index() == ctypes.sizeof(_lib.GraphIndex)
    assert L.recnn_sizeof_graph_build_args() == ctypes.sizeof(_lib.GraphBuildArgs)
    assert L.recnn_sizeof_graph_search_args() == ctypes.sizeof(_lib.GraphSearchArgs)
    for i, f in enumerate(_lib.GRAPH_BUILD_PROBE_FIELDS):
        assert L.recnn_offsetof_graph_build_args(i) == getattr(_lib.GraphBuildArgs, f).offset, f
    for i, f in enumerate(_lib.GRAPH_SEARCH_PROBE_FIELDS):
        assert L.recnn_offsetof_graph_search_args(i) == getattr(_lib.GraphSearchArgs, f).offset, f
    assert L.recnn_offsetof_graph_build_args(len(_lib.GRAPH_BUILD_PROBE_FIELDS)) == -1
    assert L.recnn_offsetof_graph_search_args(len(_lib.GRAPH_SEARCH_PROBE_FIELDS)) == -1


def test_calls_refuse_bad_arguments_before_device_work():
    L = _lib.lib()
    before = L.recnn_b200_launch_count()
    assert L.recnn_graph_search(None, None) == -1 and L.recnn_graph_build(None, None) == -1
    idx = _lib.GraphIndex(1000, 16, _lib.METRIC_L2, 32, 512, 256, 256, 256, 256)
    ws = L.recnn_graph_search_workspace_bytes(4, 64)
    a = _lib.GraphSearchArgs(idx, 256, 4, 10, 64, 1, 0, None, 0, None, 0, None, 256, 256, None, None, 256, ws)
    for field, bad in [("itopk", 48), ("itopk", 288), ("k", 65), ("search_width", 0), ("search_width", 17),
                       ("max_iterations", -1)]:
        keep = getattr(a, field)
        setattr(a, field, bad)
        assert L.recnn_graph_search(ctypes.byref(a), None) == -1, field
        setattr(a, field, keep)
    a.k, a.itopk = 40, 32
    assert L.recnn_graph_search(ctypes.byref(a), None) == -1                 # k > itopk
    a.k, a.itopk = 10, 64
    a.index.degree = 24
    assert L.recnn_graph_search(ctypes.byref(a), None) == -1                 # degree not in {16, 32, 64}
    a.index.degree, a.search_width = 64, 9
    assert L.recnn_graph_search(ctypes.byref(a), None) == -1                 # W * d > 512
    a.search_width, a.index.norms = 1, None
    assert L.recnn_graph_search(ctypes.byref(a), None) == -1                 # L2 without norms
    a.index.norms, a.index.dim = 256, 513
    assert L.recnn_graph_search(ctypes.byref(a), None) == -1                 # dim > 512
    a.index.dim, a.workspace_bytes = 16, ws - 1
    assert L.recnn_graph_search(ctypes.byref(a), None) == -3                 # one byte short
    bws = L.recnn_graph_build_workspace_bytes(1000, 32)
    b = _lib.GraphBuildArgs(idx, 256, 64, 0, 256, 256, bws - 1)
    b.index.degree = 32
    assert L.recnn_graph_build(ctypes.byref(b), None) == -3                  # one byte short
    b.workspace_bytes = bws
    b.knn_degree = 16
    assert L.recnn_graph_build(ctypes.byref(b), None) == -1                  # knn_degree < degree
    b.knn_degree = 65
    assert L.recnn_graph_build(ctypes.byref(b), None) == -1                  # knn_degree > 64
    b.knn_degree, b.error_flag = 64, None
    assert L.recnn_graph_build(ctypes.byref(b), None) == -1
    b.error_flag, b.index.n_items, b.index.degree = 256, 2 ** 25, 64
    assert L.recnn_graph_build(ctypes.byref(b), None) == -1                  # n_items * degree = 2^31
    assert L.recnn_b200_launch_count() == before


def test_workspace_queries_need_only_sizes():
    L = _lib.lib()
    a = L.recnn_graph_search_workspace_bytes(2048, 64)
    assert a > 0 and a == L.recnn_graph_search_workspace_bytes(2048, 64)
    assert L.recnn_graph_search_workspace_bytes(2048, 256) > a
    assert L.recnn_graph_search_workspace_bytes(2048, 48) == 0              # not a multiple of 32
    b = L.recnn_graph_build_workspace_bytes(100000, 32)
    assert b > 100000 * 32 * (4 + 16 + 8)
    assert L.recnn_graph_build_workspace_bytes(100000, 64) > b
    assert L.recnn_graph_build_workspace_bytes(32, 32) == 0                 # n_items <= degree
    assert L.recnn_graph_build_workspace_bytes(1000, 24) == 0
    assert L.recnn_graph_build_workspace_bytes(2 ** 25, 64) == 0              # n_items * degree reaches 2^31
    assert L.recnn_graph_build_workspace_bytes(2 ** 25 - 1, 64) > 0
